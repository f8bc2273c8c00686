"""Helper executed in a fresh interpreter by tests/test_gpu_seg_iou.py (install() rewires
sys.modules, so it must not run inside the pytest process).

    python tests/_dropin_seg_iou_run.py <reference_root> <device>

Does what part-seg/train.py:79-96 does in a test epoch, with the reference's own
models/segmenter.py Model on top of install()'s modules: test_model() on the device, then
models.losses.compute_iou(score.cpu(), seg.cpu(), label.cpu(), visualizer, opt, pc). The result must
equal the reference's own compute_iou (loaded from the same bytecode tree under another module name)
on the same tensors, and the kernel's result on the device tensors."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

ref_root, device = sys.argv[1], sys.argv[2]

import sonet_b200.install as inst  # noqa: E402
from sonet_b200 import ops  # noqa: E402

inst.install(ref_root)
from models import losses, segmenter  # noqa: E402  (segmenter is the reference's file)
import sonet_b200.losses  # noqa: E402

from helpers import build_states, golden, golden_case  # noqa: E402
from oracle import seg_iou_golden  # noqa: E402

assert losses is sonet_b200.losses
assert os.path.abspath(segmenter.__file__).startswith(os.path.abspath(ref_root)), segmenter.__file__
ref_losses = seg_iou_golden.load_ref_losses("ref_models_losses")
assert os.path.abspath(ref_losses.__file__).startswith(os.path.abspath(ref_root)), ref_losses.__file__

g = golden("segmenter_b2_n128")
opt, inp, seed = golden_case(g, "segmenter")
opt.device = torch.device(device)
opt.gpu_id = torch.device(device).index or 0
st = build_states("segmenter", opt, seed)
model = segmenter.Model(opt)
model.encoder.load_state_dict(st["encoder"])
model.segmenter.load_state_dict(st["head"])
B, N = int(g["B"]), int(g["N"])
rs = np.random.RandomState(11)
seg = torch.from_numpy(np.stack([rs.choice(ops.SHAPENET_PART_TABLE[int(k)], size=N)
                                 for k in inp["label"]]).astype(np.int64))
model.set_input(inp["pc"], inp["sn"], inp["label"], seg, inp["node"], inp["node_knn_I"])
model.test_model()
pc = inp["pc"]

args = (model.score_segmenter.cpu().data, model.input_seg.cpu().data, model.input_label.cpu().data,
        None, opt, pc.cpu().data)
got = losses.compute_iou(*args)                       # part-seg/train.py:95
want = ref_losses.compute_iou(*args)
assert type(got) is type(want) and got == want, (got, want)
per_shape = losses.compute_iou_np_array(*args)
assert np.array_equal(per_shape, ref_losses.compute_iou_np_array(*args))
on_device = losses.compute_iou_np_array(model.score_segmenter.data, model.input_seg,
                                        model.input_label, None, opt, pc)
assert np.array_equal(on_device, per_shape)
print("compute_iou %r == reference, per shape %s" % (got, per_shape))
print("SEG_IOU_DROPIN_OK")
