"""Part-segmentation IoU on the H100: the sm_90a kernel (csrc/seg_iou.cu) against the reference's
outputs (tests/golden/seg_iou.npz) and the host entry, its optional outputs, CUDA-graph replay, the
PartSegIoU accumulator, and part-seg/train.py's metric call under install()."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import golden

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = golden("seg_iou")
CASES = [str(c) for c in G["cases"]]
DEV = "cuda:0"


def case(tag, device=DEV):
    return (torch.from_numpy(G[tag + "_score"]).to(device),
            torch.from_numpy(G[tag + "_seg"]).to(device),
            torch.from_numpy(G[tag + "_label"]).to(device))


def random_batch(B, C, N, seed, ties=False):
    g = torch.Generator().manual_seed(seed)
    if ties:
        score = torch.randint(0, 3, (B, C, N), generator=g).float()
    else:
        score = torch.randn(B, C, N, generator=g)
        score[:, 7, ::11] = float("nan")
    label = torch.randint(0, 16, (B,), generator=g)
    seg = torch.randint(-2, C + 2, (B, N), generator=g)
    return score, seg, label


@pytest.mark.parametrize("tag", CASES)
def test_kernel_reproduces_the_reference(tag):
    from sonet_b200 import losses, ops
    score, seg, label = case(tag)
    iou, pred, correct = ops.seg_iou(score, seg, label, want_pred=True, want_correct=True)
    assert iou.dtype == torch.float64 and iou.is_cuda
    assert np.array_equal(iou.cpu().numpy(), G[tag + "_iou"])
    assert losses.compute_iou(score, seg, label, None, None, None) == G[tag + "_miou"]
    ref_pred = torch.max(score.cpu(), dim=1)[1]
    assert torch.equal(pred.cpu(), ref_pred)
    assert torch.equal(correct.cpu(), (ref_pred == seg.cpu()).sum(1).int())


@pytest.mark.parametrize("N", [1000, 2048, 5000])
@pytest.mark.parametrize("ties", [False, True])
def test_kernel_equals_host_entry(N, ties):
    from sonet_b200 import losses, ops
    score, seg, label = random_batch(64, 50, N, seed=N, ties=ties)
    host = losses.compute_iou_np_array(score, seg, label, None, None, None)
    iou, pred, correct = ops.seg_iou(score.to(DEV), seg.to(DEV), label.to(DEV), want_pred=True,
                                     want_correct=True)
    assert np.array_equal(iou.cpu().numpy(), host)
    ref_pred = torch.max(score, dim=1)[1]                  # CPU rules: first max, first NaN wins
    assert torch.equal(pred.cpu(), ref_pred)
    assert torch.equal(correct.cpu(), (ref_pred == seg).sum(1).int())


def test_labels_outside_the_table():
    from sonet_b200 import losses, ops
    score, seg, label = case("random")
    label = label.clone()
    label[5] = 16
    label[9] = -1
    iou, _, correct = ops.seg_iou(score, seg, label, want_correct=True)
    iou = iou.cpu().numpy()
    assert np.isnan(iou[[5, 9]]).all()
    keep = np.ones(len(iou), bool)
    keep[[5, 9]] = False
    assert np.array_equal(iou[keep], G["random_iou"][keep])
    ref_pred = torch.max(score.cpu(), dim=1)[1]
    assert torch.equal(correct.cpu(), (ref_pred == seg.cpu()).sum(1).int())
    with pytest.raises(RuntimeError, match="outside the part table"):
        losses.compute_iou(score, seg, label, None, None, None)
    meter = losses.PartSegIoU()
    meter.update(score, seg, label)
    with pytest.raises(RuntimeError, match="outside the part table"):
        meter.compute()


def test_cuda_graph_replay_gives_the_same_bits():
    from sonet_b200 import ops
    score, seg, label = (t.to(DEV) for t in random_batch(32, 50, 2048, seed=5))
    ref = ops.seg_iou(score, seg, label, want_pred=True, want_correct=True)   # uploads the table
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.seg_iou(score, seg, label, want_pred=True, want_correct=True)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.seg_iou(score, seg, label, want_pred=True, want_correct=True)
    for t in out:
        t.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, ref):
        assert torch.equal(a, b)
    new = random_batch(32, 50, 2048, seed=6)                # replay on new inputs in place
    for dst, src in zip((score, seg, label), new):
        dst.copy_(src)
    graph.replay()
    want = ops.seg_iou(score, seg, label, want_pred=True, want_correct=True)
    torch.cuda.synchronize()
    for a, b in zip(out, want):
        assert torch.equal(a, b)


def test_partsegiou_matches_numpy_and_is_deterministic():
    from sonet_b200 import losses
    batches = [random_batch(32, 50, 1024, seed=s) for s in range(4)]

    def run():
        meter = losses.PartSegIoU()
        for score, seg, label in batches:
            d = [t.to(DEV) for t in (score, seg, label)]
            meter.update(*d)
            d[2].fill_(0)          # the caller may reuse its label buffer (set_input copies into it)
        return meter.compute()

    r = run()
    iou = np.concatenate([losses.compute_iou_np_array(*b, None, None, None) for b in batches])
    lab = np.concatenate([b[2].numpy() for b in batches])
    correct = sum(int((torch.max(b[0], 1)[1] == b[1]).sum()) for b in batches)
    assert r["instance_miou"] == iou.mean()
    cats = sorted(set(lab.tolist()))
    assert list(r["category_miou"]) == cats
    for c in cats:
        assert r["category_miou"][c] == iou[lab == c].mean()
    assert r["class_miou"] == np.asarray([iou[lab == c].mean() for c in cats]).mean()
    assert r["accuracy"] == correct / (4 * 32 * 1024)
    again = run()
    assert again["instance_miou"] == r["instance_miou"] and again["class_miou"] == r["class_miou"]
    assert again["category_miou"] == r["category_miou"] and again["accuracy"] == r["accuracy"]


def test_part_seg_train_metric_under_install():
    """part-seg/train.py:95's losses.compute_iou(score.cpu(), seg.cpu(), label.cpu(), ...) after the
    reference segmenter Model's test_model() on CUDA, against the reference's own compute_iou."""
    sys.path.insert(0, ROOT)
    from oracle import build as obuild
    root = obuild.pyref_root()
    if root is None:
        pytest.fail("oracle/_ref/pyref missing: run __graft_entry__.build() where the reference "
                    "tree is available")
    script = os.path.join(ROOT, "tests", "_dropin_seg_iou_run.py")
    r = subprocess.run([sys.executable, script, root, DEV], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and "SEG_IOU_DROPIN_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
