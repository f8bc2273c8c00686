"""Helper of tests/test_gpu_dp_train.py, run as one rank under torch.distributed.run or alone:

    python tests/_dp_train_run.py <out_dir> <backend>

Trains the classifier (global batch 5: a ragged shard over two ranks), the segmenter and the
auto-encoder (global batch 4) for 3 optimize() steps under DataParallelTraining, each rank on its
shard of the same global batches, and saves every parameter, gradient, buffer and the shard losses
to <out_dir>/<task>_w<world>_r<rank>.pt. Without torch.distributed.run (WORLD_SIZE unset) it is the
one-process run over the global batch that a run over several ranks is compared with."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from helpers import build_states  # noqa: E402
from sonet_b200 import autoencoder, classifier, dist as sdist, segmenter, synth  # noqa: E402

CASES = (("classifier", 5, 512), ("segmenter", 4, 512), ("autoencoder", 4, 512))
STEPS = 3


def run(task, Bg, N, out_dir, rank, world, dev):
    opt = synth.make_opt(task, batch_size=Bg, input_pc_num=N, device=dev)
    opt.dropout = 0.1                     # at most 0.1: the layers leave nn.Dropout out
    mod = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}[task]
    head = {"classifier": "classifier", "segmenter": "segmenter", "autoencoder": "decoder"}[task]
    st = build_states(task, opt, seed=31)
    m = mod.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    getattr(m, head).load_state_dict(st["head"])
    dp = sdist.DataParallelTraining(m, Bg)
    lo, hi = dp.shard()
    losses = []
    for step in range(STEPS):
        inp = synth.synth_inputs(Bg, N, seed=40 + step)
        args = [inp["pc"], inp["sn"], inp["label"]]
        if task == "segmenter":
            args.append(torch.from_numpy(np.random.RandomState(step).randint(0, 50, size=(Bg, N))))
        args += [inp["node"], inp["node_knn_I"]]
        m.set_input(*[a[lo:hi] for a in args])
        m.optimize(epoch=None)
        loss = m.loss_segmenter if task == "segmenter" else m.loss
        losses.append(float(loss.detach()))
    dp.close()
    mods = {"encoder": m.encoder, head: getattr(m, head)}
    res = {"losses": losses, "rows": hi - lo}
    for name, mm in mods.items():
        for k, v in mm.state_dict().items():
            res["state.%s.%s" % (name, k)] = v.detach().cpu().clone()
        for k, p in mm.named_parameters():
            if p.grad is not None:
                res["grad.%s.%s" % (name, k)] = p.grad.detach().cpu().clone()
    torch.save(res, os.path.join(out_dir, "%s_w%d_r%d.pt" % (task, world, rank)))


def main():
    out_dir, backend = sys.argv[1], sys.argv[2]
    rank, local_rank, world = sdist.init_from_env(backend=backend)
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.backends.cudnn.deterministic = True
    for task, Bg, N in CASES:
        run(task, Bg, N, out_dir, rank, world, dev)
    if world > 1:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()
    print("DP_TRAIN_OK rank %d of %d" % (rank, world))


if __name__ == "__main__":
    main()
