"""Time optimize() under data-parallel training (sonet_b200.dist.DataParallelTraining).

    python -m torch.distributed.run --nproc-per-node G tools/dp_train_bench.py [--steps 10]
    python tools/dp_train_bench.py                       # one process

For the classifier (B = 32, N = 5000), the segmenter (B = 32, N = 1024) and the auto-encoder
(B = 32, N = 5000), B being the global batch split over the ranks, it reports ms per step and
clouds/s of the global batch:
  plain  the single-GPU train kernels (one process only);
  dp     DataParallelTraining: the per-cloud BatchNorm route, the BatchNorm exchanges and the
         gradient reduction (the identity without a process group);
and the time inside the BatchNorm gathers and the gradient gathers, from CUDA events around each.
Rank 0 prints one line per case; --json adds a JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "so-net_b200")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sonet_b200 import autoencoder, classifier, dist as sdist, segmenter, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--tasks", default="classifier,segmenter,autoencoder")
ap.add_argument("--json", action="store_true")
ap.add_argument("--backend", default=None, help="nccl (default with CUDA) or gloo: two ranks on "
                "one GPU need gloo, and then time the exchange, not the scaling")
a = ap.parse_args()

NPTS = {"classifier": 5000, "segmenter": 1024, "autoencoder": 5000}
MODS = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}
rank, local_rank, world = sdist.init_from_env(a.backend)
dev = torch.device("cuda", torch.cuda.current_device())


def run(task, mode):
    Bg, N = a.batch, NPTS[task]
    opt = synth.make_opt(task, batch_size=Bg, input_pc_num=N, device=dev)
    m = MODS[task].Model(opt)
    dp = sdist.DataParallelTraining(m, Bg) if mode == "dp" else None
    lo, hi = dp.shard() if dp else (0, Bg)
    inp = synth.synth_inputs(Bg, N, seed=0)
    args = [inp["pc"], inp["sn"], inp["label"]]
    if task == "segmenter":
        args.append(torch.from_numpy(np.random.RandomState(0).randint(0, 50, size=(Bg, N))))
    args += [inp["node"], inp["node_knn_I"]]
    m.set_input(*[t[lo:hi] for t in args])
    for _ in range(a.warmup):
        m.optimize()
    torch.cuda.synchronize()
    if dp:
        dp.start_timing()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        m.optimize()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    ex = dp.exchange_ms() if dp else {}
    if dp:
        dp.close()
    res = dict(task=task, mode=mode, world=world, global_batch=Bg, npts=N, ms_per_step=ms,
               clouds_per_s=Bg / ms * 1e3)
    for kind in ("bn", "grad"):
        n, t = ex.get(kind, (0, 0.0))
        res[kind + "_gathers_per_step"] = n / a.steps
        res[kind + "_gather_ms_per_step"] = t / a.steps
    return res


for task in a.tasks.split(","):
    for mode in (("plain", "dp") if world == 1 else ("dp",)):
        r = run(task, mode)
        if rank == 0:
            print("%-11s %-5s world %d  B %d  N %5d  %8.2f ms/step  %7.1f clouds/s  BN gathers %4.1f "
                  "(%.2f ms)  grad gathers %3.1f (%.2f ms)"
                  % (task, mode, world, r["global_batch"], r["npts"], r["ms_per_step"],
                     r["clouds_per_s"], r["bn_gathers_per_step"], r["bn_gather_ms_per_step"],
                     r["grad_gathers_per_step"], r["grad_gather_ms_per_step"]))
            if a.json:
                print(json.dumps(r))
        sys.stdout.flush()
if world > 1:
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()
