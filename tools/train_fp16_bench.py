"""Time optimize() with the default train kernels, under SONET_TRAIN_TC=fp16, and as the PyTorch
composition with cuDNN's TF32 on (train_ops.ENABLED = False: the reference's default arithmetic).

    python tools/train_fp16_bench.py [--steps 10] [--warmup 3] [--rounds 3] [--json]

Cases: the classifier at B = 32 and at the training scripts' default B = 8 (N = 5000), the segmenter
(B = 32, N = 1024) and the auto-encoder (B = 32, N = 5000), on synth inputs. Each round runs the three
arms one after the other (alternated, so drift in clocks or in other work on the machine spreads over
all three); ms/step is CUDA events around `--steps` steps after `--warmup`. A separate profiled step
per kernel arm gives the share of the step spent in the train GEMM entries (CUDA events around each
library call, ops.PROFILE), which slows the host, so it is not part of the timed steps."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "so-net_b200")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sonet_b200 import autoencoder, classifier, ops, segmenter, synth, train_ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--cases", default="classifier:32:5000,classifier:8:5000,segmenter:32:1024,"
                "autoencoder:32:5000")
ap.add_argument("--json", action="store_true")
a = ap.parse_args()

MODS = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}
GEMMS = ("sonet_pointwise_tc_forward_dev", "sonet_pointwise_tc_grouped_forward_dev",
         "sonet_wgrad_tc")
ARMS = ("default", "fp16", "torch_tf32")
dev = torch.device("cuda", torch.cuda.current_device())


def arm(name):
    """Set the environment and flags of an arm."""
    if name == "fp16":
        os.environ["SONET_TRAIN_TC"] = "fp16"
    else:
        os.environ.pop("SONET_TRAIN_TC", None)
    train_ops.ENABLED = name != "torch_tf32"
    torch.backends.cudnn.allow_tf32 = True          # PyTorch's default; the kernels ignore it
    torch.backends.cuda.matmul.allow_tf32 = False


def make(task, B, N):
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, device=dev)
    m = MODS[task].Model(opt)
    inp = synth.synth_inputs(B, N, seed=0)
    args = [inp["pc"], inp["sn"], inp["label"]]
    if task == "segmenter":
        args.append(torch.from_numpy(np.random.RandomState(0).randint(0, 50, size=(B, N))))
    m.set_input(*args, inp["node"], inp["node_knn_I"])
    return m


def timed(m):
    for _ in range(a.warmup):
        m.optimize()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        m.optimize()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.steps


def gemm_share(m):
    """(ms in the train GEMM entries, ms of the whole step) of one profiled step."""
    calls = []
    ops.PROFILE = calls
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    try:
        e0.record()
        m.optimize()
        e1.record()
        torch.cuda.synchronize()
    finally:
        ops.PROFILE = None
    g = sum(s.elapsed_time(e) for n, s, e, _ in calls if n.replace("_f16", "").startswith(GEMMS))
    return g, e0.elapsed_time(e1)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


print("# %s; torch %s" % (gpu_info(), torch.__version__), flush=True)
results = []
for case in a.cases.split(","):
    task, B, N = case.split(":")
    B, N = int(B), int(N)
    models = {}
    for name in ARMS:
        arm(name)
        models[name] = make(task, B, N)
    runs = {name: [] for name in ARMS}
    for _ in range(a.rounds):
        for name in ARMS:
            arm(name)
            runs[name].append(timed(models[name]))
    share = {}
    for name in ("default", "fp16"):
        arm(name)
        share[name] = gemm_share(models[name])
    arm("default")
    res = dict(task=task, batch=B, npts=N, steps=a.steps, rounds=a.rounds,
               ms_per_step={k: v for k, v in runs.items()},
               gemm_ms={k: v[0] for k, v in share.items()},
               profiled_step_ms={k: v[1] for k, v in share.items()})
    results.append(res)
    med = {k: float(np.median(v)) for k, v in runs.items()}
    print("%-11s B=%-2d N=%-4d ms/step median of %d: default %.2f  fp16 %.2f  torch+tf32 %.2f "
          "(runs %s) | train GEMMs in a profiled step: default %.2f of %.2f ms, fp16 %.2f of %.2f ms"
          % (task, B, N, a.rounds, med["default"], med["fp16"], med["torch_tf32"],
             "; ".join("%s %s" % (k, ",".join("%.2f" % x for x in v)) for k, v in runs.items()),
             share["default"][0], share["default"][1], share["fp16"][0], share["fp16"][1]),
          flush=True)
    del models
    torch.cuda.empty_cache()
if a.json:
    print(json.dumps(dict(gpu=gpu_info(), results=results)))
