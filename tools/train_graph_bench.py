"""Time optimize() eagerly and replayed as one CUDA graph (Model.enable_train_graph).

    python tools/train_graph_bench.py [--steps 20] [--warmup 3] [--rounds 3] [--json]

Cases: the classifier and the auto-encoder at N = 5000, the segmenter at N = 1024, each at the
training scripts' default B = 8 and at B = 32, on synth inputs. Each round times both arms one
after the other (alternated, so drift in clocks or in other work on the machine spreads over both);
ms/step is CUDA events around `--steps` steps after `--warmup` (the graph arm's first two calls, the
eager step of a new key and the capture, are part of its first warm-up). Also reported: the C-ABI
calls and kernels per step (ops.LAUNCHES, ops.KERNEL_LAUNCHES: the same in both arms, the graph
replays them), the host time of one optimize() call (median of five calls, each from an idle
device), the cost of a new key (the wall time of the eager step and of the capture call, each from
an idle device to the end of its work), and the memory the graph's private pool holds (the segments
of its pool in torch.cuda.memory_snapshot())."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "so-net_b200")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from sonet_b200 import autoencoder, classifier, ops, segmenter, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--cases", default="classifier:8:5000,classifier:32:5000,segmenter:8:1024,"
                "segmenter:32:1024,autoencoder:8:5000,autoencoder:32:5000")
ap.add_argument("--json", action="store_true")
a = ap.parse_args()

MODS = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}
ARMS = ("eager", "graph")
dev = torch.device("cuda", torch.cuda.current_device())


def make(task, B, N, graph):
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, device=dev)
    m = MODS[task].Model(opt)
    inp = synth.synth_inputs(B, N, seed=0)
    args = [inp["pc"], inp["sn"], inp["label"]]
    if task == "segmenter":
        args.append(torch.from_numpy(np.random.RandomState(0).randint(0, 50, size=(B, N))))
    m.set_input(*args, inp["node"], inp["node_knn_I"])
    m.enable_train_graph(graph)
    return m


def warm(m, graph):
    """Warm-up steps -> (wall ms of each warm-up call, bytes of the graph's private pool)."""
    wall = []
    for _ in range(a.warmup):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.optimize()
        torch.cuda.synchronize()
        wall.append((time.perf_counter() - t0) * 1e3)
    if not graph:
        return wall, 0
    pid = tuple(m._train_graphs[m._cur]["graph"].pool())
    return wall, sum(s["total_size"] for s in torch.cuda.memory_snapshot()
                     if tuple(s.get("segment_pool_id", ())) == pid)


def timed(m):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        m.optimize()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.steps


def counts(m):
    """(C-ABI calls, kernels) of one optimize() call, and the median host ms of five calls."""
    host = []
    for _ in range(5):
        torch.cuda.synchronize()
        k0, c0 = ops.KERNEL_LAUNCHES, ops.LAUNCHES
        t0 = time.perf_counter()
        m.optimize()
        host.append((time.perf_counter() - t0) * 1e3)
        n = (ops.LAUNCHES - c0, ops.KERNEL_LAUNCHES - k0)
    torch.cuda.synchronize()
    return n[0], n[1], float(np.median(host))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


if a.warmup < 3:
    sys.exit("--warmup must be at least 3: the graph arm's first two calls warm and capture")
print("# %s; torch %s" % (gpu_info(), torch.__version__), flush=True)
results = []
for case in a.cases.split(","):
    task, B, N = case.split(":")
    B, N = int(B), int(N)
    models = {name: make(task, B, N, name == "graph") for name in ARMS}
    warmed = {name: warm(models[name], name == "graph") for name in ARMS}
    (wall, pool), steady = warmed["graph"], warmed["eager"][0][-1]
    runs = {name: [] for name in ARMS}
    for _ in range(a.rounds):
        for name in ARMS:
            runs[name].append(timed(models[name]))
    cnt = {name: counts(models[name]) for name in ARMS}
    med = {k: float(np.median(v)) for k, v in runs.items()}
    res = dict(task=task, batch=B, npts=N, steps=a.steps, rounds=a.rounds, ms_per_step=runs,
               median_ms=med, calls_per_step=cnt["eager"][0], kernels_per_step=cnt["eager"][1],
               graph_calls_per_step=cnt["graph"][0], graph_kernels_per_step=cnt["graph"][1],
               host_ms_per_call={k: v[2] for k, v in cnt.items()}, graph_pool_mb=pool / 2 ** 20,
               new_key_ms=dict(eager_step=wall[0], capture=wall[1], steady_eager_step=steady),
               peak_allocated_mb=torch.cuda.max_memory_allocated(dev) / 2 ** 20)
    results.append(res)
    print("%-11s B=%-2d N=%-4d ms/step median of %d: eager %.2f  graph %.2f (%.1f%%) | runs %s | "
          "%d C-ABI calls, %d kernels per step | host ms per call: eager %.2f graph %.2f | "
          "graph pool %.0f MB | new key: eager step %.1f ms + capture call %.1f ms (a warm eager "
          "step from an idle device: %.1f ms)"
          % (task, B, N, a.rounds, med["eager"], med["graph"],
             100.0 * (med["eager"] - med["graph"]) / med["eager"],
             "; ".join("%s %s" % (k, ",".join("%.2f" % x for x in v)) for k, v in runs.items()),
             cnt["eager"][0], cnt["eager"][1], cnt["eager"][2], cnt["graph"][2], pool / 2 ** 20,
             wall[0], wall[1], steady),
          flush=True)
    del models
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
if a.json:
    print(json.dumps(dict(gpu=gpu_info(), results=results)))
