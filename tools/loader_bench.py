"""loader_bench.py — time augmentation.DeviceDataset.batch() (the loader's point choice, augmentation
and SOM-node kNN on the device) at two shapes, in both modes of drawing:

  cfg2   B=64 clouds of P=10,000 points -> N=5,000, M=64 SOM nodes, som_k=9, train (ModelNet rule,
         both rotations and the shift on)
  cfg3   B=32 clouds of P in [2,000, 3,000] -> N=1,024 with part labels, M=64, som_k=9, train
         (ShapeNet rule)

    python tools/loader_bench.py [--iters 200] [--warmup 10] [--out FILE]

For each mode (in-kernel draws, host numpy draws) it prints one JSON line: us per batch from CUDA
events around `iters` back-to-back batch() calls, clouds/s, the device-memory bytes the batch moves
(from shapes: source rows and labels read, the sample written, the augmentation's read and write,
host noise uploaded) and their share of 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth), plus the
sample_points kernel alone. A numpy restatement of the loader's per-item work (choice, gather,
rotations, jitter, scale, shift; no kNN) is timed on one host core and reported with the core count.
The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

HBM_BPS = 3.35e12
SHAPES = {
    "cfg2": dict(B=64, S=128, P=(10000, 10000), N=5000, M=64, dataset="modelnet", seg=False),
    "cfg3": dict(B=32, S=256, P=(2000, 3000), N=1024, M=64, dataset="shapenet", seg=True),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still printed, without the card's settings
        return "unknown (%s)" % e


def make_dataset(cfg, seed=0):
    from sonet_b200 import augmentation as A
    rs = np.random.RandomState(seed)
    counts = rs.randint(cfg["P"][0], cfg["P"][1] + 1, size=cfg["S"])
    pts = [rs.uniform(-1, 1, size=(P, 6)).astype(np.float32) for P in counts]
    som = [rs.uniform(-1, 1, size=(cfg["M"], 3)).astype(np.float32) for _ in counts]
    seg = [rs.randint(0, 50, size=P) for P in counts] if cfg["seg"] else None
    ds = A.DeviceDataset(pts, rs.randint(0, 16, size=cfg["S"]), som, seg=seg, device="cuda:0")
    return ds, pts


def batch_bytes(cfg, host_noise):
    B, N, M = cfg["B"], cfg["N"], cfg["M"]
    lab = 4 + 8 if cfg["seg"] else 0
    sample = B * N * (24 + 24 + lab)           # source rows (+ labels) read, pc/sn (+ seg) written
    augment = B * (N * 48 + M * 24)            # pc, sn, som read and written
    noise = B * (2 * N + M) * 24 if host_noise else 0
    return sample + augment + noise


def numpy_item(pts, N, M, rng, rule_fill):
    """The loader's per-item work for one cloud (modelnet_shrec_loader.py:198,218-256)."""
    data = pts[rng.randint(len(pts))]
    P = len(data)
    if rule_fill and N >= P:
        idx = np.concatenate([np.arange(P), rng.choice(P, N - P, replace=True)])
    else:
        idx = rng.choice(P, N, replace=False)
    d = data[idx]
    pc, sn = d[:, :3], d[:, 3:]
    som = rng.uniform(-1, 1, size=(M, 3)).astype(np.float32)
    if not rule_fill:
        a = rng.uniform() * 2 * np.pi
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        pc, sn, som = np.dot(pc, R), np.dot(sn, R), np.dot(som, R)
    pc = np.clip(0.01 * rng.randn(N, 3), -0.05, 0.05) + pc
    sn = np.clip(0.01 * rng.randn(N, 3), -0.05, 0.05) + sn
    som = np.clip(0.04 * rng.randn(M, 3), -0.1, 0.1) + som
    s = rng.uniform(0.8, 1.2)
    return (pc * s).T.astype(np.float32), (sn * s).T.astype(np.float32), (som * s).T.astype(np.float32)


def run(name, cfg, iters, warmup):
    from sonet_b200 import ops
    ds, pts = make_dataset(cfg)
    opt = types.SimpleNamespace(dataset=cfg["dataset"], input_pc_num=cfg["N"], node_num=cfg["M"],
                                som_k=9, rot_horizontal=True, rot_perturbation=True,
                                translation_perturbation=True)
    B = cfg["B"]
    order = np.random.RandomState(1).randint(0, cfg["S"], size=(iters + warmup, B))
    rows = []
    for mode, host_noise in (("in_kernel", False), ("host_draws", True)):
        rng = np.random.RandomState(2)
        for i in range(warmup):
            ds.batch(order[i], opt, train=True, rng=rng, seed=i, host_noise=host_noise)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            ds.batch(order[warmup + i], opt, train=True, rng=rng, seed=i, host_noise=host_noise)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / iters
        nbytes = batch_bytes(cfg, host_noise)
        rows.append(dict(shape=name, mode=mode, B=B, N=cfg["N"], P=list(cfg["P"]),
                         us_per_batch=round(us, 1), clouds_per_s=round(B / us * 1e6),
                         bytes_per_batch=nbytes, hbm_share=round(nbytes / (us * 1e-6) / HBM_BPS, 4)))
    # the sample_points kernel alone, in-kernel draws
    cid = torch.from_numpy(order[0]).to("cuda:0")
    rule = ops.SAMPLE_FILL if cfg["dataset"] == "shapenet" else ops.SAMPLE_SUBSET
    maxp = int(ds.counts.max())
    for i in range(warmup):
        ops.sample_points(ds.data, ds.offsets, cid, cfg["N"], rule, maxp, labels=ds.seg if
                          cfg["seg"] else None, seed=i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        ops.sample_points(ds.data, ds.offsets, cid, cfg["N"], rule, maxp, labels=ds.seg if
                          cfg["seg"] else None, seed=i)
    e1.record()
    torch.cuda.synchronize()
    us_k = e0.elapsed_time(e1) * 1e3 / iters
    kbytes = B * cfg["N"] * (48 + (12 if cfg["seg"] else 0))
    rows.append(dict(shape=name, mode="sample_points_kernel", us_per_batch=round(us_k, 1),
                     bytes_per_batch=kbytes, hbm_share=round(kbytes / (us_k * 1e-6) / HBM_BPS, 4)))
    # the loader's per-item numpy work on one host core
    rng = np.random.RandomState(3)
    n_items = max(2 * B, 64)
    t0 = time.perf_counter()
    for _ in range(n_items):
        numpy_item(pts, cfg["N"], cfg["M"], rng, cfg["dataset"] == "shapenet")
    per_item = (time.perf_counter() - t0) / n_items
    cores = os.cpu_count()
    rows.append(dict(shape=name, mode="numpy_per_item_one_core", us_per_item=round(per_item * 1e6, 1),
                     clouds_per_s_one_core=round(1 / per_item), host_cores=cores,
                     clouds_per_s_all_cores_ideal=round(cores / per_item)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loader_bench.py needs a CUDA device")
    info = dict(card=card(), torch=torch.__version__)
    print(json.dumps(info))
    rows = []
    for name, cfg in SHAPES.items():
        for r in run(name, cfg, a.iters, a.warmup):
            print(json.dumps(r))
            rows.append(r)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
