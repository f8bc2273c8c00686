"""Cost of full-resolution part segmentation on ShapeNet-like shapes: B = 32 clouds of P_i points
drawn from 2,000-3,000, the segmenter at N = 1024 sampled points, synthetic weights.

  test_model        ms per batch of Model.test_model() alone
  full              ms per batch of test_model() + score_points() over all points + compute_iou_full
  score_points      ms of score_points() alone, and its split (a second, profiled pass through
                    ops.PROFILE, which adds an event pair per library call): assignment
                    (sonet_seg_points_assign_f32), first PointResNet (its kernels), head (the rest:
                    the node/cloud addend, layers 1-5, the k-copy mean)

CUDA events, medians over --reps batches after --warmup. Prints one JSON line with the GPU's name
and power limit read in the same run.

    python tools/seg_full_bench.py [--reps 20] [--warmup 3] [--out results/seg_full.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sonet_b200 import losses, networks, ops, segmenter, synth  # noqa: E402

B, N, M = 32, 1024, 64
FIRST_PRN = ("sonet_pointresnet_tc_forward", "sonet_pointresnet_tc_forward_f16",
             "sonet_pointresnet_tc_forward_act")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception as e:  # the name from torch still identifies the card
        name, power = torch.cuda.get_device_name(0), "unknown (%s)" % e
    return name, power


def make_case(seed=0):
    rs = np.random.RandomState(seed)
    sizes = rs.randint(2000, 3001, size=B)
    clouds = []
    for P in sizes:
        xyz = rs.uniform(-1, 1, size=(P, 3)).astype(np.float32)
        n = rs.normal(size=(P, 3))
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        clouds.append(np.concatenate([xyz, n.astype(np.float32)], axis=1))
    pc, sn, node = [], [], []
    for c in clouds:
        sel = rs.choice(len(c), N, replace=False)
        pc.append(c[sel, :3].T)
        sn.append(c[sel, 3:].T)
        node.append(c[rs.choice(len(c), M, replace=False), :3].T)
    node = np.ascontiguousarray(np.stack(node), dtype=np.float32)
    d = ((node[:, :, :, None].astype(np.float64) - node[:, :, None, :]) ** 2).sum(axis=1)
    knn = np.argsort(d, axis=2, kind="stable")[:, :, :9].astype(np.int64)
    label = rs.randint(0, 16, size=B).astype(np.int64)
    batch = [torch.from_numpy(np.ascontiguousarray(a)) for a in
             (np.stack(pc), np.stack(sn), label, np.zeros((B, N), np.int64), node, knn)]
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    seg = np.concatenate([rs.choice(ops.SHAPENET_PART_TABLE[l], size=P) for l, P in zip(label, sizes)])
    return batch, np.concatenate(clouds), offsets, seg, sizes


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seg_full_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    opt = synth.make_opt("segmenter", batch_size=B, input_pc_num=N)
    enc_st = synth.synth_state_dict(networks.Encoder(opt), seed=1)
    head_st = synth.synth_state_dict(networks.Segmenter(opt), seed=2)
    opt.device = dev
    m = segmenter.Model(opt)
    m.encoder.load_state_dict(enc_st)
    m.segmenter.load_state_dict(head_st)
    batch, pts, offs, seg, sizes = make_case()
    batch = [t.to(dev) for t in batch]
    pts, off = torch.from_numpy(pts).to(dev), torch.from_numpy(offs).to(dev)
    seg, label = torch.from_numpy(seg).to(dev), batch[2]
    m.set_input(*batch)

    def eval_only():
        m.test_model()

    def full():
        m.test_model()
        losses.compute_iou_full(m.score_points(pts, off), seg, label, off)

    def score_only():
        m.score_points(pts, off)

    name, power = gpu_info()
    r = dict(gpu=name, power_limit=power, B=B, N=N, M=M, k=opt.k, points=int(offs[-1]),
             P_min=int(sizes.min()), P_max=int(sizes.max()), sonet_tc=os.environ.get("SONET_TC", "1"))
    r["test_model_ms"] = timed(eval_only, a.reps, a.warmup)
    r["full_ms"] = timed(full, a.reps, a.warmup)
    m.test_model()
    r["score_points_ms"] = timed(score_only, a.reps, a.warmup)

    split = {"assignment": [], "first_pointresnet": [], "head": []}
    for _ in range(a.reps):
        ops.PROFILE = []
        score_only()
        torch.cuda.synchronize()
        acc = dict.fromkeys(split, 0.0)
        for call, e0, e1, _args in ops.PROFILE:
            part = ("assignment" if call == "sonet_seg_points_assign_f32" else
                    "first_pointresnet" if call in FIRST_PRN else "head")
            acc[part] += e0.elapsed_time(e1)
        for kk in split:
            split[kk].append(acc[kk])
    ops.PROFILE = None
    r["score_points_split_ms"] = {kk: float(np.median(v)) for kk, v in split.items()}
    line = json.dumps(r)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
