"""Time the part-segmentation metric three ways at part-seg's batch shapes (C = 50 parts):

  reference   the reference's compute_iou (models/losses.py:119-189, from the bytecode tree
              oracle/_ref/pyref) called as part-seg/train.py:95 does: score, seg and label copied
              from the device with .cpu(), copies included
  host        sonet_b200.losses.compute_iou on the same host tensors (C++ host entry), with torch's
              thread count and with 1 and 4 threads
  device      ops.seg_iou on the device tensors, CUDA events: `call` = eager calls back to back,
              `kernel` = the same call replayed from a CUDA graph; plus `compute_iou` =
              losses.compute_iou on the device tensors, host clock, including the copy of the [B]
              result and the mean

    python tools/seg_iou_bench.py [--out results.jsonl]

Prints one JSON line per (B, N) with medians in ms, and the GPU's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle.seg_iou_golden import load_ref_losses  # noqa: E402
from sonet_b200 import losses, ops  # noqa: E402

SHAPES = ((32, 1024), (32, 2048))


def host_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def event_ms(fn, inner, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(inner):
            fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) / inner)
    return float(np.median(ts))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seg_iou_bench needs a CUDA device")
    ref = load_ref_losses()
    dev = torch.device("cuda:0")
    rows = []
    for B, N in SHAPES:
        g = torch.Generator(device=dev).manual_seed(B * N)
        score = torch.randn(B, 50, N, device=dev, generator=g)
        label = torch.randint(0, 16, (B,), device=dev, generator=g)
        table = torch.tensor([p for parts in ops.SHAPENET_PART_TABLE for p in parts], device=dev)
        offs = torch.tensor([0] + list(np.cumsum([len(p) for p in ops.SHAPENET_PART_TABLE])),
                            device=dev)
        pick = torch.randint(0, 1 << 20, (B, N), device=dev, generator=g)
        cnt = (offs[1:] - offs[:-1])[label][:, None]
        seg = table[offs[:-1][label][:, None] + pick % cnt]               # a part of the category
        score.scatter_add_(1, seg[:, None, :], torch.full((B, 1, N), 2.0, device=dev))
        h = (score.cpu(), seg.cpu(), label.cpu())
        want = ref.compute_iou(*h, None, None, None)
        assert losses.compute_iou(*h, None, None, None) == want
        assert losses.compute_iou(score, seg, label, None, None, None) == want
        r = dict(B=B, N=N, C=50, gpu=gpu_info(), cpu_threads=torch.get_num_threads())
        r["reference_ms"] = host_ms(lambda: ref.compute_iou(score.cpu().data, seg.cpu().data,
                                                            label.cpu().data, None, None, None),
                                    max(5, a.reps // 3))
        r["copy_to_host_ms"] = host_ms(lambda: (score.cpu(), seg.cpu(), label.cpu()), a.reps)
        r["host_ms"] = host_ms(lambda: losses.compute_iou(*h, None, None, None), a.reps)
        default_threads = torch.get_num_threads()
        r["host_ms_by_threads"] = {}
        for t in (1, 4):                    # the host entry splits shapes over torch's thread count
            torch.set_num_threads(t)
            r["host_ms_by_threads"][t] = host_ms(lambda: losses.compute_iou(*h, None, None, None),
                                                 a.reps)
        torch.set_num_threads(default_threads)
        call = lambda: ops.seg_iou(score, seg, label)                   # noqa: E731
        r["device_call_ms"] = event_ms(call, 100, a.reps)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            call()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(100):
                call()
        r["device_kernel_ms"] = event_ms(graph.replay, 1, a.reps) / 100
        r["device_compute_iou_ms"] = host_ms(
            lambda: losses.compute_iou(score, seg, label, None, None, None), a.reps)
        rows.append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
