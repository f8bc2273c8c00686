"""Time the batch-statistics BatchNorm at the training shapes, CUDA events around back-to-back
calls: the forward (sonet_bn_cloud_partials_f32's per-cloud records, then sonet_bn_sync_forward_f32's
fold and normalise + ReLU) and the backward (the backward records, then sonet_bn_sync_backward_f32).

    python tools/bn_train_bench.py [--baseline-lib other/libsonet_b200.so] [--out results.jsonl]

With --baseline-lib the same call of another build of the library is timed in the same process,
alternating with this tree's in every repetition, so that both see the same clocks and neighbours;
both builds' statistics are compared too. Prints one JSON line per shape and direction with medians
in ms and the GPU's name and power limit.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sonet_b200 import _C  # noqa: E402

# (B, C, P): the first PointResNet's BN layers at N = 5000 (3 copies of the cloud per point) and
# the KNN module's (64 nodes x 9 neighbours)
SHAPES = ((64, 64, 15000), (64, 512, 576))
ENTRIES = ("sonet_bn_cloud_partials_f32", "sonet_bn_sync_forward_f32", "sonet_bn_sync_backward_f32")


def load(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    for name in ENTRIES:
        fn = getattr(lib, name)
        fn.argtypes = _C._SIGNATURES[name]
        fn.restype = ctypes.c_int
    return lib


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--inner", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bn_train_bench needs a CUDA device")
    libs = {"this": load(_C.LIB_PATH)}
    if a.baseline_lib:
        libs["baseline"] = load(a.baseline_lib)
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    rows = []
    for B, C, P in SHAPES:
        g = torch.Generator(device=dev).manual_seed(B + C + P)
        x = torch.randn(B, C, P, device=dev, generator=g) * 2 + torch.randn(C, 1, device=dev, generator=g)
        dy = torch.randn(B, C, P, device=dev, generator=g)
        gamma = torch.rand(C, device=dev, generator=g) + 0.5
        beta = torch.randn(C, device=dev, generator=g) * 0.2
        out = {}
        for k, lib in libs.items():
            rec = torch.empty(B * C * _C.CONSTANTS["SONET_BN_REC_FWD"], dtype=torch.float64, device=dev)
            y, dx = torch.empty_like(x), torch.empty_like(x)
            st = [torch.empty(C, device=dev) for _ in range(5)]      # mean, var, invstd, dgamma, dbeta
            p = lambda t: t.data_ptr()

            def fwd(lib=lib, rec=rec, y=y, st=st):
                _C.check(lib.sonet_bn_cloud_partials_f32(p(x), None, None, None, None, None, B, C, P, 1,
                                                         0, p(rec), stream), ENTRIES[0])
                _C.check(lib.sonet_bn_sync_forward_f32(p(rec), p(x), p(gamma), p(beta), B, B, C, P, 1e-5,
                                                       1, p(y), *[p(t) for t in st[:3]], stream),
                         ENTRIES[1])

            def bwd(lib=lib, rec=rec, dx=dx, st=st):
                mean, _, invstd, dgamma, dbeta = st
                _C.check(lib.sonet_bn_cloud_partials_f32(p(x), p(dy), p(mean), p(invstd), p(gamma),
                                                         p(beta), B, C, P, 1, 1, p(rec), stream),
                         ENTRIES[0])
                _C.check(lib.sonet_bn_sync_backward_f32(p(rec), p(dy), p(x), p(mean), p(invstd),
                                                        p(gamma), p(beta), B, B, C, P, 1, p(dx),
                                                        p(dgamma), p(dbeta), stream), ENTRIES[2])
            out[k] = dict(forward=fwd, backward=bwd, stats=st)
            fwd()
            bwd()
        torch.cuda.synchronize()
        for direction in ("forward", "backward"):
            times = {k: [] for k in libs}
            for _ in range(a.reps):
                for k in libs:                     # alternate the builds within every repetition
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.inner):
                        out[k][direction]()
                    e1.record()
                    e1.synchronize()
                    times[k].append(e0.elapsed_time(e1) / a.inner)
            # forward: read x twice, write y; backward: read x and dy twice, write dx
            nbytes = (3 if direction == "forward" else 5) * 4 * B * C * P
            r = dict(B=B, C=C, P=P, direction=direction, gpu=gpu_info(), bytes_per_call=nbytes)
            for k in libs:
                r[k + "_ms"] = float(np.median(times[k]))
                r[k + "_ms_spread"] = [float(np.min(times[k])), float(np.max(times[k]))]
            if "baseline" in out and direction == "forward":
                v64 = x.double().var(dim=(0, 2), unbiased=False)
                for k in libs:
                    r[k + "_var_max_rel_err"] = float(((out[k]["stats"][1].double() - v64).abs() / v64).max())
            rows.append(r)
            print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
