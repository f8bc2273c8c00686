"""CUDA-event times of the three eval wgmma kernels in the default hi/lo split (3 fp16 products per
MAC) and the opt-in fp16 mode (1 product, the `_f16` entries), on the cfg-2 encoder's shapes
(B=64, N=5000, k=3, 8x8 SOM, som_k=9) and two generic-layer shapes. Modes alternate within each
repetition, so both see the same clocks; the L2 is flushed before every timed launch.

    python tools/fp16_kernel_time.py [--reps 15] [--json out.json]     (on a GPU box)
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "so-net_b200")):
    sys.path.insert(0, p)
import torch  # noqa: E402

from sonet_b200 import layers, ops, synth  # noqa: E402

DEV = "cuda"


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _cases():
    """name -> (launch(f16), useful FLOPs per launch)."""
    B, N, k, M, K = 64, 5000, 3, 64, 9
    torch.manual_seed(0)
    net = layers.PointResNet(6, [64, 128, 256, 384], 'relu', 'batch')
    net.load_state_dict(synth.synth_state_dict(net, seed=1))
    net = net.eval().to(DEV)
    blob, fpar = net._tc_params()
    inp = synth.synth_inputs(B, N, seed=0)
    pc, sn, node = inp["pc"].to(DEV), inp["sn"].to(DEV), inp["node"].to(DEV)
    a = ops.som_assign(pc, node, k)
    xs, ns, p0i = ops.som_sort_decenter(pc, sn, a["cluster_mean"], a["min_idx_i32"], a["count"], k)
    rows = B * k * N
    pr_flops = 2.0 * rows * (64 * 128 + 128 * 256 + 320 * 384)

    def pool(f16):
        ops.pointresnet_tc_pool(xs, blob, fpar, ns, p0i, M, f16=f16)

    def plain(f16):
        ops.pointresnet_tc(xs, blob, fpar, f16=f16)

    knn = layers.KNNModule(3 + 384, (512, 512), 'relu', 'batch').eval().to(DEV)
    pk = knn._tc_params()
    coord = torch.rand(B, 3, M, device=DEV) * 2 - 1
    idx = ops.node_knn(coord.contiguous(), K)
    y = torch.randn(B, M, 512, device=DEV).transpose(1, 2)

    def knn_l2(f16):
        ops.knn_mlp_tc(coord, coord, idx, K, y, pk["w1"], pk["blob2"], pk["inv2"], pk["shift2"],
                       f16=f16)

    def generic(Cin, Cout, Bg, P):
        x = torch.randn(Bg, Cin, P, device=DEV)
        W = torch.randn(Cout, Cin) * (2.0 / Cin) ** 0.5
        b, inv = ops.pointwise_tc_pack(W)
        b = b.to(DEV)
        sh = torch.zeros(Cout, device=DEV)
        return (lambda f16: ops.pointwise_layer_tc(x, b, inv, sh, Cout, True, f16=f16)), \
            2.0 * Bg * P * Cin * Cout

    return {
        "pointresnet_tc_pool (cfg-2, 960k rows)": (pool, pr_flops),
        "pointresnet_tc (cfg-2, 960k rows)": (plain, pr_flops),
        "knn_mlp_tc layer 2 (cfg-2, 36.9k rows)": (knn_l2, 2.0 * B * M * K * 512 * 512),
        "pointwise_tc 515->768 (final PointNet, 4096 rows)": generic(515, 768, B, M),
        "pointwise_tc 1024->512 (segmenter layer 2, 49k rows)": generic(1024, 512, 16, 3072),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    card = _card()
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=DEV)
    res = {}
    with torch.no_grad():
        for name, (fn, flops) in _cases().items():
            for f16 in (False, True):       # warm-up: module load, smem attribute
                fn(f16)
            torch.cuda.synchronize()
            ms = {False: [], True: []}
            for _ in range(args.reps):
                for f16 in (False, True):
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn(f16)
                    e1.record()
                    torch.cuda.synchronize()
                    ms[f16].append(e0.elapsed_time(e1))
            row = {}
            for f16, mode in ((False, "split"), (True, "fp16")):
                t = sorted(ms[f16])
                med = t[len(t) // 2]
                row[mode] = dict(median_ms=med, min_ms=t[0], max_ms=t[-1],
                                 useful_tflops=flops / med / 1e9)
            row["speedup"] = row["split"]["median_ms"] / row["fp16"]["median_ms"]
            res[name] = row
            print("%-52s split %.4f ms (%.0f TFLOP/s)  fp16 %.4f ms (%.0f TFLOP/s)  x%.2f"
                  % (name, row["split"]["median_ms"], row["split"]["useful_tflops"],
                     row["fp16"]["median_ms"], row["fp16"]["useful_tflops"], row["speedup"]))
    print("card:", card, "| medians of %d alternated launches, L2 flushed" % args.reps)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card, reps=args.reps, kernels=res), f, indent=1)


if __name__ == "__main__":
    main()
