"""Eval-forward time of the cfg-3 segmenter (B=32, N=1024) and the cfg-4 auto-encoder shapes (B=32,
N=5000; output_fc_pc_num=0, since the reference's FC branch cannot run with instance norm) built
with normalization='batch' and 'instance', and of the instance models on the PyTorch composition
they ran on before the instance-norm kernel (layers.KERNEL_NORMALIZATIONS = (None, 'batch')).
Arms alternate within each round. Prints one JSON line per (config, arm) with CUDA-event times,
and one per config with the instance-norm kernel's own time (CUDA events around each launch of
one forward, ops.PROFILE) and achieved bytes/s against the H100 SXM's 3.35 TB/s: every launch
reads z once and writes its output once (4 bytes each). The card's name and power limit are read
in the same call.

    python tools/norm_bench.py [--steps 20] [--warmup 3] [--rounds 3]
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
from sonet_b200 import autoencoder, layers, networks, ops, segmenter, synth  # noqa: E402

CONFIGS = {"cfg3": ("segmenter", 32, 1024), "cfg4": ("autoencoder", 32, 5000)}
HBM_BYTES_PER_S = 3.35e12


def build(task, B, N, norm):
    kw = dict(normalization=norm, output_fc_pc_num=0) if task == "autoencoder" else \
        dict(normalization=norm)
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, device="cuda:0", **kw)
    cpu = synth.make_opt(task, batch_size=B, input_pc_num=N, **kw)
    inp = synth.synth_inputs(B, N, seed=0)
    m = {"segmenter": segmenter, "autoencoder": autoencoder}[task].Model(opt)
    m.encoder.load_state_dict(synth.synth_state_dict(networks.Encoder(cpu), seed=1))
    if task == "segmenter":
        m.segmenter.load_state_dict(synth.synth_state_dict(networks.Segmenter(cpu), seed=2))
        m.set_input(inp["pc"], inp["sn"], inp["label"], torch.zeros(B, N, dtype=torch.int64),
                    inp["node"], inp["node_knn_I"])
    else:
        m.decoder.load_state_dict(synth.synth_state_dict(networks.Decoder(cpu), seed=2))
        m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    return m


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sum(ts) / len(ts)


def kernel_share(m, B):
    """(ms, bytes) of the instance-norm launches of one forward, and the bytes per cloud."""
    ops.PROFILE = []
    try:
        m.test_model()
        torch.cuda.synchronize()
        calls = [(e0.elapsed_time(e1), a) for n, e0, e1, a in ops.PROFILE
                 if n == "sonet_instance_norm_f32"]
    finally:
        ops.PROFILE = None
    ms = sum(t for t, _ in calls)
    nbytes = 0
    for _, a in calls:
        b, c, p, reduce, k = a[3], a[4], a[5], a[8], a[9]
        nbytes += 4 * b * c * p + 4 * b * c * (p if reduce == ops.REDUCE_NONE else p // k)
    return ms, nbytes, len(calls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "norm_bench needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    kernel_norms = layers.KERNEL_NORMALIZATIONS
    for cfg, (task, B, N) in CONFIGS.items():
        models = {"batch": build(task, B, N, "batch"), "instance": build(task, B, N, "instance")}
        arms = [("batch", models["batch"], kernel_norms),
                ("instance", models["instance"], kernel_norms),
                ("instance_pytorch", models["instance"], (None, "batch"))]
        times = {a: [] for a, _, _ in arms}
        with torch.no_grad():
            for _ in range(args.rounds):
                for arm, m, norms in arms:
                    layers.KERNEL_NORMALIZATIONS = norms
                    try:
                        times[arm].append(timed(m.test_model, args.steps, args.warmup))
                    finally:
                        layers.KERNEL_NORMALIZATIONS = kernel_norms
            ms, nbytes, n = kernel_share(models["instance"], B)
        for arm, ts in times.items():
            print(json.dumps(dict(config=cfg, task=task, B=B, N=N, arm=arm, ms_best=min(ts),
                                  ms_rounds=[round(t, 4) for t in ts], card=card)))
        print(json.dumps(dict(config=cfg, kernel="sonet_instance_norm_f32", launches=n,
                              kernel_ms=round(ms, 4), mbytes=round(nbytes / 1e6, 1),
                              mbytes_per_cloud=round(nbytes / 1e6 / B, 1),
                              tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
                              share_of_hbm=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3),
                              card=card)))


if __name__ == "__main__":
    main()
