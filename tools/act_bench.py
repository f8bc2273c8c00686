"""Eval-forward time of the cfg-2 classifier (B=64, N=5000) and the cfg-3 segmenter (B=32, N=1024)
built with activation='relu' and 'elu', and of the ELU models on the PyTorch composition they ran on
before the kernels had an ELU epilogue (every layer treated as kernel-ineligible). Prints one JSON
line per (config, arm) with the mean and spread of CUDA-event times, and the card it ran on.

    python tools/act_bench.py [--steps 20] [--warmup 3] [--rounds 3]
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
from sonet_b200 import classifier, layers, networks, segmenter, synth  # noqa: E402

CONFIGS = {"cfg2": ("classifier", 64, 5000), "cfg3": ("segmenter", 32, 1024)}


def build(task, B, N, act):
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, device="cuda:0", activation=act)
    cpu = synth.make_opt(task, batch_size=B, input_pc_num=N, activation=act)
    inp = synth.synth_inputs(B, N, seed=0)
    m = {"classifier": classifier, "segmenter": segmenter}[task].Model(opt)
    m.encoder.load_state_dict(synth.synth_state_dict(networks.Encoder(cpu), seed=1))
    if task == "segmenter":
        m.segmenter.load_state_dict(synth.synth_state_dict(networks.Segmenter(cpu), seed=2))
        m.set_input(inp["pc"], inp["sn"], inp["label"], torch.zeros(B, N, dtype=torch.int64),
                    inp["node"], inp["node_knn_I"])
    else:
        m.classifier.load_state_dict(synth.synth_state_dict(networks.Classifier(cpu), seed=2))
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "act_bench needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    kernel_acts = layers.KERNEL_ACTIVATIONS
    for cfg, (task, B, N) in CONFIGS.items():
        models = {"relu": build(task, B, N, "relu"), "elu": build(task, B, N, "elu")}
        arms = [("relu", models["relu"], kernel_acts), ("elu", models["elu"], kernel_acts),
                ("elu_pytorch", models["elu"], (None, "relu"))]
        times = {a: [] for a, _, _ in arms}
        with torch.no_grad():
            for _ in range(args.rounds):        # arms alternate within each round
                for arm, m, acts in arms:
                    layers.KERNEL_ACTIVATIONS = acts
                    try:
                        times[arm].append(timed(m.test_model, args.steps, args.warmup))
                    finally:
                        layers.KERNEL_ACTIVATIONS = kernel_acts
        for arm, ts in times.items():
            print(json.dumps(dict(config=cfg, task=task, B=B, N=N, arm=arm, ms_best=min(ts),
                                  ms_rounds=[round(t, 4) for t in ts], card=card)))


if __name__ == "__main__":
    main()
