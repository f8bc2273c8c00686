"""Time one classifier training step (forward + backward + Adam) with the sm_90a train kernels
(sonet_b200/train_ops.py) against the PyTorch composition the reference trains with.
    python tools/train_step_bench.py [--batch 32] [--npts 5000] [--steps 6]"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "so-net_b200")):
    sys.path.insert(0, p)
import torch  # noqa: E402

from sonet_b200 import classifier, networks, synth, train_ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--npts", type=int, default=5000)
ap.add_argument("--steps", type=int, default=6)
a = ap.parse_args()
B, N = a.batch, a.npts
inp = synth.synth_inputs(B, N, seed=0)


def run(enabled, tf32):
    train_ops.ENABLED = enabled
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device="cuda:0")
    cpu = synth.make_opt("classifier", batch_size=B, input_pc_num=N)
    m = classifier.Model(opt)
    m.encoder.load_state_dict(synth.synth_state_dict(networks.Encoder(cpu), seed=1))
    m.classifier.load_state_dict(synth.synth_state_dict(networks.Classifier(cpu), seed=2))
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    for _ in range(2):
        m.optimize()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        m.optimize()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    return ms, float(m.loss)


for name, en, tf in (("sonet train kernels (wgmma fwd/dgrad/wgrad, fused BN)", True, False),
                     ("PyTorch composition, strict fp32", False, False),
                     ("PyTorch composition, TF32 allowed (torch default for cuDNN)", False, True)):
    ms, loss = run(en, tf)
    print("%-62s %8.2f ms/step  %7.1f clouds/s  loss %.4f" % (name, ms, B / ms * 1e3, loss))
train_ops.ENABLED = True
