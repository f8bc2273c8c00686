"""Time the auto-encoder's training step and its decoder's six up-convolution stages with the sm_90a
train kernels (train_ops.UpConvTC + the shared norm / activation kernels) against the PyTorch
composition the reference trains with (nearest x2 up-sampling + cuDNN 3x3 conv + batch_norm + act).

    python tools/ae_train_bench.py [--batch 32] [--npts 5000] [--steps 6] [--rounds 3] [--iters 50]

1. autoencoder.Model.optimize() at the cfg-4 shape: kernels on, kernels off in strict fp32, kernels
   off with TF32 allowed, alternated over --rounds rounds (the median of each is printed).
2. Each DecoderConv stage (feature_num 1024) alone, forward + backward in train mode, both paths
   (the kernels forced on every stage, whichever side of train_ops.UPCONV_MIN_HW it falls),
   CUDA events over --iters launches after a warm-up; the parity-form FLOP count (16/36 of the
   direct 3x3 work on the up-sampled grid) turns the times into rates. A stage whose output does not
   reach the loss (deconv6 unless output_conv_pc_num = 4096) still has its backward timed here.
3. Where one kernels step of each stage goes, per C-ABI entry, and the copy of dz's parity planes
   the wgrad reads.
The card's name and power limit are read once and printed with the numbers."""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "so-net_b200")):
    sys.path.insert(0, p)
import torch  # noqa: E402

from sonet_b200 import autoencoder, layers, networks, ops, synth, train_ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--npts", type=int, default=5000)
ap.add_argument("--steps", type=int, default=6)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--iters", type=int, default=50)
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("ae_train_bench: needs a CUDA device")
B, N = a.batch, a.npts


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return "%s, power limit %s" % (name, pl or "unknown")


MODES = (("train kernels (wgmma parity GEMMs fwd/dgrad/wgrad)", True, False),
         ("PyTorch composition, strict fp32", False, False),
         ("PyTorch composition, TF32 allowed", False, True))


def set_mode(enabled, tf32):
    train_ops.ENABLED = enabled
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32


def make_model():
    opt = synth.make_opt("autoencoder", batch_size=B, input_pc_num=N, device="cuda:0")
    cpu = synth.make_opt("autoencoder", batch_size=B, input_pc_num=N)
    m = autoencoder.Model(opt)
    m.encoder.load_state_dict(synth.synth_state_dict(networks.Encoder(cpu), seed=1))
    m.decoder.load_state_dict(synth.synth_state_dict(networks.Decoder(cpu), seed=2))
    inp = synth.synth_inputs(B, N, seed=0)
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    return m


def time_steps(m, mode):
    set_mode(*mode[1:])
    for _ in range(2):
        m.optimize()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        m.optimize()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / a.steps, float(m.loss)


print("card:", card())
print("== autoencoder.Model.optimize(), B=%d N=%d, %d steps per timing, %d rounds alternated" % (
    B, N, a.steps, a.rounds))
models = [make_model() for _ in MODES]
times = [[] for _ in MODES]
for r in range(a.rounds):
    for i, mode in enumerate(MODES):
        ms, loss = time_steps(models[i], mode)
        times[i].append((ms, loss))
for (name, _, _), t in zip(MODES, times):
    ms = statistics.median(x[0] for x in t)
    print("%-52s %8.2f ms/step  %7.1f clouds/s  (rounds: %s; first loss %.5f)" % (
        name, ms, B / ms * 1e3, " ".join("%.2f" % x[0] for x in t), t[0][1]))

STAGES = [("deconv1", 1024, 1024, 1), ("deconv2", 1024, 512, 2), ("deconv3", 512, 256, 4),
          ("deconv4", 256, 128, 8), ("deconv5", 128, 128, 16), ("deconv6", 128, 128, 32)]


def stage_time(mod, x, w, mode):
    set_mode(*mode[1:])
    train_ops.UPCONV_MIN_HW = 1          # both sides of the map-size rule, every stage
    xg = x.clone().requires_grad_(True)

    def step():
        mod.zero_grad(set_to_none=True)
        xg.grad = None
        mod(xg).backward(w)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        step()
    e1.record()
    torch.cuda.synchronize()
    elapsed = e0.elapsed_time(e1) / a.iters
    train_ops.UPCONV_MIN_HW = MIN_HW
    return elapsed


def kernel_breakdown(mod, x, w, cout, h):
    set_mode(*MODES[0][1:])
    train_ops.UPCONV_MIN_HW = 1
    xg = x.clone().requires_grad_(True)
    ops.PROFILE = []
    try:
        mod(xg).backward(w)
        torch.cuda.synchronize()
        agg = {}
        for n, e0, e1, _ in ops.PROFILE:
            agg[n] = agg.get(n, 0.0) + e0.elapsed_time(e1)
    finally:
        ops.PROFILE = None
        train_ops.UPCONV_MIN_HW = MIN_HW
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        w.view(B, cout, h, 2, h, 2).permute(3, 5, 0, 1, 2, 4).reshape(4, B, cout, h * h)
    e1.record()
    torch.cuda.synchronize()
    agg["parity-plane copy"] = e0.elapsed_time(e1) / a.iters
    return sorted(agg.items(), key=lambda kv: -kv[1])


MIN_HW = train_ops.UPCONV_MIN_HW
breakdown = []
print("(optimize() above takes the parity-GEMM kernels for input maps >= %d pixels; the table "
      "below times the kernels at every stage)" % MIN_HW)
print("== DecoderConv stages alone, train mode, forward + backward (dx, dW, db, BN), B=%d, %d iters"
      % (B, a.iters))
print("%-8s %-16s %12s %12s %9s %14s %14s" % ("stage", "Cin>Cout map", "kernels ms", "cuDNN ms",
                                              "speedup", "kern TFLOP/s", "cuDNN TFLOP/s"))
torch.manual_seed(0)
for name, cin, cout, h in STAGES:
    mod = layers.UpConv(cin, cout, activation="relu", normalization="batch").cuda().train()
    x = torch.randn(B, cin, h, h, device="cuda")
    w = torch.randn(B, cout, 2 * h, 2 * h, device="cuda")
    # parity-form work: forward, dgrad and wgrad are each 16 * B * H*W * Cin * Cout MACs
    flop = 3 * 2 * 16 * B * h * h * cin * cout
    tk = stage_time(mod, x, w, MODES[0])
    tc = stage_time(mod, x, w, MODES[1])
    print("%-8s %4d>%-4d %2dx%-2d %12.3f %12.3f %8.2fx %14.1f %14.1f" % (
        name, cin, cout, h, h, tk, tc, tc / tk, flop / tk / 1e9, flop / tc / 1e9))
    breakdown.append((name, kernel_breakdown(mod, x, w, cout, h)))
print("== where a kernels step goes: CUDA events around each C-ABI call of one forward + backward "
      "(summed per entry, ms), and the copy of dz's four parity planes the wgrad reads")
for name, parts in breakdown:
    print("%-8s %s" % (name, ", ".join("%s %.3f" % kv for kv in parts)))
set_mode(True, False)
