"""Timing probe of the generic wgmma layer at a given shape, with / without the gathered addend
(segmenter head layer 1). usage: python tools/probe_layer.py [B C P Cout]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "so-net_b200")):
    sys.path.insert(0, p)
import torch  # noqa: E402

from sonet_b200 import ops  # noqa: E402

B, C, P, COUT = [int(v) for v in (sys.argv[1:5] if len(sys.argv) >= 5 else (32, 396, 3072, 1024))]
C0 = int(sys.argv[5]) if len(sys.argv) >= 6 else 0      # > 0: two sources x0 [C0] + x1 [C - C0]
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(1)
x = torch.randn(B, C, P, generator=g).to(dev)
w = (torch.randn(COUT, C, generator=g) * 0.05)
blob, inv = ops.pointwise_tc_pack(w)
blob = blob.to(dev)
shift = torch.randn(COUT, generator=g).to(dev)
M = 64
addend = torch.randn(B, COUT, M, generator=g).to(dev)
gidx = torch.randint(0, M, (B, P), generator=g, dtype=torch.int32).to(dev)
gsorted = torch.sort(gidx, dim=1)[0].contiguous()
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def t(fn, reps=5):
    best = 1e9
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best


fl = 2.0 * C * COUT * B * P * 3
xa = x[:, :C0].contiguous() if C0 else None
xb = x[:, C0:].contiguous() if C0 else None
extra = ()
if C0:
    extra = (("two sources", lambda: ops.pointwise_layer_tc(xa, blob, inv, shift, COUT, True, x1=xb)),
             ("two sources+addend", lambda: ops.pointwise_layer_tc(xa, blob, inv, shift, COUT, True, x1=xb,
                                                                   addend=addend, gidx=gidx)))
for name, fn in extra + (
        ("plain", lambda: ops.pointwise_layer_tc(x, blob, inv, shift, COUT, True)),
        ("addend random idx", lambda: ops.pointwise_layer_tc(x, blob, inv, shift, COUT, True,
                                                             addend=addend, gidx=gidx)),
        ("addend sorted idx", lambda: ops.pointwise_layer_tc(x, blob, inv, shift, COUT, True,
                                                             addend=addend, gidx=gsorted))):
    ms = t(fn)
    print("%-20s %.1f us  executed %.0f TFLOP/s  out %.0f GB/s" %
          (name, ms * 1e3, fl / ms / 1e9, B * COUT * P * 4 / ms / 1e6))
