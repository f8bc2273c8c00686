"""-m gpu: the opt-in fp16 mode (SONET_TC=fp16): every eval-mode wgmma GEMM as ONE fp16 product
per MAC, y = (sum_k rn16sat(x_k) * rn16(s * w_k)) / s with fp32 accumulation.

  1. each `_f16` entry against an fp64 GEMM of the rounded operands, at the generic layer's tile
     edges and in all its modes, and the KNN kernel on both Y layouts. A kernel that still adds a
     lo product lands ~2^-11 of sum |w x| away from this reference, ~500x outside the bar;
  2. the fused first PointResNet against the layer chain emulated in fp64 with rounding at every
     wgmma input, and its pool variant against the per-node max of the plain variant, bit for bit;
  3. the classifier, segmenter and auto-encoder goldens under SONET_TC=fp16;
  4. every tensor-core launch of an fp16 forward is an `_f16` entry, and none of a default one;
  5. CUDA-graph replays follow SONET_TC flips; 6. train mode ignores the mode;
  7. determinism, saturation beyond 65504 and NaN inputs as the split handles them.
"""
import contextlib
import glob
import os

import pytest
import torch

from helpers import F16_C, GOLDEN, build_states, golden, golden_case, sampled

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# The error bar of one fp16-mode GEMM output, F16_C, is stated (and its calibration recorded) in
# helpers.py.
# Model-level bound under SONET_TC=fp16, per output tensor: max |got - golden| / max |golden|.
# Measured on the same card over every fixture and the encoder tensors below: 1.4e-3 at most
# (the auto-encoder's and segmenter's outputs; 2.9e-4 .. 8.6e-4 for the classifier scores and the
# encoder tensors). The bound is 2.5x that.
F16_MODEL_REL = 3.5e-3

TC_ENTRIES = ("sonet_pointresnet_tc_forward", "sonet_pointresnet_tc_pool_forward",
              "sonet_pointwise_tc_forward", "sonet_pointwise_tc_forward_rows",
              "sonet_pointwise_tc_grouped_forward", "sonet_knn_mlp_tc_forward")


@contextlib.contextmanager
def profiled():
    from sonet_b200 import ops
    calls = []
    ops.PROFILE = calls
    try:
        yield calls
    finally:
        ops.PROFILE = None


@contextlib.contextmanager
def tc_mode(value):
    """SONET_TC = value (None: unset) inside the block."""
    old = os.environ.get("SONET_TC")
    if value is None:
        os.environ.pop("SONET_TC", None)
    else:
        os.environ["SONET_TC"] = value
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("SONET_TC", None)
        else:
            os.environ["SONET_TC"] = old


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def r16(x):
    """fp16 round-to-nearest with saturation to +-65504 (cvt.rn.satfinite), NaN kept, as fp64."""
    return x.clamp(-65504.0, 65504.0).half().double()


def w16(W, inv):
    """The hi image of a blob: rn16(s * W) with s = 1 / inv (a power of two), as fp64."""
    return (W.to(DEV, torch.float32) * (1.0 / inv)).half().double()


_WORST = {}


def check(got, y, m, what, relu=False):
    """|got - y| <= F16_C * m everywhere (relu applied to y here); records err / m."""
    if relu:
        y = y.clamp(min=0)
    got = got.to(y.device, torch.float64)
    err = (got - y).abs()
    rel = float((err / m.clamp(min=1e-300)).max())
    _WORST[what] = rel
    print("\n[fp16] %s: max err / m = %.3e" % (what, rel))
    assert bool(torch.isfinite(got).all()), what
    assert bool((err <= F16_C * m).all()), "%s: err / m = %.3e > F16_C = %.1e" % (what, rel, F16_C)


def gemm16(W16, inv, X16):
    """fp64 (W16 x16) / s and sum |W16 x16| / s over the channel axis of X16 [B,K,P]."""
    y = torch.einsum("ok,bkp->bop", W16, X16) * inv
    m = torch.einsum("ok,bkp->bop", W16.abs(), X16.abs()) * inv
    return y, m


# ---- 1a. the generic layer, plain and point-major rows -----------------------------------------
# (B, C0, C1, P, Cout, relu, shift, G): K remainders 16/32/48/64 over 1-7 chunks, Cout not a
# multiple of 128 or 256, rows not a multiple of 128, two sources, gathered addends
SHAPES = [
    (1, 3, 0, 100, 1, True, True, 0),          # rem 16; rows < 128
    (1, 20, 0, 255, 3, False, True, 0),        # rem 32; 2 * 128 - 1 rows
    (1, 40, 0, 257, 50, True, False, 0),       # rem 48; 2 * 128 + 1 rows
    (3, 64, 0, 43, 64, True, True, 0),         # rem 64; P < 64
    (2, 100, 0, 128, 127, True, True, 0),      # 2 chunks rem 48
    (1, 130, 0, 383, 129, True, True, 0),      # 3 chunks rem 16; widths 128 + 64
    (1, 224, 0, 640, 385, True, True, 0),      # 4 chunks rem 32; n-tile 1 widths 128 + 64
    (1, 424, 0, 129, 1000, True, True, 0),     # 7 chunks rem 48; Cout 1000
    (2, 387, 0, 576, 512, True, True, 0),      # the KNN module's first layer
    (1, 31, 33, 300, 200, True, True, 0),      # two sources
    (3, 63, 130, 65, 257, True, True, 0),      # two sources, rem 16 across them
    (2, 396, 0, 300, 1024, True, False, 64),   # the segmenter's gathered addend
    (3, 128, 0, 99, 300, False, True, 7),      # G = 7, no ReLU
]


def _shape_id(c):
    return "B%d-C%d+%d-P%d-O%d%s%s%s" % (c[0], c[1], c[2], c[3], c[4], "" if c[5] else "-lin",
                                           "" if c[6] else "-noshift", "-G%d" % c[7] if c[7] else "")


def _layer_case(B, C0, C1, P, Cout, relu, with_shift, G, seed, xscale=1.0):
    from sonet_b200 import ops
    g = _gen(seed)
    Cin = C0 + C1
    x = (torch.randn(B, Cin, P, generator=g).clamp(-3.5, 3.5) * xscale).to(DEV)
    W = torch.randn(Cout, Cin, generator=g) * (2.0 / Cin) ** 0.5
    shift = (torch.randn(Cout, generator=g) * 0.3).to(DEV) if with_shift else None
    add = gidx = None
    if G:
        add = torch.randn(B, Cout, G, generator=g).to(DEV)
        gidx = torch.randint(0, G, (B, P), generator=g).int().to(DEV)
    blob, inv = ops.pointwise_tc_pack(W)
    x0, x1 = x[:, :C0].contiguous(), (x[:, C0:].contiguous() if C1 else None)
    args = (x0, blob.to(DEV), inv, shift, Cout, relu)
    kw = dict(x1=x1, addend=add, gidx=gidx)
    y, m = gemm16(w16(W, inv), inv, r16(x))
    if shift is not None:
        y = y + shift.double()[None, :, None]
        m = m + shift.double().abs()[None, :, None]
    if add is not None:
        ga = torch.gather(add, 2, gidx.long()[:, None, :].expand(B, Cout, P)).double()
        y, m = y + ga, m + ga.abs()
    return args, kw, y, m


@pytest.mark.parametrize("rows", [False, True], ids=["channel-major", "rows"])
@pytest.mark.parametrize("case", SHAPES, ids=_shape_id)
def test_generic_layer_f16(case, rows):
    from sonet_b200 import ops
    B, C0, C1, P, Cout, relu, sh, G = case
    args, kw, y, m = _layer_case(*case, seed=sum(case[:5]))
    with profiled() as calls:
        got = ops.pointwise_layer_tc(*args, **kw, rows=rows, f16=True)
    again = ops.pointwise_layer_tc(*args, **kw, rows=rows, f16=True)
    want = "sonet_pointwise_tc_forward_rows_f16" if rows else "sonet_pointwise_tc_forward_f16"
    assert [c[0] for c in calls] == [want]
    assert torch.equal(got, again), "re-run differs"
    if rows:
        got = got.transpose(1, 2)
        assert torch.equal(got, ops.pointwise_layer_tc(*args, **kw, f16=True))
    check(got, y, m, "layer %s%s" % (_shape_id(case), " rows" if rows else ""), relu=relu)
    assert not torch.equal(ops.pointwise_layer_tc(*args, **kw), got), "the split's result"


@pytest.mark.parametrize("xscale", [2.0 ** -14, 2.0 ** 8], ids=["2^-14", "2^8"])
def test_generic_layer_f16_input_scale(xscale):
    """Small activations are fp16 subnormals (rn16 rounds them absolutely, the reference does the
    same); large ones stay inside fp16's range."""
    from sonet_b200 import ops
    args, kw, y, m = _layer_case(2, 256, 0, 700, 192, True, False, 0, seed=5, xscale=xscale)
    got = ops.pointwise_layer_tc(*args, **kw, f16=True)
    check(got, y, m, "layer x%.3g" % xscale, relu=True)


# ---- 1b. grouped, split-K and parity scatter ------------------------------------------------------
def _grouped_ref(Wg, inv, xg, groups, B, shift, relu, scat_w):
    """fp64 reference of the grouped launch from the group operands xg [G*B, K, P]."""
    ys, ms = [], []
    for gi in range(groups):
        y, m = gemm16(w16(Wg[gi], inv), inv, r16(xg[gi * B:(gi + 1) * B]))
        if shift is not None:
            y = y + shift.double()[None, :, None]
            m = m + shift.double().abs()[None, :, None]
        ys.append(y.clamp(min=0) if relu else y)
        ms.append(m)
    if not scat_w:
        return torch.cat(ys), torch.cat(ms)
    Bq, Cout, P = ys[0].shape
    H = P // scat_w
    out_y = ys[0].new_zeros(Bq, Cout, 2 * H, 2 * scat_w)
    out_m = torch.zeros_like(out_y)
    for gi in range(4):
        py, px = gi >> 1, gi & 1
        out_y[:, :, py::2, px::2] = ys[gi].view(Bq, Cout, H, scat_w)
        out_m[:, :, py::2, px::2] = ms[gi].view(Bq, Cout, H, scat_w)
    return out_y.view(Bq, Cout, -1), out_m.view(Bq, Cout, -1)


@pytest.mark.parametrize("splits", [1, 2, 4])
def test_grouped_split_k_f16(splits):
    """One group, K split over CTAs (the segmenter's node-level GEMM)."""
    from sonet_b200 import ops
    g = _gen(60 + splits)
    B, Cin, P, Cout = 2, 2048, 100, 1024                              # 32 K chunks
    x = torch.randn(B, Cin, P, generator=g).to(DEV)
    Wg = torch.randn(1, Cout, Cin, generator=g) * (2.0 / Cin) ** 0.5
    blob, per, inv = ops.pointwise_tc_pack_groups(Wg)
    blob = blob.to(DEV)
    with profiled() as calls:
        got = ops.pointwise_tc_grouped(x, blob, per, inv, None, Cout, False, groups=1, splits=splits,
                                       f16=True)
    assert [c[0] for c in calls] == ["sonet_pointwise_tc_grouped_forward_f16"]
    assert calls[0][3][11] == splits
    again = ops.pointwise_tc_grouped(x, blob, per, inv, None, Cout, False, groups=1, splits=splits,
                                     f16=True)
    assert torch.equal(got, again), "re-run differs"
    y, m = _grouped_ref(Wg, inv, x, 1, B, None, False, 0)
    check(got, y, m, "grouped splits=%d" % splits)


@pytest.mark.parametrize("conv", [False, True], ids=["im2col", "conv"])
@pytest.mark.parametrize("splits", [1, 2])
def test_upconv_parity_scatter_f16(conv, splits):
    """Four parity groups of a x2 up-convolution scattered into the output map, from the im2col
    operand or (conv) from the three horizontally shifted copies with in-kernel vertical shifts."""
    from sonet_b200 import ops
    g = _gen(70 + splits + 2 * conv)
    B, Cin, H, W, Cout = 2, 64, 8, 16, 130
    img = torch.randn(B, Cin, H, W, generator=g).to(DEV)
    Wg = torch.randn(4, Cout, 4 * Cin, generator=g) * (2.0 / (4 * Cin)) ** 0.5
    shift = (torch.randn(Cout, generator=g) * 0.3).to(DEV)
    blob, per, inv = ops.pointwise_tc_pack_groups(Wg)
    blob = blob.to(DEV)
    xcol = ops.upconv_im2col(img)                                     # [4B, 4Cin, HW]
    xin = ops.upconv_hshift(img) if conv else xcol
    with profiled() as calls:
        got = ops.pointwise_tc_grouped(xin, blob, per, inv, shift, Cout, True, groups=4,
                                       splits=splits, scat_w=W, conv=conv, f16=True)
    assert "sonet_pointwise_tc_grouped_forward_f16" in [c[0] for c in calls]
    again = ops.pointwise_tc_grouped(xin, blob, per, inv, shift, Cout, True, groups=4,
                                     splits=splits, scat_w=W, conv=conv, f16=True)
    assert torch.equal(got, again), "re-run differs"
    y, m = _grouped_ref(Wg, inv, xcol, 4, B, shift, True, W)
    check(got, y, m, "upconv scatter splits=%d %s" % (splits, "conv" if conv else "im2col"))


# ---- 1c. the fused KNN kernel ---------------------------------------------------------------------
def _fma32(a, b, c):
    """fp32 fmaf(a, b, c): the product is exact in fp64, then one rounding to fp32."""
    return (a.double() * b.double() + c.double()).float()


@pytest.mark.parametrize("yvec", [False, True], ids=["Y-channel-major", "Y-node-major"])
@pytest.mark.parametrize("K", [2, 9, 16])
def test_knn_mlp_f16(K, yvec):
    from sonet_b200 import ops
    g = _gen(80 + K + yvec)
    B, M = 3, 40
    coord = (torch.rand(B, 3, M, generator=g) * 2 - 1).to(DEV)
    center = (torch.rand(B, 3, M, generator=g) * 2 - 1).to(DEV)
    idx = torch.randint(0, M, (B, M, K + 2), generator=g).to(DEV)
    W1d = torch.randn(512, 3, generator=g)
    s1 = torch.randn(512, generator=g) * 0.2
    w1 = torch.cat((W1d, s1[:, None]), 1).contiguous().to(DEV)
    W2 = torch.randn(512, 512, generator=g) * (2.0 / 512) ** 0.5
    s2 = (torch.randn(512, generator=g) * 0.2).to(DEV)
    blob, inv = ops.knn_mlp_tc_pack(W2)
    blob = blob.to(DEV)
    y_cm = (torch.randn(B, 512, M, generator=g) * 2).to(DEV)
    Y = y_cm.transpose(1, 2).contiguous().transpose(1, 2) if yvec else y_cm
    with profiled() as calls:
        got = ops.knn_mlp_tc(coord, center, idx, K, Y, w1, blob, inv, s2, f16=True)
    assert [c[0] for c in calls] == ["sonet_knn_mlp_tc_forward_f16"]
    assert (calls[0][3][8] == 1) == yvec                              # y_cstride: the YVEC path
    assert torch.equal(got, ops.knn_mlp_tc(coord, center, idx, K, Y, w1, blob, inv, s2, f16=True))
    # layer 1 as the kernel computes it in fp32: v = Y + shift1, then three fmaf, ReLU
    nb = idx[:, :, :K]                                                # [B,M,K]
    bi = torch.arange(B, device=DEV)[:, None, None]
    dec = [(coord[:, c][bi, nb] - center[:, c][:, :, None]) for c in range(3)]   # [B,M,K] fp32
    yg = y_cm.transpose(1, 2)[bi, nb]                                 # [B,M,K,512]
    w1d = w1.to(DEV)
    v = yg + w1d[:, 3]
    for c in range(3):
        v = _fma32(w1d[:, c], dec[c][..., None], v)
    h1 = r16(v.clamp(min=0)).view(B, M * K, 512).transpose(1, 2)      # [B,512,M*K]
    y2, m2 = gemm16(w16(W2, inv), inv, h1)
    y2 = (y2 + s2.double()[None, :, None]).clamp(min=0).view(B, 512, M, K).amax(3)
    m2 = (m2 + s2.double().abs()[None, :, None]).view(B, 512, M, K).amax(3)
    check(got, y2, m2, "knn K=%d %s" % (K, "node-major" if yvec else "channel-major"))


# ---- 2. the fused first PointResNet --------------------------------------------------------------
def _resnet(cin, seed):
    from sonet_b200 import layers, synth
    net = layers.PointResNet(cin, [64, 128, 256, 384], 'relu', 'batch')
    net.load_state_dict(synth.synth_state_dict(net, seed=seed))
    return net.eval().to(DEV)


def _r16_slack(h, e):
    """(rn16(h), delta): where h (fp64) lies within e of a rounding midpoint of fp16, a value the
    kernel holds within e of h may round to the neighbour: delta is that neighbour's distance,
    else 0. h >= 0 (ReLU outputs), below 65504."""
    hv = h.half()
    bits = hv.view(torch.int16)
    up = (bits + 1).view(torch.float16).double()
    down = torch.where(bits > 0, (bits - 1).view(torch.float16).double(), hv.double() - 2.0 ** -24)
    hd = hv.double()
    near = (h + e >= (hd + up) / 2) | (h - e <= (hd + down) / 2)
    return hd, torch.where(near, torch.maximum(up - hd, hd - down), torch.zeros_like(hd))


def _resnet_chain16(net, x):
    """Layer 0 in fp32 as the kernel runs it; layers 1-3 in fp64 on fp16-rounded inputs, with the
    error bar carried along the chain. Returns (y [B,384,P], bar)."""
    blob, fpar = net._tc_params()
    f = fpar.to(DEV)
    W0 = f[:384].view(64, 6)
    sh0 = f[384:448]
    inv1, inv2, inv3 = (float(v) for v in f[1216:1219])
    (_, _), (w1, s1), (w2, s2), (w3, s3) = [l.folded() for l in net.layers]
    B, cin, P = x.shape
    a = sh0[None, :, None].expand(B, 64, P)
    for c in range(6):
        xc = x[:, c:c + 1] if c < cin else torch.zeros_like(x[:, :1])
        a = _fma32(W0[None, :, c, None], xc, a)
    act0 = r16(a.clamp(min=0))
    W1, W2, W3 = w16(w1, inv1), w16(w2, inv2), w16(w3, inv3)
    y1, m1 = gemm16(W1, inv1, act0)
    y1, m1 = y1 + s1.double()[None, :, None], m1 + s1.double().abs()[None, :, None]
    h1, d1 = _r16_slack(y1.clamp(min=0), F16_C * m1)
    y2, m2 = gemm16(W2, inv2, h1)
    e2 = F16_C * (m2 + s2.double().abs()[None, :, None]) + torch.einsum("ok,bkp->bop", W2.abs(), d1) * inv2
    y2 = y2 + s2.double()[None, :, None]
    h2, d2 = _r16_slack(y2.clamp(min=0), e2)
    y3, m3 = gemm16(W3, inv3, torch.cat((act0, h2), 1))
    e3 = F16_C * (m3 + s3.double().abs()[None, :, None]) \
        + torch.einsum("ok,bkp->bop", W3[:, 64:].abs(), d2) * inv3
    return y3 + s3.double()[None, :, None], e3, (float((d1 > 0).double().mean()),
                                                 float((d2 > 0).double().mean()))


@pytest.mark.parametrize("cin,B,P", [(3, 2, 77), (6, 1, 1000), (6, 3, 383)])
def test_pointresnet_f16_chain(cin, B, P):
    from sonet_b200 import ops
    net = _resnet(cin, seed=cin * 100 + P)
    x = (torch.rand(B, cin, P, generator=_gen(P)) * 2 - 1).to(DEV)
    blob, fpar = net._tc_params()
    with profiled() as calls:
        got = ops.pointresnet_tc(x, blob, fpar, f16=True)
    assert [c[0] for c in calls] == ["sonet_pointresnet_tc_forward_f16"]
    assert torch.equal(got, ops.pointresnet_tc(x, blob, fpar, f16=True)), "re-run differs"
    y, bar, flips = _resnet_chain16(net, x)
    err = (got.double() - y).abs()
    u = float((err / bar).max())
    print("\n[fp16] pointresnet cin=%d B=%d P=%d: %.3f bar units, max err / max|y| %.3e, "
          "rounding-boundary fractions act1 %.2e act2 %.2e"
          % (cin, B, P, u, float(err.max() / y.abs().max()), flips[0], flips[1]))
    assert u <= 1.0, "pointresnet: error is %.3g x the chained bar" % u
    assert not torch.equal(got, ops.pointresnet_tc(x, blob, fpar))


@pytest.mark.parametrize("cin,B,P,M", [(3, 2, 300, 16), (6, 3, 1000, 64)])
def test_pointresnet_pool_f16_equals_max_of_plain(cin, B, P, M):
    from sonet_b200 import ops
    net = _resnet(cin, seed=cin + P)
    g = _gen(cin * P)
    x = (torch.rand(B, cin, P, generator=g) * 2 - 1).to(DEV)
    blob, fpar = net._tc_params()
    full = ops.pointresnet_tc(x, blob, fpar, f16=True)
    node = torch.sort(torch.randint(0, M, (B, P), generator=g), dim=1)[0]
    node[node == M // 2] = M // 2 + 1                                   # one empty node
    pos0 = torch.randint(0, P, (B,), generator=g)
    ns, p0 = node.int().to(DEV), pos0.int().to(DEV)
    with profiled() as calls:
        got = ops.pointresnet_tc_pool(x, blob, fpar, ns, p0, M, f16=True)
    assert "sonet_pointresnet_tc_pool_forward_f16" in [c[0] for c in calls]
    want = full.new_full((B, 384, M), float("-inf")).scatter_reduce(
        2, node.to(DEV)[:, None, :].expand(B, 384, P), full, "amax")
    empty = torch.bincount((node + torch.arange(B)[:, None] * M).view(-1), minlength=B * M).view(B, M) == 0
    first = full[torch.arange(B), :, pos0.to(DEV)]
    want = torch.where(empty.to(DEV)[:, None, :], first[:, :, None].expand(B, 384, M), want)
    assert torch.equal(got, want)


# ---- 3 + 4. model level ------------------------------------------------------------------------------
FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "*.npz"))
                  if os.path.basename(p).split("_")[0] in ("classifier", "segmenter", "autoencoder"))
HEAD = {"classifier": "classifier", "segmenter": "segmenter", "autoencoder": "decoder"}
OUT = {"classifier": "score", "segmenter": "score_segmenter", "autoencoder": "predicted_pc"}


def _model(task, opt, st):
    import copy

    from sonet_b200 import autoencoder, classifier, segmenter
    gopt = copy.copy(opt)
    gopt.device, gopt.gpu_id = torch.device(DEV), 0
    mod = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}[task]
    m = mod.Model(gopt)
    m.encoder.load_state_dict(st["encoder"])
    getattr(m, HEAD[task]).load_state_dict(st["head"])
    return m


def _set_input(m, task, inp):
    if task == "segmenter":
        seg = torch.zeros(inp["pc"].shape[0], inp["pc"].shape[2], dtype=torch.int64)
        m.set_input(inp["pc"], inp["sn"], inp["label"], seg, inp["node"], inp["node_knn_I"])
    else:
        m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])


def _forward(m, task, inp):
    _set_input(m, task, inp)
    with profiled() as calls:
        m.test_model()
        torch.cuda.synchronize()
    return [c[0] for c in calls]


def _tc_calls(names):
    return [n for n in names if n.replace("_f16", "") in TC_ENTRIES]


@pytest.mark.parametrize("name", FIXTURES)
def test_golden_models_f16(name):
    task = name.split("_")[0]
    g = golden(name)
    opt, inp, seed = golden_case(g, task)
    m = _model(task, opt, build_states(task, opt, seed))
    with tc_mode(None):
        names = _forward(m, task, inp)
    tc = _tc_calls(names)
    assert tc and not any(n.endswith("_f16") for n in names), tc
    with tc_mode("fp16"):
        names = _forward(m, task, inp)
    tc = _tc_calls(names)
    assert tc and all(n.endswith("_f16") for n in tc), tc
    assert {n.replace("_f16", "") for n in tc} <= set(TC_ENTRIES)
    outs = [("out", getattr(m, OUT[task]), OUT[task])]
    enc = m.encoder
    for n in ("first_pn_out_masked_max", "final_pn_out", "feature"):
        outs.append((n, getattr(enc, n), n))
    if opt.som_k >= 2:
        outs.append(("knn_feature_1", enc.knn_feature_1, "knn_feature_1"))
    worst = 0.0
    for what, t, key in outs:
        ref = torch.from_numpy(g[key]).double()
        got = sampled(g, key, t).double()
        e = float((got - ref).abs().max() / ref.abs().max())
        worst = max(worst, e)
        print("\n[fp16] %s %s: max |err| / max |golden| = %.3e" % (name, what, e))
        assert e <= F16_MODEL_REL, "%s %s: %.3e > %.1e" % (name, what, e, F16_MODEL_REL)
    _WORST["model " + name] = worst
    if task == "classifier":
        ref = torch.from_numpy(g["score"]).double().view(m.score.shape)
        top2 = ref.topk(2, dim=1)[0]
        sure = (top2[:, 0] - top2[:, 1]) > 10 * F16_MODEL_REL * ref.abs().max()
        agree = m.score.cpu().argmax(1) == ref.argmax(1)
        print("[fp16] %s: top-1 agrees on %d of %d clouds, %d with a clear margin"
              % (name, int(agree.sum()), agree.numel(), int(sure.sum())))
        assert bool(agree[sure].all())


# ---- 5. mode flips with CUDA graphs on ---------------------------------------------------------------
def test_cuda_graph_follows_mode_flips():
    g = golden("classifier_b2_n256")
    opt, inp, seed = golden_case(g, "classifier")
    st = build_states("classifier", opt, seed)
    graphed, eager = _model("classifier", opt, st), _model("classifier", opt, st)
    graphed.enable_cuda_graph(True)
    for mm in (graphed, eager):
        _set_input(mm, "classifier", inp)
    got = {}
    for i, mode in enumerate((None, "fp16", "0", None)):
        with tc_mode(mode):
            graphed.test_model()
            eager.test_model()
            torch.cuda.synchronize()
            assert torch.equal(graphed.score, eager.score), "replay %d (SONET_TC=%s)" % (i, mode)
            got[i] = graphed.score.clone()
    assert torch.equal(got[3], got[0])
    assert not torch.equal(got[1], got[0]) and not torch.equal(got[2], got[0])


# ---- 6. train mode ignores the mode ------------------------------------------------------------------
def _train_step(mode):
    from sonet_b200 import classifier, synth
    B, N = 4, 512
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device=DEV)
    opt.device = torch.device(DEV)
    st = build_states("classifier", opt, seed=29)
    inp = synth.synth_inputs(B, N, seed=29)
    with tc_mode(mode):
        m = classifier.Model(opt)
        m.encoder.load_state_dict(st["encoder"])
        m.classifier.load_state_dict(st["head"])
        m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
        torch.manual_seed(0)
        with profiled() as calls:
            m.optimize(epoch=2)
            torch.cuda.synchronize()
    assert not any(c[0].endswith("_f16") for c in calls)
    mods = (m.encoder, m.classifier)
    state = {"%d.%s" % (i, k): v.detach().clone() for i, mm in enumerate(mods)
             for k, v in mm.state_dict().items()}
    grads = {"%d.%s" % (i, k): p.grad.detach().clone() for i, mm in enumerate(mods)
             for k, p in mm.named_parameters() if p.grad is not None}
    return state, grads, opt.lr


def test_train_step_ignores_fp16_mode():
    """No `_f16` entry runs in a training step (asserted in _train_step), and the step under
    SONET_TC=fp16 equals the default's up to the train path's run-to-run spread: one step is not
    bit-reproducible (a few tensors of the first PointResNet's layer 0 differ between two default
    steps in the last bits), so gradients are held to 1e-5 of each tensor's largest value (for a
    bias, of its weight's too: its gradient is a largely cancelling sum over the batch) and
    parameters, after Adam, to 1e-5 of their scale or one Adam step (lr) where a gradient near zero
    changes sign. Every tensor two default steps reproduce bit for bit is counted."""
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    try:
        s0, g0, lr = _train_step(None)
        s1, g1, _ = _train_step("fp16")
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev
    assert g0 and s0.keys() == s1.keys() and g0.keys() == g1.keys()
    same = 0
    for kind, a, b in (("gradient", g0, g1), ("state", s0, s1)):
        for k in a:
            if torch.equal(a[k], b[k]):
                same += 1
                continue
            d = (a[k].double() - b[k].double()).abs()
            tol = 1e-5 * float(a[k].double().abs().max())
            w = k[:-len("bias")] + "weight"
            if kind == "gradient" and k.endswith("bias") and w in a:
                # a bias gradient sums the whole batch's output gradient: largely cancelling (zero
                # analytically in front of a batch-statistics BN), so its scale is its weight's
                tol = max(tol, 1e-5 * float(a[w].double().abs().max()))
            if kind == "state" and a[k].is_floating_point() and not k.endswith(
                    ("running_mean", "running_var")):
                tol = max(tol, 2 * lr)
            assert float(d.max()) <= tol, "%s %s: %.3e > %.3e" % (kind, k, float(d.max()), tol)
    print("\n[fp16] train step: %d of %d tensors bit-identical to the default step"
          % (same, len(g0) + len(s0)))


# ---- 7. range and NaN --------------------------------------------------------------------------------
def test_generic_layer_f16_saturates_beyond_fp16():
    from sonet_b200 import ops
    g = _gen(8)
    B, Cin, P, Cout = 2, 64, 300, 64
    x = torch.randn(B, Cin, P, generator=g).clamp(-3.5, 3.5)
    x[:, 5, :] = 1e6
    x[:, 9, ::3] = -3e38
    x[:, 11, 1::3] = 65520.0                      # rounds to inf without saturation
    W = torch.randn(Cout, Cin, generator=g) * (2.0 / Cin) ** 0.5
    blob, inv = ops.pointwise_tc_pack(W)
    xd = x.to(DEV)
    got = ops.pointwise_layer_tc(xd, blob.to(DEV), inv, None, Cout, False, f16=True)
    assert bool(torch.isfinite(got).all())
    y, m = gemm16(w16(W, inv), inv, r16(xd))
    check(got, y, m, "saturated input")


@pytest.mark.parametrize("relu", [False, True])
def test_generic_layer_f16_nan_as_the_split(relu):
    """A NaN input reaches the same outputs, as the same values, as in the split; every other
    output stays inside the bar."""
    from sonet_b200 import ops
    args, kw, y, m = _layer_case(2, 96, 0, 300, 130, relu, True, 0, seed=9)
    x = args[0].clone()
    x[1, 7, 5::17] = float("nan")
    args = (x,) + args[1:]
    got = ops.pointwise_layer_tc(*args, **kw, f16=True)
    split = ops.pointwise_layer_tc(*args, **kw)
    hit = torch.zeros_like(got, dtype=torch.bool)
    hit[1, :, 5::17] = True
    assert torch.equal(torch.isnan(got), torch.isnan(split))
    assert torch.equal(got[hit].nan_to_num(1.5), split[hit].nan_to_num(1.5))
    h = got[hit]
    print("\n[fp16] NaN input, relu=%s: of %d hit outputs %d NaN, %d -inf, %d zero, %d other"
          % (relu, h.numel(), int(torch.isnan(h).sum()), int(torch.isneginf(h).sum()),
             int((h == 0).sum()), int(torch.isfinite(h).sum() - (h == 0).sum())))
    check(torch.where(hit, y.clamp(min=0) if relu else y, got.double()), y, m, "NaN rows", relu=relu)


def test_report_worst_ratios():
    """Last in the file: the largest err / m of the kernel cases and rel error of the models
    (the numbers F16_C and F16_MODEL_REL are calibrated from)."""
    k = [v for n, v in _WORST.items() if not n.startswith("model ")]
    mo = [v for n, v in _WORST.items() if n.startswith("model ")]
    print("\n[fp16] worst kernel err / m: %s; worst model rel error: %s"
          % (max(k) if k else None, max(mo) if mo else None))
