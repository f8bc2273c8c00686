"""-m gpu: the fp16 hi/lo tensor-core GEMMs (csrc/tc_common.cuh) at every tile remainder,
scheduling depth and operand magnitude, against fp64 with error bars that scale with the result.

Kernels under test: the generic wgmma layer (csrc/pointwise_tc.cu) in its eval, split-K and
device-packed forms, the fused first PointResNet (csrc/pointmlp_tc.cu, plain and per-node pool)
and the wgrad GEMM (csrc/train.cu). Each case checks that it reached the launch and tile
configuration it was written for, that a re-run gives identical bits, and that its result lies
inside the error bar of helpers.tc_reference and within TC_FP32_FACTOR of a strict-fp32 GEMM of
the same operands (helpers.py states the bar and how it was calibrated).
"""
import contextlib

import numpy as np
import pytest
import torch

from helpers import (TC_FP32_FACTOR, assert_in_tc_envelope, assert_rows_close, bar_units,
                     fp32_gemm, row_rel_err, tc_reference)

DEV = "cuda:0"
gpu = pytest.mark.gpu


@contextlib.contextmanager
def profiled():
    """Record every C-ABI call (name, args) issued inside the block."""
    from sonet_b200 import ops
    calls = []
    ops.PROFILE = calls
    try:
        yield calls
    finally:
        ops.PROFILE = None


def names(calls):
    return [c[0] for c in calls]


# ---- tile configuration of the generic layer (mirrors pointwise_tc.cu's Dims / item_width) ------
def pw_config(Cin, Cout, rows, splits=1):
    cin_pad = (Cin + 15) // 16 * 16
    kch = (cin_pad + 63) // 64
    rem = cin_pad - 64 * (kch - 1)                 # channels of the last K chunk: 16, 32, 48, 64
    cpad = (Cout + 63) // 64 * 64
    ntiles = (cpad + 127) // 128
    items = []                                     # (nt, sub, item width) of every out-channel item
    for s in range(ntiles):
        nt, sub = s >> 1, s & 1
        items.append((nt, sub, min(128, min(256, cpad - nt * 256) - sub * 128)))
    row_tiles = (rows + 127) // 128
    return dict(rem=rem, halves=2 if rem > 32 else 1, nks=rem // 16, kch=kch, items=items,
                n_items=row_tiles * ntiles * splits, row_tiles=row_tiles, last_rows=rows - 128 * (row_tiles - 1))


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _acts(B, C, P, g, scale=1.0):
    # N(0,1) clipped to +-3.5: at scale 2^14 every value stays inside fp16's range
    return (torch.randn(B, C, P, generator=g).clamp(-3.5, 3.5) * scale).float()


def _weights(Cout, Cin, g, row_decades=0.0):
    W = torch.randn(Cout, Cin, generator=g) * (2.0 / Cin) ** 0.5
    if row_decades:
        # folded weights whose rows span 10^2 .. 10^(2 + row_decades)
        W = W * torch.logspace(2, 2 + row_decades, Cout, dtype=torch.float64).float()[
            torch.randperm(Cout, generator=g)][:, None]
    return W.float()


def run_generic(B, C0, C1, P, Cout, relu=True, with_shift=True, G=0, xscale=1.0, chscale=None,
                row_decades=0.0, seed=0):
    """One sonet_pointwise_tc_forward launch against fp64 and strict fp32; returns (bar units,
    config, the call's args)."""
    from sonet_b200 import ops
    g = _gen(seed)
    Cin = C0 + C1
    x = _acts(B, Cin, P, g, xscale)
    if chscale is not None:
        x = x * chscale[None, :, None]
    W = _weights(Cout, Cin, g, row_decades)
    shift = torch.randn(Cout, generator=g) * float(W.abs().sum(1).mean()) * 0.1 * xscale \
        if with_shift else None
    add = gidx = gathered = None
    if G:
        add = torch.randn(B, Cout, G, generator=g) * xscale
        gidx = torch.randint(0, G, (B, P), generator=g).int()
        gathered = torch.gather(add, 2, gidx.long()[:, None, :].expand(B, Cout, P)).to(DEV)
    blob, inv = ops.pointwise_tc_pack(W)
    xd = x.to(DEV)
    x0, x1 = xd[:, :C0].contiguous(), (xd[:, C0:].contiguous() if C1 else None)
    args = (x0, blob.to(DEV), inv, None if shift is None else shift.to(DEV), Cout, relu)
    kw = dict(x1=x1, addend=None if add is None else add.to(DEV),
              gidx=None if gidx is None else gidx.to(DEV))
    with profiled() as calls:
        got = ops.pointwise_layer_tc(*args, **kw)
    again = ops.pointwise_layer_tc(*args, **kw)
    assert names(calls) == ["sonet_pointwise_tc_forward"]
    a = calls[0][3]
    assert (a[1], a[3], a[4], a[5], a[9], a[10], a[13]) == (C0, C1, B, P, Cout, int(relu), G)
    assert torch.equal(got, again), "re-run differs"
    y, bar = tc_reference(W, xd, shift, gathered, w_scale=1.0 / inv)
    ref32 = fp32_gemm(W, xd, shift, gathered)
    what = "layer B=%d C=%d+%d P=%d Cout=%d" % (B, C0, C1, P, Cout)
    print("\n[envelope] %s x%.3g: wgmma %.3f, fp32 %.3f bar units" % (
        what, xscale, bar_units(got, y, bar, relu),
        bar_units(ref32.clamp(min=0) if relu else ref32, y, bar, relu)))
    u = assert_in_tc_envelope(got, y, bar, what, relu=relu, fp32=ref32)
    return u, pw_config(Cin, Cout, B * P)


# ---- 1. shape sweep -----------------------------------------------------------------------------
# (B, C0, C1, P, Cout, relu, shift, G). Every K remainder with 1..4 chunks, every item width with
# nt = 0 and nt >= 1, row counts below / at / around multiples of 128 and P < 64, two sources
# split inside and at 16-channel groups, ReLU off, no shift, gathered addends with G = 1 and 7.
SHAPES = [
    (1, 3, 0, 100, 1, True, True, 0),          # rem 16, 1 chunk; Cout 1; rows < 128
    (1, 20, 0, 255, 3, False, True, 0),        # rem 32; 128*2 - 1 rows
    (1, 40, 0, 257, 50, True, False, 0),       # rem 48 (Cin not a multiple of 16); 128*2 + 1 rows
    (3, 64, 0, 43, 64, True, True, 0),         # rem 64; 129 rows, P < 64
    (5, 90, 0, 37, 65, False, True, 0),        # 2 chunks rem 32; P < 64
    (2, 100, 0, 128, 127, True, True, 0),      # 2 chunks rem 48; exactly 2 row tiles
    (1, 130, 0, 383, 129, True, True, 0),      # 3 chunks rem 16; nt 0 widths 128 + 64
    (2, 150, 0, 300, 192, True, False, 0),     # 3 chunks rem 48 (nks 3)
    (1, 176, 0, 513, 257, True, True, 0),      # 3 chunks rem 48; nt 1 width 64
    (2, 208, 0, 200, 320, False, True, 0),     # 4 chunks rem 16; nt 1 width 64
    (1, 224, 0, 640, 385, True, True, 0),      # 4 chunks rem 32; nt 1 widths 128 + 64 (nw 192)
    (3, 256, 0, 100, 448, True, True, 0),      # 4 chunks rem 64; nt 1 nw 192
    (1, 424, 0, 129, 1000, True, True, 0),     # 7 chunks rem 48; nt 3 full, Cout 1000
    (2, 387, 0, 576, 512, True, True, 0),      # the KNN module's first layer (rem 16)
    (2, 1, 64, 130, 96, True, True, 0),        # two sources, C0 = 1
    (1, 31, 33, 300, 200, True, True, 0),      # C0 = 31
    (2, 32, 100, 127, 129, False, True, 0),    # C0 = 32
    (1, 33, 31, 256, 64, True, True, 0),       # C0 = 33
    (3, 63, 130, 65, 257, True, True, 0),      # C0 = 63, rem 16 across the sources
    (2, 65, 60, 333, 385, True, False, 0),     # C0 = 65
    (2, 396, 0, 300, 1024, True, False, 64),   # the segmenter's gathered addend
    (2, 70, 0, 250, 130, True, False, 1),      # G = 1
    (3, 128, 0, 99, 300, False, True, 7),      # G = 7, no ReLU
]


def _shape_id(c):
    return "B%d-C%d+%d-P%d-O%d%s%s%s" % (c[0], c[1], c[2], c[3], c[4], "" if c[5] else "-lin",
                                           "" if c[6] else "-noshift", "-G%d" % c[7] if c[7] else "")


def test_shape_sweep_covers_every_tile_edge():
    """Host-only: the sweep reaches every K remainder at 1..4+ chunks, every item width with nt = 0
    and nt >= 1, partial last row tiles of every kind, and each two-source split point."""
    rems, widths, rows = set(), set(), set()
    for B, C0, C1, P, Cout, relu, sh, G in SHAPES:
        c = pw_config(C0 + C1, Cout, B * P)
        rems.add((c["rem"], min(c["kch"], 4)))
        widths.update((nt >= 1, w) for nt, _, w in c["items"])
        rows.add("below" if B * P < 128 else ("exact" if c["last_rows"] == 128 else
                 ("+1" if c["last_rows"] == 1 else ("-1" if c["last_rows"] == 127 else "ragged"))))
        if P < 64:
            rows.add("P<64")
    assert {r for r, _ in rems} == {16, 32, 48, 64}
    assert {(16, 1), (32, 1), (48, 1), (64, 1), (32, 2), (48, 2), (16, 3), (48, 3), (16, 4)} <= rems
    assert widths == {(False, 64), (False, 128), (True, 64), (True, 128)}
    assert {"below", "exact", "+1", "-1", "ragged", "P<64"} <= rows
    assert {c[1] for c in SHAPES if c[2]} == {1, 31, 32, 33, 63, 65}
    assert {c[7] for c in SHAPES} == {0, 1, 7, 64}
    assert {c[5] for c in SHAPES} == {True, False} and {c[6] for c in SHAPES} == {True, False}
    assert {c[4] for c in SHAPES} >= {1, 3, 50, 64, 65, 127, 129, 192, 257, 320, 385, 448, 1000}


@gpu
@pytest.mark.parametrize("case", SHAPES, ids=_shape_id)
def test_generic_layer_shape_sweep(case):
    B, C0, C1, P, Cout, relu, sh, G = case
    run_generic(B, C0, C1, P, Cout, relu=relu, with_shift=sh, G=G, seed=sum(case[:5]))


# ---- 2. persistent depth --------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("Cin,Cout", [(200, 512), (387, 129)])
def test_generic_layer_persistent_depth(Cin, Cout):
    """At least 3 items per SM: every CTA walks several items, so the weight ring's phases wrap
    across items inside one launch."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cfg = pw_config(Cin, Cout, 1)
    per_tile = len(cfg["items"])
    rows = 128 * (-(-3 * sms // per_tile)) - 37                  # ragged last row tile
    B = 7
    P = -(-rows // B)
    cfg = pw_config(Cin, Cout, B * P)
    assert cfg["n_items"] >= 3 * sms, (cfg["n_items"], sms)
    run_generic(B, Cin, 0, P, Cout, seed=Cin + Cout)


@gpu
def test_generic_layer_row_placement_is_bit_exact():
    """The rows of one cloud give the same bits alone as inside a larger batch (other row tile
    offsets, other CTAs, other persistent iterations)."""
    from sonet_b200 import ops
    g = _gen(11)
    B, Cin, P, Cout = 9, 150, 1000, 385
    x = _acts(B, Cin, P, g).to(DEV)
    W = _weights(Cout, Cin, g)
    shift = torch.randn(Cout, generator=g).to(DEV)
    blob, inv = ops.pointwise_tc_pack(W)
    blob = blob.to(DEV)
    assert pw_config(Cin, Cout, B * P)["n_items"] > torch.cuda.get_device_properties(0).multi_processor_count
    full = ops.pointwise_layer_tc(x, blob, inv, shift, Cout, True)
    for b in (0, 4, 8):
        alone = ops.pointwise_layer_tc(x[b:b + 1].contiguous(), blob, inv, shift, Cout, True)
        assert torch.equal(alone[0], full[b]), b


# ---- 3. magnitude sweep ---------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("xscale", [2.0 ** -14, 2.0 ** -8, 1.0, 2.0 ** 8, 2.0 ** 14],
                         ids=["2^-14", "2^-8", "1", "2^8", "2^14"])
def test_generic_layer_input_scale(xscale):
    run_generic(2, 256, 0, 700, 192, xscale=xscale, seed=5)


@gpu
def test_generic_layer_mixed_channel_scales():
    """Per input channel scales from 2^-14 to 2^14 within one tensor."""
    g = _gen(6)
    ch = torch.pow(2.0, torch.randint(-14, 15, (320,), generator=g).float())
    run_generic(2, 320, 0, 500, 257, chscale=ch, seed=6)


@gpu
@pytest.mark.parametrize("decades", [0.0, 2.0, 4.0])
def test_generic_layer_weight_rows_spread(decades):
    """One power-of-two pre-scale per matrix: rows 10^2..10^6 below the largest one lean on the
    weight-side floor of the bar, and must stay inside it."""
    run_generic(2, 192, 0, 600, 320, row_decades=decades, seed=7)


# ---- 4. beyond the fp16 range ---------------------------------------------------------------------
@gpu
def test_generic_layer_saturates_activations_beyond_fp16():
    """hi and lo each saturate at fp16's 65504, so an activation with |x| >= 2 * 65504 = 131008
    acts as +-131008 (include/sonet_b200.h): the result is finite and equals the layer applied to
    the saturated input. There lo(x) is as large as hi(x), so the dropped lo(x)*lo(w) product
    costs up to 2^-12 of each such term: the bar gains 2^-11 * sum_k |W[o,k]| lo(x_k)."""
    from sonet_b200 import ops
    g = _gen(8)
    B, Cin, P, Cout = 2, 64, 300, 64
    x = _acts(B, Cin, P, g)
    x[:, 5, :] = 1e6
    x[:, 9, ::3] = -3e38
    x[:, 11, 1::3] = 131008.0
    W = _weights(Cout, Cin, g)
    blob, inv = ops.pointwise_tc_pack(W)
    got = ops.pointwise_layer_tc(x.to(DEV), blob.to(DEV), inv, None, Cout, False)
    assert bool(torch.isfinite(got).all())
    xs = x.clamp(-131008.0, 131008.0).to(DEV)
    y, bar = tc_reference(W, xs, w_scale=1.0 / inv)
    lo = (xs.abs() - 65504.0).clamp(min=0)
    bar = bar + 2.0 ** -11 * torch.einsum("ok,bkp->bop", W.to(DEV, torch.float64).abs(), lo.double())
    assert_in_tc_envelope(got, y, bar, "saturated input")


# ---- 5. the fused first PointResNet ---------------------------------------------------------------
def _resnet(cin, seed, scale=1.0):
    """PointResNet(cin) with seeded weights; scale multiplies every conv bias and BN mean / shift,
    so the network is s * f(x / s): its activations all scale with the input."""
    from sonet_b200 import layers, synth
    net = layers.PointResNet(cin, [64, 128, 256, 384], 'relu', 'batch')
    st = synth.synth_state_dict(net, seed=seed)
    for k in st:
        if k.endswith("conv.bias") or k.endswith("norm.running_mean") or k.endswith("norm.bias"):
            st[k] = st[k] * scale
    net.load_state_dict(st)
    return net.eval()


def _resnet_fp64(net, x):
    import torch.nn.functional as F

    def layer(l, t):
        y = F.conv1d(t, l.conv.weight.double(), l.conv.bias.double())
        if l.normalization == 'batch':                               # the last layer is bare
            n = l.norm
            y = (y - n.running_mean.double()[None, :, None]) / torch.sqrt(
                n.running_var.double()[None, :, None] + n.eps) * n.weight.double()[None, :, None] \
                + n.bias.double()[None, :, None]
            y = F.relu(y)
        return y
    x = x.double()
    l0 = layer(net.layers[0], x)
    t = layer(net.layers[2], layer(net.layers[1], l0))
    return layer(net.layers[3], torch.cat((l0, t), 1))


def _tensor_rel(a, ref):
    ref = ref.double().cpu()
    return float((a.double().cpu() - ref).abs().max() / ref.abs().max())


def _resnet_case(cin, B, P, scale, seed):
    from sonet_b200 import ops
    net = _resnet(cin, seed, scale)
    x = _acts(B, cin, P, _gen(seed)) * scale
    want = _resnet_fp64(net, x)
    net = net.to(DEV)
    blob, fpar = net._tc_params()
    xd = x.to(DEV)
    with profiled() as calls:
        got = ops.pointresnet_tc(xd, blob, fpar)
    assert names(calls) == ["sonet_pointresnet_tc_forward"] and calls[0][3][1:4] == (cin, B, P)
    assert torch.equal(ops.pointresnet_tc(xd, blob, fpar), got)
    return net, xd, got, want


@gpu
@pytest.mark.parametrize("cin,B,P", [(1, 2, 77), (2, 1, 129), (3, 3, 1), (4, 2, 255), (5, 1, 1000),
                                     (6, 4, 383)])
def test_pointresnet_tc_every_cin(cin, B, P, monkeypatch):
    net, xd, got, want = _resnet_case(cin, B, P, 1.0, seed=cin * 100 + P)
    monkeypatch.setenv("SONET_TC", "0")
    with torch.no_grad():
        simt = net(xd)
    e, e32 = _tensor_rel(got, want), _tensor_rel(simt, want)
    assert e <= max(TC_FP32_FACTOR * e32, 2e-6), (e, e32)


@gpu
@pytest.mark.parametrize("scale,limit", [(2.0 ** -14, 5e-4), (2.0 ** -8, None), (1.0, None),
                                         (2.0 ** 8, None), (2.0 ** 12, 5e-5)],
                         ids=["2^-14", "2^-8", "1", "2^8", "2^12"])
def test_pointresnet_tc_input_scale(scale, limit, monkeypatch):
    """The whole network scaled by s (inputs, biases, BN shifts): from 2^-8 to 2^8 the error
    relative to the output stays of the order of the fp32 CUDA-core path's. Outside that range
    the kernel's inner activations meet the limits csrc/tc_common.cuh states, and the measured
    error (H100: 1.8e-4 at 2^-14, the 2^-25 subnormal floor; 1.1e-5 at 2^12, activations past
    65504) is pinned with headroom."""
    net, xd, got, want = _resnet_case(6, 2, 1000, scale, seed=21)
    monkeypatch.setenv("SONET_TC", "0")
    with torch.no_grad():
        simt = net(xd)
    e, e32 = _tensor_rel(got, want), _tensor_rel(simt, want)
    print("\n[envelope] pointresnet scale %.3g: wgmma %.2e, fp32 %.2e" % (scale, e, e32))
    if limit is None:
        assert e <= max(TC_FP32_FACTOR * e32, 2e-6), (e, e32)
    else:
        assert e <= limit, (e, e32)


@gpu
@pytest.mark.parametrize("cin,B,P,M", [(1, 2, 300, 16), (2, 1, 129, 5), (4, 3, 77, 64), (5, 2, 1000, 33)])
def test_pointresnet_tc_pool_every_cin(cin, B, P, M):
    """Per-node max of the fused pool kernel == the per-node max of the plain kernel's output, with
    empty nodes taking the feature of the row at pos0."""
    from sonet_b200 import ops
    net, xd, full, _ = _resnet_case(cin, B, P, 1.0, seed=cin + P)
    g = _gen(cin * P)
    node = torch.sort(torch.randint(0, M, (B, P), generator=g), dim=1)[0]
    node[node == M // 2] = M // 2 + 1 if M > 2 else 0          # at least one empty node
    pos0 = torch.randint(0, P, (B,), generator=g)
    blob, fpar = net._tc_params()
    ns, p0 = node.int().to(DEV), pos0.int().to(DEV)
    with profiled() as calls:
        got = ops.pointresnet_tc_pool(xd, blob, fpar, ns, p0, M)
    assert "sonet_pointresnet_tc_pool_forward" in names(calls)
    want = full.new_full((B, 384, M), float("-inf")).scatter_reduce(
        2, node.to(DEV)[:, None, :].expand(B, 384, P), full, "amax")
    empty = torch.bincount((node + torch.arange(B)[:, None] * M).view(-1), minlength=B * M).view(B, M) == 0
    assert bool(empty.any())
    first = full[torch.arange(B), :, pos0.to(DEV)]                 # [B,384]
    want = torch.where(empty.to(DEV)[:, None, :], first[:, :, None].expand(B, 384, M), want)
    assert torch.equal(got, want)


# ---- 6. train-mode GEMMs ----------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("splits", [1, 2, 4])
def test_forward_dev_split_k(splits):
    """sonet_pointwise_tc_forward_dev with the K split over CTAs and the fixed-order reduce."""
    from sonet_b200 import _C, ops, train_ops
    g = _gen(30 + splits)
    B, Cin, P, Cout = 3, 500, 333, 320                           # 8 K chunks, rem 52 -> 64
    x = _acts(B, Cin, P, g).to(DEV)
    W = _weights(Cout, Cin, g).to(DEV)
    shift = torch.randn(Cout, generator=g).to(DEV)
    blob, scale2 = train_ops._pack_device(W, False)
    out = torch.empty(B, Cout, P, device=DEV)
    scratch = torch.empty(splits * B * Cout * P, device=DEV)
    res = []
    for _ in range(2):
        with profiled() as calls:
            ops._call("sonet_pointwise_tc_forward_dev", _C.ptr(x), Cin, B, P, _C.ptr(blob),
                      _C.ptr(scale2[1:]), None, _C.ptr(shift), Cout, 1, splits, _C.ptr(out),
                      _C.ptr(scratch), ops._stream(x))
        assert names(calls) == ["sonet_pointwise_tc_forward_dev"] and calls[0][3][10] == splits
        res.append(out.clone())
    assert pw_config(Cin, Cout, B * P)["kch"] % splits == 0
    assert torch.equal(res[0], res[1])
    y, bar = tc_reference(W, x, shift, w_scale=float(scale2[0]))
    assert_in_tc_envelope(res[0], y, bar, "forward_dev splits=%d" % splits, relu=True,
                          fp32=fp32_gemm(W, x, shift))


def _spread_dy(B, C, P, g, lo=-7.0, sparse_k=0):
    """dy [B,C,P] whose channels span 10^lo .. 1 (log-spaced, shuffled); sparse_k > 0: only k
    points per (b, c) row are non-zero, the pattern index_max's backward produces."""
    dy = torch.randn(B, C, P, generator=g) * torch.logspace(lo, 0, C, dtype=torch.float64).float()[
        torch.randperm(C, generator=g)][None, :, None]
    if sparse_k:
        keep = torch.zeros(B, C, P)
        keep.scatter_(2, torch.randint(0, P, (B, C, sparse_k), generator=g), 1.0)
        dy = dy * keep
    return dy


def _strict_fp32(fn):
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return fn()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


@gpu
@pytest.mark.parametrize("sparse_k", [0, 3])
def test_dgrad_with_gradients_spanning_seven_decades(sparse_k):
    """dx = W^T dy (ConvTC backward) with dy channels from 1e-7 to 1: every row of dx within a
    small factor of strict fp32's per-row error."""
    from sonet_b200 import train_ops
    g = _gen(40 + sparse_k)
    B, Cin, Cout, P = 3, 128, 384, 777
    x = _acts(B, Cin, P, g).to(DEV).requires_grad_(True)
    W = _weights(Cout, Cin, g).to(DEV).requires_grad_(True)
    dy = _spread_dy(B, Cout, P, g, sparse_k=sparse_k).to(DEV)
    y = train_ops.ConvTC.apply(x, W, None)
    with profiled() as calls:
        y.backward(dy)
    assert "sonet_pointwise_tc_forward_dev" in names(calls)
    want = torch.einsum("oi,bop->bip", W.detach().double(), dy.double())
    ref32 = _strict_fp32(lambda: torch.einsum("oi,bop->bip", W.detach(), dy))
    got = x.grad.permute(1, 0, 2)                                  # rows = input channels
    e32 = float(row_rel_err(ref32.permute(1, 0, 2), want.permute(1, 0, 2)).max())
    e = assert_rows_close(got, want.permute(1, 0, 2), "dgrad rows", max(TC_FP32_FACTOR * e32, 1e-5))
    print("\n[envelope] dgrad sparse=%d: wgmma rows %.2e, fp32 rows %.2e" % (sparse_k, e, e32))


WGRAD = [  # (B, Cin, Cout, P, dy decades, sparse points per row)
    (4, 16, 64, 700, -7.0, 0),        # Cin 16
    (3, 40, 128, 513, -7.0, 0),       # Cin 40: not a multiple of 16
    (2, 65, 192, 1000, -7.0, 3),      # Cin 65, the index_max backward pattern
    (64, 387, 512, 9, -7.0, 0),       # the KNN module's first layer
    (1, 128, 64, 100, -5.0, 0),       # B*P = 100 < 64 * splits
    (50, 64, 128, 1, -7.0, 0),        # P = 1
    (8, 384, 384, 576, -7.0, 0),      # the first PointResNet's last layer, batch of 8
]


@gpu
@pytest.mark.parametrize("case", WGRAD, ids=lambda c: "B%d-Cin%d-Cout%d-P%d%s" % (
    c[0], c[1], c[2], c[3], "-sparse" if c[5] else ""))
def test_wgrad_rows_keep_their_own_precision(case):
    """dW = sum_{b,p} dy x^T with dy channels from 10^lo to 1: Adam updates each parameter from its
    own gradient, so every ROW of dW must carry the precision strict fp32 gives it."""
    from sonet_b200 import train_ops
    B, Cin, Cout, P, lo, sk = case
    g = _gen(B + Cin + Cout + P)
    x = _acts(B, Cin, P, g).to(DEV)
    dy = _spread_dy(B, Cout, P, g, lo, sk).to(DEV)
    with profiled() as calls:
        got = train_ops.wgrad_tc(dy, x)
    assert names(calls) == ["sonet_wgrad_tc_f32"]
    splits = calls[0][3][6]
    if B * P < 128:
        assert B * P < 64 * splits                                # a K split with an empty tail
    assert torch.equal(train_ops.wgrad_tc(dy, x), got)
    want = torch.einsum("bop,bip->oi", dy.double(), x.double())
    ref32 = _strict_fp32(lambda: torch.einsum("bop,bip->oi", dy, x))
    e32 = float(row_rel_err(ref32, want).max())
    e = assert_rows_close(got, want, "wgrad rows (splits=%d)" % splits, max(TC_FP32_FACTOR * e32, 1e-5))
    print("\n[envelope] wgrad %s splits=%d: wgmma rows %.2e, fp32 rows %.2e" % (case, splits, e, e32))


# ---- 7. calibration record ----------------------------------------------------------------------------
@gpu
def test_envelope_calibration_cases():
    """The measurement behind TC_R / TC_F (helpers.py): at input scale 2^8 the floor term is
    negligible and max |err| / m is the relative error; at 2^-14 the floor rules and
    max |err| / floor is its coefficient. Strict fp32 must itself sit inside the bar."""
    from helpers import TC_F, TC_R
    from sonet_b200 import ops
    for xscale in (2.0 ** 8, 2.0 ** -14):
        g = _gen(99)
        B, Cin, P, Cout = 4, 1024, 1000, 512
        x = _acts(B, Cin, P, g, xscale).to(DEV)
        W = _weights(Cout, Cin, g)
        blob, inv = ops.pointwise_tc_pack(W)
        got = ops.pointwise_layer_tc(x, blob.to(DEV), inv, None, Cout, False)
        y, m, floor = tc_reference(W, x, w_scale=1.0 / inv, parts=True)
        err = (got.double() - y).abs()
        err32 = (fp32_gemm(W, x).double() - y).abs()
        print("\n[envelope] calibration x*%.3g: max err/m wgmma %.3e fp32 %.3e; max err/floor "
              "wgmma %.3e fp32 %.3e" % (xscale, float((err / m).max()), float((err32 / m).max()),
                                        float((err / floor).max()), float((err32 / floor).max())))
        assert bar_units(got, y, TC_R * m + TC_F * floor) <= 1.0
        assert bar_units(fp32_gemm(W, x), y, TC_R * m + TC_F * floor) <= 1.0
