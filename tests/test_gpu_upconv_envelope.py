"""-m gpu: the auto-encoder's up-convolution decoder (csrc/upconv.cu, csrc/pointwise_tc.cu) at
every route, tile edge and operand range.

A x2 nearest up-sampling followed by a 3x3 convolution is four parity GEMMs over the
low-resolution map (K = 4*Cin, the taps that coincide after up-sampling summed on the host). The
kernels under test are the grouped mode of pointwise_tc_kernel, its parity scatter (in the
epilogue, or in splitk_reduce_kernel when K is split), the split-K partials and their fixed-order
reduce, the im2col-free conv mode, and the prep kernels upconv_im2col (scalar and vec4) and
upconv_hshift.

  1. the route: a host mirror of UpConv.forward's choices (1x1 dense layer, conv mode, im2col
     vec4 / scalar, pick_splits), every combination reached, each launch as the mirror predicts;
  2. a shape sweep in both precision modes, every activation and splits 1 / 2 / all K chunks,
     against fp64 (helpers.tc_reference per parity group, interleaved, or helpers.F16_C for the
     fp16 mode) and against the fp64 convolution of the unfolded weights;
  3. exact oracles: conv mode == im2col mode, the in-kernel scatter == the host interleave, the
     device-scale entry == the host-scale entry, the prep kernels == a torch restatement,
     determinism and cloud independence, all bit for bit;
  4. magnitudes from 2^-14 to 2^14, weight rows over four decades, one parity group 2^-10 of the
     others, saturation beyond fp16's range;
  5. NaN inputs: exactly the 4x4 output block that reads the pixel changes, to 0 under ReLU, -inf
     without an activation and NaN under ELU, whatever the split, operand route or precision.
"""
import contextlib
import math

import pytest
import torch
import torch.nn.functional as F

from helpers import F16_C, TC_F, TC_R, tc_reference

DEV = "cuda:0"
gpu = pytest.mark.gpu
ACTS = (None, "relu", "elu")
GROUPED = "sonet_pointwise_tc_grouped_forward"
_WORST = {}          # family -> largest error seen, in units of its bar


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


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _record(family, u):
    _WORST[family] = max(_WORST.get(family, 0.0), u)


# ---- 1. the route ---------------------------------------------------------------------------------
def mirror(B, Cin, H, W, Cout):
    """What UpConv.forward launches for an eval-mode [B, Cin, H, W] input (layers.py)."""
    from sonet_b200 import ops
    if H == 1 and W == 1:
        kch = (Cin + 63) // 64
        s = ops.pick_splits(kch, ((B + 127) // 128) * ((4 * Cout + 255) // 256))
        return dict(route="dense", splits=s, groups=1, scat_w=0, conv_w=0, prep=None)
    P = H * W
    kch = (4 * Cin + 63) // 64
    s = ops.pick_splits(kch, 4 * ((B * P + 127) // 128) * ((Cout + 255) // 256))
    conv = ops.upconv_conv_mode(Cin, H, W)
    route = "conv" if conv else ("im2col_vec4" if W % 4 == 0 else "im2col_scalar")
    return dict(route=route, splits=s, groups=4, scat_w=W, conv_w=W if conv else 0,
                prep="sonet_upconv_hshift_f32" if conv else "sonet_upconv_im2col_f32")


# (B, Cin, H, W, Cout): each route with pick_splits choosing 1 and more than 1
UPCONV_CASES = [
    (2, 16, 1, 1, 64),         # dense, one K chunk
    (2, 128, 1, 1, 65),        # dense, split 2
    (2, 16, 3, 5, 64),         # im2col scalar, one K chunk
    (2, 32, 5, 7, 65),         # im2col scalar, split 2
    (2, 48, 4, 16, 64),        # im2col vec4 (Cin % 64 != 0), three K chunks
    (2, 32, 2, 32, 130),       # im2col vec4, split 2
    (4, 64, 32, 32, 64),       # conv, 128 items: no split
    (2, 64, 8, 8, 64),         # conv, split 4
    (3, 128, 16, 4, 192),      # conv on a non-square map, split 8
]


def _upconv_id(c):
    return "B%d-C%d-%dx%d-O%d" % c


def test_upconv_cases_reach_every_route():
    """Host-only: the UpConv cases reach every {route} x {split or not} x {activation}."""
    combos = {(mirror(*c)["route"], mirror(*c)["splits"] > 1, a) for c in UPCONV_CASES for a in ACTS}
    want = {(r, s, a) for r in ("dense", "im2col_scalar", "im2col_vec4", "conv")
            for s in (False, True) for a in ACTS}
    assert combos == want, sorted(want - combos)


SETS = (((0,), (1, 2)), ((0, 1), (2,)))        # [parity][tap] -> the 3x3 kernel rows it collects


def fold(w4):
    """[Cout, Cin, 3, 3] -> Wg [4, Cout, 4*Cin] in w4's dtype, the taps summed in UpConv._packed's
    order: Wg[(py, px)][co][(a, c)*Cin + ci]."""
    Cout, Cin = w4.shape[:2]
    Wg = torch.zeros(4, Cout, 4, Cin, dtype=w4.dtype, device=w4.device)
    for py in range(2):
        for px in range(2):
            for a in range(2):
                for c in range(2):
                    acc = 0
                    for dy in SETS[py][a]:
                        for dx in SETS[px][c]:
                            acc = acc + w4[:, :, dy, dx]
                    Wg[py * 2 + px, :, a * 2 + c] = acc
    return Wg.view(4, Cout, 4 * Cin)


def im2col_ref(x):
    """x [B, Cin, H, W] -> [4B, 4Cin, HW]: row (g*B + b, t*Cin + ci) holds x[b, ci] shifted by
    (a-1+py, c-1+px), zero outside (upconv_im2col_kernel's layout)."""
    B, Cin, H, W = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    cols = []
    for g in range(4):
        taps = []
        for t in range(4):
            dy, dx = (t >> 1) - 1 + (g >> 1), (t & 1) - 1 + (g & 1)
            taps.append(xp[:, :, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W])
        cols.append(torch.cat(taps, 1).reshape(B, 4 * Cin, H * W))
    return torch.cat(cols, 0)


def hshift_ref(x):
    """x [B, Cin, H, W] -> [3B, Cin, HW]: x shifted horizontally by -1, 0, +1, zero at row ends."""
    B, Cin, H, W = x.shape
    xp = F.pad(x, (1, 1))
    return torch.cat([xp[..., k:k + W].reshape(B, Cin, H * W) for k in range(3)], 0)


def interleave(flat, B, H, W):
    """[4B, C, HW] (group g = parity (py, px) at rows g*B..) -> [B, C, 4HW] of the 2H x 2W map."""
    C = flat.shape[1]
    out = flat.new_empty(B, C, 2 * H, 2 * W)
    for g in range(4):
        out[:, :, g >> 1::2, g & 1::2] = flat[g * B:(g + 1) * B].reshape(B, C, H, W)
    return out.reshape(B, C, 4 * H * W)


def _nanzero(t):
    return torch.where(torch.isnan(t), torch.zeros_like(t), t)


def same_bits(a, b):
    """Bit-identical, every NaN matched by a NaN (payloads aside)."""
    return (a.shape == b.shape and torch.equal(torch.isnan(a), torch.isnan(b))
            and torch.equal(_nanzero(a).contiguous().view(torch.int32),
                            _nanzero(b).contiguous().view(torch.int32)))


def act_ref(y, act):
    if act == "relu":
        return y.clamp(min=0)
    if act == "elu":
        return torch.where(y > 0, y, torch.expm1(y))
    return y


def units(got, y, bar, act):
    """max |got - act(y)| / bar; ELU (1-Lipschitz, as ReLU) adds its own rounding, 2^-21 |elu|."""
    ref = act_ref(y, act)
    if act == "elu":
        bar = bar + 2.0 ** -21 * ref.abs()
    return float(((got.double() - ref).abs() / bar).max())


def _tc_ref(Wg, inv, xcol, shift, B, H, W):
    """Per parity group, fp64 W x + shift and the tensor-core bar, interleaved into the output map."""
    ys, bars = [], []
    for g in range(4):
        y, m, fl = tc_reference(Wg[g], xcol[g * B:(g + 1) * B], shift, w_scale=1.0 / inv, parts=True)
        ys.append(y)
        bars.append(TC_R * m + TC_F * fl)
    return interleave(torch.cat(ys), B, H, W), interleave(torch.cat(bars), B, H, W)


def r16(x):
    """fp16 round-to-nearest with saturation to +-65504, NaN kept, as fp64."""
    return x.clamp(-65504.0, 65504.0).half().double()


def _f16_ref(Wg, inv, xcol, shift, B, H, W):
    """The fp16 mode: fp64 GEMM of rn16(x) and rn16(s W), / s, + shift; bar F16_C * sum |.|."""
    xs = r16(xcol.double())
    ys, ms = [], []
    for g in range(4):
        w16 = (Wg[g].to(DEV, torch.float32) * (1.0 / inv)).half().double()
        xg = xs[g * B:(g + 1) * B]
        y = torch.einsum("ok,bkp->bop", w16, xg) * inv
        m = torch.einsum("ok,bkp->bop", w16.abs(), xg.abs()) * inv
        if shift is not None:
            y = y + shift.double()[None, :, None]
            m = m + shift.double().abs()[None, :, None]
        ys.append(y)
        ms.append(m)
    return interleave(torch.cat(ys), B, H, W), F16_C * interleave(torch.cat(ms), B, H, W)


def kchunks(Cin):
    return (4 * Cin + 63) // 64


def split_set(Cin):
    """splits 1, 2 and the largest: one K chunk per item."""
    k = kchunks(Cin)
    return sorted({1, k} | ({2} if k % 2 == 0 else set()))


def conv_ok(Cin, H, W):
    return (H * W) % 64 == 0 and Cin % 64 == 0


class Layer:
    """Seeded 3x3 conv weights, their fp32 and fp64 folds and the packed blobs."""

    def __init__(self, Cin, Cout, seed, row_decades=0.0):
        g = _gen(seed)
        w = torch.randn(Cout, Cin, 3, 3, generator=g) * (2.0 / (9 * Cin)) ** 0.5
        if row_decades:
            w = w * torch.logspace(0, row_decades, Cout, dtype=torch.float64).float()[
                torch.randperm(Cout, generator=g)][:, None, None, None]
        self.w = w.float()
        self.bias = (torch.randn(Cout, generator=g) * 0.1).float().to(DEV)
        self.Wg = fold(self.w)                       # fp32, the host's fold
        self.Wg64 = fold(self.w.double())
        self.Cout = Cout
        self.pack()

    def pack(self):
        from sonet_b200 import ops
        blob, self.per, self.inv = ops.pointwise_tc_pack_groups(self.Wg)
        self.blob = blob.to(DEV)

    def run(self, xin, act, splits, f16, scat_w, conv=False):
        from sonet_b200 import ops
        return ops.pointwise_tc_grouped(xin, self.blob, self.per, self.inv, self.bias, self.Cout, act,
                                        groups=4, splits=splits, scat_w=scat_w, conv=conv, f16=f16)


def _acts(B, C, H, W, g, scale=1.0):
    # N(0,1) clipped to +-3.5: at scale 2^14 every value stays inside fp16's range
    return (torch.randn(B, C, H, W, generator=g).clamp(-3.5, 3.5) * scale).float()


@gpu
@pytest.mark.parametrize("act", ACTS, ids=lambda a: str(a))
@pytest.mark.parametrize("case", UPCONV_CASES, ids=_upconv_id)
def test_upconv_route_and_fp64(case, act, monkeypatch):
    """UpConv (BatchNorm folded) launches what the mirror predicts, and lies inside the bar of
    the fp64 convolution of its unfolded weights: the tensor-core bar of the folded fp32 GEMM plus
    the fp32 rounding of the BN fold and of the tap sums, both known exactly."""
    from sonet_b200 import layers
    monkeypatch.delenv("SONET_TC", raising=False)
    monkeypatch.delenv("SONET_UPCONV_IM2COL", raising=False)
    B, Cin, H, W, Cout = case
    torch.manual_seed(sum(case))
    up = layers.UpConv(Cin, Cout, activation=act, normalization="batch")
    with torch.no_grad():
        bn = up.conv.norm
        bn.running_mean.normal_(0, 0.5)
        bn.running_var.uniform_(0.5, 2.0)
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0, 0.3)
        up.conv.conv.bias.normal_(0, 0.1)
    up = up.to(DEV).eval()
    x = _acts(B, Cin, H, W, _gen(sum(case) + 1)).to(DEV)
    want = mirror(*case)
    with torch.no_grad():
        with profiled() as calls:
            got = up(x)
        again = up(x)
    names = [c[0] for c in calls]
    assert names == ([want["prep"]] if want["prep"] else []) + [GROUPED], names
    a = calls[-1][3]
    assert (a[10], a[11], a[12], a[13]) == (want["groups"], want["splits"], want["scat_w"],
                                           want["conv_w"]), (a[10:14], want)
    assert same_bits(got, again), "re-run differs"

    pk = up._packed()
    inv = pk["inv1"] if want["route"] == "dense" else pk["inv4"]
    w32, shift32 = (t.detach() for t in up.conv.folded())
    c = up.conv.conv
    s64 = bn.weight.detach().double() / torch.sqrt(bn.running_var.double() + bn.eps)
    w64 = c.weight.detach().double() * s64[:, None, None, None]
    sh64 = (c.bias.detach().double() - bn.running_mean.double()) * s64 + bn.bias.detach().double()
    Wg32 = fold(w32.view(Cout, Cin, 3, 3))
    dW = (Wg32.double() - fold(w64)).abs()
    xcol = im2col_ref(x).double()
    y, bar = _tc_ref(Wg32, inv, xcol, shift32, B, H, W)
    extra = torch.cat([torch.einsum("ok,bkp->bop", dW[g], xcol[g * B:(g + 1) * B].abs())
                       for g in range(4)])
    bar = bar + interleave(extra, B, H, W) + (shift32.double() - sh64).abs()[None, :, None]
    xu = F.interpolate(x.double(), scale_factor=2, mode="nearest")
    y64 = F.conv2d(xu, w64, sh64, padding=1).reshape(B, Cout, -1)
    u = units(got.reshape(B, Cout, -1), y64, bar, act)
    _record("route", u)
    print("\n[upconv] %s %s %s splits=%d: %.3f bar units" % (_upconv_id(case), act, want["route"],
                                                             want["splits"], u))
    assert u <= 1.0, u


# ---- 2. shape sweep -------------------------------------------------------------------------------
# (B, Cin, H, W, Cout). Maps: 1x1, one pixel high / wide, non-square conv-mode maps, odd maps on the
# scalar im2col, a conv-mode tile straddling clouds (P = 64, B = 3). Cin: the 16-channel padding
# (17, 65: a 16-channel tail), one K chunk (16) and K = 4096 (1024). Cout: every n-tile width and
# the n64 path. B*P below, at and above multiples of 128.
SHAPES = [
    (2, 16, 1, 1, 64),          # 1x1: P = 1, one K chunk; scalar im2col
    (3, 64, 1, 64, 65),         # one pixel high; conv; 192 rows
    (2, 128, 64, 1, 130),       # one pixel wide; conv; n-tile widths 128 + 64
    (2, 17, 2, 32, 192),        # vec4; Cin tail (K 68 -> 80)
    (1, 65, 4, 16, 257),        # vec4; K 260 -> 272, five chunks; n-tile 1 width 64
    (3, 48, 16, 4, 320),        # vec4 at W = 4; three chunks
    (2, 64, 3, 5, 256),         # scalar; 30 rows
    (3, 17, 5, 7, 64),          # scalar; 105 rows
    (3, 64, 8, 8, 65),          # conv; a 128-row tile over clouds 0 and 1
    (1, 1024, 8, 8, 1024),      # conv; K = 4096 (64 chunks); Cout 1024
    (2, 128, 8, 24, 192),       # conv on 8x24
    (2, 64, 32, 32, 65),        # conv on 32x32, 2048 rows
    (1, 48, 3, 43, 64),         # scalar; 129 rows
    (1, 16, 5, 25, 192),        # scalar; 125 rows
]


def _shape_id(c):
    return "B%d-C%d-%dx%d-O%d" % c


def test_shape_sweep_covers_the_edges():
    """Host-only: the sweep reaches the maps, Cin, Cout and row counts it is written for."""
    maps = {(c[2], c[3]) for c in SHAPES}
    assert {(1, 1), (1, 64), (64, 1), (2, 32), (4, 16), (16, 4), (3, 5), (5, 7), (8, 8), (8, 24),
            (32, 32)} <= maps
    assert {16, 17, 48, 64, 65, 128, 1024} <= {c[1] for c in SHAPES}
    assert {64, 65, 130, 192, 256, 257, 320, 1024} <= {c[4] for c in SHAPES}
    assert any(conv_ok(C, H, W) and B == 3 and H * W == 64 for B, C, H, W, _ in SHAPES)
    conv_maps = {(H, W) for B, C, H, W, _ in SHAPES if conv_ok(C, H, W)}
    assert {(1, 64), (64, 1), (8, 24)} <= conv_maps
    routes = {"conv" if conv_ok(C, H, W) else ("vec4" if W % 4 == 0 else "scalar")
              for B, C, H, W, _ in SHAPES}
    assert routes == {"conv", "vec4", "scalar"}
    rows = {B * H * W for B, C, H, W, _ in SHAPES}
    assert {r % 128 for r in rows} >= {0, 1, 125} and min(rows) < 128
    assert kchunks(1024) == 64 and kchunks(16) == 1


def _check_prep(x):
    """upconv_im2col (vec4 for W % 4 == 0, scalar otherwise) and upconv_hshift == restatement."""
    from sonet_b200 import ops
    xcol = ops.upconv_im2col(x)
    assert same_bits(xcol, im2col_ref(x)), "upconv_im2col %s" % (tuple(x.shape),)
    hs = ops.upconv_hshift(x)
    assert same_bits(hs, hshift_ref(x)), "upconv_hshift %s" % (tuple(x.shape),)
    return xcol, hs


def _sweep(B, Cin, H, W, Cout, layer, x, family, acts=ACTS, splits=None, ground_truth=True,
           f16s=(False, True), sat=None):
    """Every activation x split x precision: the result inside its bar; conv mode, the host
    interleave of the unscattered launch and a re-run all bit-identical to it."""
    xcol, hs = _check_prep(x)
    conv = conv_ok(Cin, H, W)
    xr = x if sat is None else x.clamp(-sat, sat)
    xcol64 = im2col_ref(xr).double()
    refs = {False: _tc_ref(layer.Wg, layer.inv, xcol64, layer.bias, B, H, W),
            True: _f16_ref(layer.Wg, layer.inv, im2col_ref(x), layer.bias, B, H, W)}
    if sat is not None:          # hi and lo each saturate: the dropped lo(x) lo(w) product, 2^-11
        lo = (xcol64.abs() - 65504.0).clamp(min=0)
        extra = torch.cat([torch.einsum("ok,bkp->bop", layer.Wg[g].to(DEV, torch.float64).abs(),
                                        lo[g * B:(g + 1) * B]) for g in range(4)])
        refs[False] = (refs[False][0], refs[False][1] + 2.0 ** -11 * interleave(extra, B, H, W))
    gt = None
    if ground_truth:
        y64 = F.conv2d(F.interpolate(xr.double(), scale_factor=2, mode="nearest"),
                       layer.w.to(DEV, torch.float64), layer.bias.double(), padding=1)
        dW = (layer.Wg.double() - layer.Wg64).to(DEV).abs()
        ex = torch.cat([torch.einsum("ok,bkp->bop", dW[g], xcol64[g * B:(g + 1) * B].abs())
                        for g in range(4)])
        gt = (y64.reshape(B, Cout, -1), refs[False][1] + interleave(ex, B, H, W))
    for f16 in f16s:
        y, bar = refs[f16]
        for s in (splits or split_set(Cin)):
            for act in acts:
                what = "%s f16=%s splits=%d act=%s" % (_shape_id((B, Cin, H, W, Cout)), f16, s, act)
                got = layer.run(xcol, act, s, f16, W)
                assert same_bits(layer.run(xcol, act, s, f16, W), got), what + ": re-run differs"
                flat = layer.run(xcol, act, s, f16, 0)
                assert same_bits(interleave(flat, B, H, W), got), what + ": scatter != interleave"
                if conv:
                    assert same_bits(layer.run(hs, act, s, f16, W, conv=True), got), \
                        what + ": conv mode != im2col mode"
                if sat is not None:
                    assert bool(torch.isfinite(got).all()), what + ": not finite"
                u = units(got, y, bar, act)
                _record(family, u)
                assert u <= 1.0, "%s: %.3g x the bar" % (what, u)
                if gt is not None and not f16:
                    u = units(got, gt[0], gt[1], act)
                    _record(family + " (fp64 conv)", u)
                    assert u <= 1.0, "%s: %.3g x the bar of the fp64 convolution" % (what, u)


@gpu
@pytest.mark.parametrize("case", SHAPES, ids=_shape_id)
def test_shape_sweep(case):
    B, Cin, H, W, Cout = case
    layer = Layer(Cin, Cout, seed=sum(case))
    x = _acts(B, Cin, H, W, _gen(sum(case) + 7)).to(DEV)
    _sweep(B, Cin, H, W, Cout, layer, x, "shape")


@gpu
@pytest.mark.parametrize("H,W", [(1, 1), (1, 4), (1, 5), (4, 1), (5, 1), (3, 4), (2, 5), (7, 12)])
def test_prep_kernels_small_maps(H, W):
    """W = 1, H = 1, W = 4 (vec4) and W = 5 (scalar), with signed zeros and infinities carried."""
    g = _gen(H * 31 + W)
    x = _acts(3, 5, H, W, g)
    x.view(-1)[::7] = -0.0
    x.view(-1)[3::11] = float("inf")
    x.view(-1)[5::13] = float("-inf")
    _check_prep(x.to(DEV))


# ---- 3. exact oracles ------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("case", [(3, 64, 8, 8, 65), (2, 48, 5, 7, 130)], ids=_shape_id)
def test_forward_dev_equals_host_scale_entry(case):
    """sonet_pointwise_tc_grouped_forward_dev (device pack, 1 / pre-scale read from scale2[1]) gives
    the host-scale entry's bits, with a NaN pixel in the input."""
    from sonet_b200 import _C, ops, train_ops
    B, Cin, H, W, Cout = case
    layer = Layer(Cin, Cout, seed=3 + sum(case))
    blob_d, per, scale2 = train_ops._pack_groups_device(layer.Wg.to(DEV))
    assert torch.equal(blob_d, layer.blob) and float(scale2[1]) == layer.inv
    x = _acts(B, Cin, H, W, _gen(4)).to(DEV)
    x[B - 1, Cin - 1, H // 2, W // 2] = float("nan")
    P = H * W
    for conv in ([False, True] if conv_ok(Cin, H, W) else [False]):
        xin = ops.upconv_hshift(x) if conv else ops.upconv_im2col(x)
        for s in split_set(Cin):
            for act in ACTS:
                want = layer.run(xin, act, s, False, W, conv=conv)
                out = torch.empty(B, Cout, 4 * P, device=DEV)
                scratch = torch.empty(4 * s * B * Cout * P, device=DEV)
                ops._call("sonet_pointwise_tc_grouped_forward_dev", _C.ptr(xin), xin.shape[1], B, P,
                          _C.ptr(blob_d), per, _C.ptr(scale2[1:]), _C.ptr(layer.bias), Cout,
                          ops.act_code(act), 4, s, W, W if conv else 0, 4 * P, 0, _C.ptr(out),
                          _C.ptr(scratch), ops._stream(x))
                assert same_bits(out, want), (conv, s, act)


@gpu
@pytest.mark.parametrize("f16", [False, True], ids=["split", "fp16"])
@pytest.mark.parametrize("case", [(3, 64, 8, 8, 65), (3, 48, 5, 7, 64)], ids=_shape_id)
def test_cloud_independence(case, f16):
    """With cloud 1 changed, clouds 0 and 2 keep their bits (a 128-row tile spans clouds)."""
    B, Cin, H, W, Cout = case
    layer = Layer(Cin, Cout, seed=5 + sum(case))
    x = _acts(B, Cin, H, W, _gen(6)).to(DEV)
    x2 = x.clone()
    x2[1] = _acts(1, Cin, H, W, _gen(7)).to(DEV)[0] * 3
    from sonet_b200 import ops
    for conv in ([False, True] if conv_ok(Cin, H, W) else [False]):
        prep = ops.upconv_hshift if conv else ops.upconv_im2col
        for s in (1, kchunks(Cin)):
            a = layer.run(prep(x), "relu", s, f16, W, conv=conv)
            b = layer.run(prep(x2), "relu", s, f16, W, conv=conv)
            assert same_bits(a[0], b[0]) and same_bits(a[2], b[2]), (conv, s)
            assert not torch.equal(a[1], b[1])


# ---- 4. magnitudes and saturation --------------------------------------------------------------------
MAG = (2, 64, 8, 8, 130)       # conv-mode map: every check also runs the im2col operand


@gpu
@pytest.mark.parametrize("xscale", [2.0 ** -14, 2.0 ** -8, 1.0, 2.0 ** 8, 2.0 ** 14],
                         ids=["2^-14", "2^-8", "1", "2^8", "2^14"])
def test_input_scale(xscale):
    B, Cin, H, W, Cout = MAG
    layer = Layer(Cin, Cout, seed=40)
    x = _acts(B, Cin, H, W, _gen(41), xscale).to(DEV)
    _sweep(B, Cin, H, W, Cout, layer, x, "magnitude", acts=(None,), splits=(1, kchunks(Cin)))


@gpu
def test_mixed_channel_scales():
    """Per input channel scales from 2^-14 to 2^14 within one map."""
    B, Cin, H, W, Cout = MAG
    layer = Layer(Cin, Cout, seed=42)
    ch = torch.pow(2.0, torch.randint(-14, 15, (Cin,), generator=_gen(43)).float())
    x = (_acts(B, Cin, H, W, _gen(44)) * ch[None, :, None, None]).to(DEV)
    _sweep(B, Cin, H, W, Cout, layer, x, "magnitude", acts=(None, "elu"), splits=(1, kchunks(Cin)))


@gpu
def test_weight_rows_over_four_decades():
    B, Cin, H, W, Cout = MAG
    layer = Layer(Cin, Cout, seed=45, row_decades=4.0)
    x = _acts(B, Cin, H, W, _gen(46)).to(DEV)
    _sweep(B, Cin, H, W, Cout, layer, x, "magnitude", acts=(None, "relu"), splits=(1, kchunks(Cin)))


@gpu
@pytest.mark.parametrize("small", [0, 3])
def test_one_parity_group_far_below_the_others(small):
    """The pre-scale is common to the four groups: a group 2^-10 of the others sits near fp16's
    subnormal floor, and the bar's w_scale floor term must cover it."""
    B, Cin, H, W, Cout = MAG
    layer = Layer(Cin, Cout, seed=47 + small)
    layer.Wg[small] *= 2.0 ** -10
    layer.pack()
    x = _acts(B, Cin, H, W, _gen(48)).to(DEV)
    _sweep(B, Cin, H, W, Cout, layer, x, "magnitude", acts=(None,), splits=(1, kchunks(Cin)),
           ground_truth=False)


@gpu
@pytest.mark.parametrize("case", [MAG, (2, 48, 5, 7, 64)], ids=_shape_id)
def test_saturation_beyond_fp16(case):
    """|x| >= 131008 acts as +-131008 (fp16 mode: |x| >= 65504 as +-65504) and the output stays
    finite: 65520, 131008, 1e6, -3e38 and +-inf."""
    B, Cin, H, W, Cout = case
    layer = Layer(Cin, Cout, seed=50 + Cin)
    x = _acts(B, Cin, H, W, _gen(51))
    x[:, 5] = 1e6
    x[:, 9, ::2] = -3e38
    x[:, 11, 1::2] = 131008.0
    x[:, 13, :, ::3] = 65520.0
    x[0, 20, 1, 1:3] = float("inf")
    x[B - 1, 21, 2, 0:2] = float("-inf")
    _sweep(B, Cin, H, W, Cout, layer, x.to(DEV), "saturation", acts=(None, "relu"),
           splits=(1, kchunks(Cin)), ground_truth=False, sat=131008.0)


# ---- 5. NaN inputs ------------------------------------------------------------------------------------
NAN_VALUE = {None: float("-inf"), "relu": 0.0, "elu": float("nan")}


def nan_pixels(B, Cin, H, W):
    """(cloud, channel, row, column): a corner, an edge and an interior pixel in the first and the
    last cloud."""
    return [(0, 0, 0, 0), (0, Cin - 1, H // 2, W - 1), (0, Cin // 2, H // 2, W // 2),
            (B - 1, Cin - 1, H - 1, W - 1), (B - 1, 0, 0, W // 2), (B - 1, 1, H // 2 - 1, 1)]


def hit_mask(B, Cout, H, W, pixels):
    """The outputs whose receptive field holds a pixel: output rows 2i-1 .. 2i+2 and columns
    2j-1 .. 2j+2 of its cloud (every channel), clipped to the map."""
    hit = torch.zeros(B, Cout, 2 * H, 2 * W, dtype=torch.bool, device=DEV)
    for b, _, i, j in pixels:
        hit[b, :, max(2 * i - 1, 0):2 * i + 3, max(2 * j - 1, 0):2 * j + 3] = True
    return hit.reshape(B, Cout, -1)


@gpu
@pytest.mark.parametrize("act", ACTS, ids=lambda a: str(a))
@pytest.mark.parametrize("case", [(3, 64, 8, 8, 65), (2, 48, 5, 7, 130), (2, 17, 4, 16, 64)],
                         ids=_shape_id)
def test_nan_input(case, act):
    """A NaN pixel changes exactly the 4x4 output block that reads it, to INTEGRATION.md's value
    (0 after ReLU, -inf without an activation, NaN under ELU); everything else keeps the bits of
    the clean run. The same at every split, on both operand routes and in both precision modes."""
    from sonet_b200 import ops
    B, Cin, H, W, Cout = case
    layer = Layer(Cin, Cout, seed=60 + sum(case))
    x = _acts(B, Cin, H, W, _gen(61)).to(DEV)
    xn = x.clone()
    pix = nan_pixels(B, Cin, H, W)
    for b, c, i, j in pix:
        xn[b, c, i, j] = float("nan")
    hit = hit_mask(B, Cout, H, W, pix)
    assert bool(hit.any()) and not bool(hit.all())
    want = NAN_VALUE[act]
    bad = []
    for conv in ([False, True] if conv_ok(Cin, H, W) else [False]):
        prep = ops.upconv_hshift if conv else ops.upconv_im2col
        for f16 in (False, True):
            for s in split_set(Cin):
                clean = layer.run(prep(x), act, s, f16, W, conv=conv)
                got = layer.run(prep(xn), act, s, f16, W, conv=conv)
                what = "conv=%s f16=%s splits=%d" % (conv, f16, s)
                assert same_bits(got[~hit], clean[~hit]), what + ": outputs outside the block changed"
                h = got[hit]
                ok = bool(torch.isnan(h).all()) if math.isnan(want) else bool((h == want).all())
                if not ok:
                    vals = torch.unique(_nanzero(h)).tolist()[:4]
                    bad.append("%s: %d NaN, other values %s" % (what, int(torch.isnan(h).sum()), vals))
    assert not bad, "act=%s: the block is not %s in %s" % (act, want, "; ".join(bad))


@gpu
@pytest.mark.parametrize("act", ACTS, ids=lambda a: str(a))
def test_forward_dev_split_nan_as_unsplit(act):
    """sonet_pointwise_tc_forward_dev (the train-mode dgrad's layer): a split gives the unsplit
    layer's value for a NaN input row, and every other output keeps its clean bits."""
    from sonet_b200 import _C, ops, train_ops
    g = _gen(70)
    B, Cin, P, Cout = 2, 256, 200, 130                             # 4 K chunks
    x = torch.randn(B, Cin, P, generator=g).to(DEV)
    W = (torch.randn(Cout, Cin, generator=g) * (2.0 / Cin) ** 0.5).to(DEV)
    shift = torch.randn(Cout, generator=g).to(DEV)
    blob, scale2 = train_ops._pack_device(W, False)
    xn = x.clone()
    xn[1, 77, 33] = float("nan")
    xn[0, 3, 199] = float("nan")
    hit = torch.zeros(B, Cout, P, dtype=torch.bool, device=DEV)
    hit[1, :, 33] = hit[0, :, 199] = True

    def run(inp, s):
        out = torch.empty(B, Cout, P, device=DEV)
        scratch = torch.empty(s * B * Cout * P, device=DEV)
        ops._call("sonet_pointwise_tc_forward_dev", _C.ptr(inp), Cin, B, P, _C.ptr(blob),
                  _C.ptr(scale2[1:]), None, _C.ptr(shift), Cout, ops.act_code(act), s, _C.ptr(out),
                  _C.ptr(scratch), ops._stream(inp))
        return out
    want = NAN_VALUE[act]
    for s in (1, 2, 4):
        got, clean = run(xn, s), run(x, s)
        assert same_bits(got[~hit], clean[~hit]), s
        h = got[hit]
        assert bool(torch.isnan(h).all()) if math.isnan(want) else bool((h == want).all()), \
            "splits=%d: %s" % (s, torch.unique(_nanzero(h)).tolist()[:4])


@gpu
def test_report_worst_bar_fractions():
    """Last in the file: the largest error per family in units of its bar."""
    print("\n[upconv] worst bar fraction per family: %s"
          % ", ".join("%s %.3f" % kv for kv in sorted(_WORST.items())))
