"""The opt-in fp16 train mode (SONET_TRAIN_TC=fp16): the one-product twins of the train GEMM entries,
every train-layer kind, one optimize() step of each model, a short training run, and the mode's
isolation from the default train path and from eval mode.

Error bars. Against the fp64 GEMM of the rounded, pre-scaled operands,
    y16 = (sum_k rn16sat(s_x x_k) rn16(s_w w_k)) / (s_x s_w),
a twin is within helpers.F16_C * sum_k |x16_k w16_k| / (s_x s_w): the fp32 accumulation inside the
tensor cores and, with a K split, the fp32 partial sums (the bar the eval `_f16` entries are held
to). Against the exact operands it is further within 2^-10 * sum_k |w_k x_k| (each operand rounds to
nearest fp16, 2^-11 relative) plus 2^-24 of the operand sums over the other operand's pre-scale,
which covers operands that fall into fp16's subnormal range (2^-25 absolute in scaled units).

Layers and models are held to a multiple of the error of the reference's default composition
(train_ops.ENABLED = False, cuDNN's TF32 on), which rounds every convolution operand to TF32's 10
mantissa bits as this mode rounds them to fp16's.
"""
import contextlib
import copy
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from helpers import F16_C, build_states, row_rel_err, trained_like_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
gpu = pytest.mark.gpu
TWINS = {"sonet_pointwise_tc_forward_dev_f16": "sonet_pointwise_tc_forward_dev",
         "sonet_pointwise_tc_grouped_forward_dev_f16": "sonet_pointwise_tc_grouped_forward_dev",
         "sonet_wgrad_tc_f16": "sonet_wgrad_tc_f32"}
SUB = 2.0 ** -148
ROUND = 2.0 ** -10             # both operands rounded to nearest fp16: 2 * 2^-11 per product


@contextlib.contextmanager
def train_tc(value):
    prev = os.environ.get("SONET_TRAIN_TC")
    if value is None:
        os.environ.pop("SONET_TRAIN_TC", None)
    else:
        os.environ["SONET_TRAIN_TC"] = value
    try:
        yield
    finally:
        if prev is None:
            os.environ.pop("SONET_TRAIN_TC", None)
        else:
            os.environ["SONET_TRAIN_TC"] = prev


@contextlib.contextmanager
def profiled():
    from sonet_b200 import ops
    calls = []
    ops.PROFILE = calls
    try:
        yield calls
    finally:
        ops.PROFILE = None


def names(calls):
    return [c[0] for c in calls]


# ---- host: the switch and the C-ABI -------------------------------------------------------------
@pytest.mark.parametrize("value,on", [(None, False), ("fp16", True), ("1", False), ("0", False),
                                      ("bf16", False), ("", False), ("FP16", False)])
def test_switch_values(value, on):
    from sonet_b200 import train_ops
    with train_tc(value):
        assert train_ops.train_f16() is on


def _prototypes():
    from sonet_b200 import _C
    return _C.parse_header(open(os.path.join(ROOT, "include", "sonet_b200.h")).read())[0]


def test_twins_declared_with_their_split_signatures():
    protos = _prototypes()
    assert protos["sonet_pointwise_tc_forward_dev_f16"] == protos["sonet_pointwise_tc_forward_dev"]
    assert protos["sonet_wgrad_tc_f16"] == protos["sonet_wgrad_tc_f32"]
    # the grouped twin takes the activations' pre-scale after the inverse weight pre-scale
    g16, g = protos["sonet_pointwise_tc_grouped_forward_dev_f16"], protos[
        "sonet_pointwise_tc_grouped_forward_dev"]
    assert g16[:7] + g16[8:] == g and g16[7] is ctypes.c_void_p


def test_twins_bound_exported_and_not_eval_entries(lib_built):
    from sonet_b200 import _C
    h = ctypes.CDLL(lib_built)
    for n in TWINS:
        assert n in _C.TRAIN_F16_ENTRIES and n not in _C.F16_ENTRIES
        assert hasattr(h, n) and n in _C.EXPORTED_SYMBOLS
    assert sorted(_C.TRAIN_F16_ENTRIES) == sorted(TWINS)


def test_twins_reject_bad_arguments_without_a_device(lib_built):
    """SONET_ERR_BAD_ARG before any CUDA call, as from the split entries."""
    from sonet_b200 import _C
    lib, n, bad = _C.lib(), None, _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    p = ctypes.c_void_p(16)          # never dereferenced: validation fails first
    assert lib.sonet_pointwise_tc_forward_dev_f16(p, 64, 1, 1, p, n, n, n, 64, 0, 1, p, n, n) == bad
    assert "inv_scale" in _C.last_error()
    assert lib.sonet_pointwise_tc_forward_dev_f16(p, 64, 1, 1, p, p, n, n, 64, 7, 1, p, n, n) == bad
    assert "activation code 7" in _C.last_error()
    assert lib.sonet_pointwise_tc_forward_dev_f16(p, 64, 1, 1, p, p, n, n, 64, 0, 2, p, n, n) == bad
    assert "scratch" in _C.last_error()
    assert lib.sonet_pointwise_tc_grouped_forward_dev_f16(p, 64, 1, 1, p, 0, n, n, n, 64, 0, 1, 1, 0,
                                                          0, 0, 0, p, n, n) == bad
    assert "inv_scale" in _C.last_error()
    assert lib.sonet_pointwise_tc_grouped_forward_dev_f16(p, 64, 1, 1, p, 0, p, p, n, 64, 0, 1, 2, 0,
                                                          0, 0, 0, p, n, n) == bad
    assert "scratch" in _C.last_error()
    assert lib.sonet_wgrad_tc_f16(p, p, 1, 63, 16, 1, 1, p, p, p, p, p, n) == bad
    assert "Cout" in _C.last_error()
    assert lib.sonet_wgrad_tc_f16(p, n, 1, 64, 16, 1, 1, p, p, p, p, p, n) == bad
    assert "null" in _C.last_error()


# ---- reference arithmetic ------------------------------------------------------------------------
def pow2(m, cap=126):
    m = float(m)
    if not m > 0 or math.isinf(m):
        return 1.0
    return math.ldexp(1.0, min(9 - math.frexp(m)[1], cap))


def r16(t, s):
    """rn16sat(s * t) in fp64 (s a number or a broadcastable tensor of powers of two)."""
    v = (t.double() * s).clamp(-65504, 65504)
    return v.to(torch.float16).double()


def bars(A, X, s_a, s_x, eq):
    """(y16, bar16, y, bar): the GEMM `eq` of the rounded operands and its accumulation bar, and of
    the exact operands and its bar. A is the weight-side operand (pre-scale s_a), X the activation
    (s_x); each scale a number or a tensor broadcastable to its operand."""
    Sa = torch.ones_like(A, dtype=torch.float64) * s_a
    Sx = torch.ones_like(X, dtype=torch.float64) * s_x
    A16, X16 = r16(A, Sa) / Sa, r16(X, Sx) / Sx            # exact: the scales are powers of two
    y16 = torch.einsum(eq, A16, X16)
    m16 = torch.einsum(eq, A16.abs(), X16.abs())
    A64, X64 = A.double(), X.double()
    y = torch.einsum(eq, A64, X64)
    m = torch.einsum(eq, A64.abs(), X64.abs())
    floor = torch.einsum(eq, A64.abs(), 1.0 / Sx) + torch.einsum(eq, 1.0 / Sa, X64.abs())
    return y16, F16_C * m16, y, ROUND * m + 2.0 ** -24 * floor


WORST = {}


def check(got, y16, bar16, y, bar, what):
    got = got.detach().double()
    sc16 = bar16 + SUB
    u16 = float(((got - y16).abs() / sc16).max())
    u = float(((got - y).abs() / (bar + sc16)).max())
    WORST[what.split()[0]] = max(WORST.get(what.split()[0], 0.0), u16, u)
    assert u16 <= 1.0, "%s: %.3g x the accumulation bar against the rounded operands" % (what, u16)
    assert u <= 1.0, "%s: %.3g x the bar against the exact operands" % (what, u)
    return u16, u


def channel_scales(dy):
    m = dy.abs().amax(dim=(0, 2))
    return torch.tensor([pow2(v) for v in m.tolist()], dtype=torch.float64, device=dy.device)


# ---- 1. the entries at every tile edge and split of the envelope test -----------------------------
def _sweep():
    from test_gpu_train_tc_envelope import SWEEP
    return SWEEP


def _case_id(c):
    return "B%d-Cin%d-Cout%d-P%d" % c


def run_convtc16(B, cin, cout, P, seed, xs=1.0, ws=1.0, dys=1.0):
    """One ConvTC forward + backward under SONET_TRAIN_TC=fp16 against both references."""
    from sonet_b200 import train_ops
    from test_gpu_tc_envelope import _spread_dy
    from test_gpu_train_tc_envelope import wgrad_on_tc, wgrad_plan
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, cin, P, generator=g).clamp(-3.5, 3.5) * xs
    W0 = torch.randn(cout, cin, generator=g) * (2.0 / cin) ** 0.5 * ws
    dy = (_spread_dy(B, cout, P, g) * dys).to(DEV)
    x, W = x0.to(DEV).requires_grad_(True), W0.to(DEV).requires_grad_(True)
    with train_tc("fp16"):
        with profiled() as fc:
            y = train_ops.ConvTC.apply(x, W, None)
    with profiled() as bc:
        y.backward(dy)
    assert names(fc) == ["sonet_pointwise_tc_pack_device", "sonet_absmax_scale_f32",
                         "sonet_pointwise_tc_forward_dev_f16"]
    want = ["sonet_pointwise_tc_pack_device", "sonet_absmax_scale_f32",
            "sonet_pointwise_tc_forward_dev_f16"]
    if wgrad_on_tc(cin, cout):
        want.append("sonet_wgrad_tc_f16")
        assert bc[3][3][6] == wgrad_plan(B, P, cin, cout)[0]        # the split entry's splits
    assert names(bc) == want
    what = "B=%d Cin=%d Cout=%d P=%d" % (B, cin, cout, P)
    xd, Wd = x0.to(DEV), W0.to(DEV)
    s_w, s_x, s_dy = pow2(Wd.abs().max()), pow2(xd.abs().max()), pow2(dy.abs().max())
    check(y, *bars(Wd, xd, s_w, s_x, "nk,bkp->bnp"), "forward " + what)
    check(x.grad, *bars(Wd.t(), dy, s_w, s_dy, "nk,bkp->bnp"), "dgrad " + what)
    if wgrad_on_tc(cin, cout):
        s_c = channel_scales(dy)[None, :, None]
        check(W.grad, *bars(xd, dy, s_x, s_c, "bip,bop->oi"), "wgrad " + what)
    return y.detach(), x.grad, W.grad


@gpu
@pytest.mark.parametrize("case", _sweep(), ids=_case_id)
def test_convtc_f16_shape_sweep(case):
    a = run_convtc16(*case, seed=sum(case))
    b = run_convtc16(*case, seed=sum(case))
    for t, u, n in zip(a, b, ("y", "dx", "dW")):
        assert torch.equal(t, u), "re-run changed %s" % n


@gpu
@pytest.mark.parametrize("splits", [1, 2, 4, 8])
def test_forward_dev_f16_splits(splits):
    """The K-split launch of the forward twin (the up-convolution's dgrad GEMM takes it) against the
    rounded operands; every split gives the unsplit bits up to the fp32 partial sums."""
    from sonet_b200 import _C, ops, train_ops
    B, cin, cout, P = 2, 512, 192, 300
    g = torch.Generator().manual_seed(splits)
    x = torch.randn(B, cin, P, generator=g).to(DEV)
    W = (torch.randn(cout, cin, generator=g) * 0.05).to(DEV)
    blob, scale2 = train_ops._pack_device(W, False)
    s_x = train_ops._absmax_scale(x)
    out = torch.empty(B, cout, P, device=DEV)
    scratch = torch.empty(splits * B * cout * P, device=DEV) if splits > 1 else None
    ops._call("sonet_pointwise_tc_forward_dev_f16", _C.ptr(x), cin, B, P, _C.ptr(blob),
              _C.ptr(scale2[1:] * s_x[1:]), _C.ptr(s_x[:1]), None, cout, 0, splits, _C.ptr(out),
              _C.ptr(scratch), ops._stream(x))
    check(out, *bars(W, x, pow2(W.abs().max()), pow2(x.abs().max()), "nk,bkp->bnp"),
          "split forward splits=%d" % splits)


# exponent range: each operand scaled to max 2^e, subnormals included
EXPONENTS = [-149, -140, -126, -118, -100, -64, 0, 64, 100, 127]


def _to_max(t, e):
    return (t / t.abs().max()).double().mul(2.0 ** e).float()


@gpu
@pytest.mark.parametrize("e", EXPONENTS)
@pytest.mark.parametrize("operand", ["x", "W", "dy"])
def test_f16_exponent_range(operand, e):
    """Operands across the fp32 exponent range: no saturation, no spurious non-finite output,
    within the bars wherever the scaled operands stay above the cap."""
    from sonet_b200 import train_ops
    B, cin, cout, P = 2, 96, 128, 200
    g = torch.Generator().manual_seed(7 + e)
    x0 = torch.randn(B, cin, P, generator=g)
    W0 = torch.randn(cout, cin, generator=g) * 0.1
    dy0 = torch.randn(B, cout, P, generator=g)
    x0, W0, dy0 = (_to_max(t, e) if operand == n else t for t, n in ((x0, "x"), (W0, "W"), (dy0, "dy")))
    x, W, dy = x0.to(DEV).requires_grad_(True), W0.to(DEV).requires_grad_(True), dy0.to(DEV)
    with train_tc("fp16"):
        y = train_ops.ConvTC.apply(x, W, None)
    y.backward(dy)
    xd, Wd = x0.to(DEV), W0.to(DEV)
    s_w, s_x, s_dy = pow2(Wd.abs().max()), pow2(xd.abs().max()), pow2(dy.abs().max())
    refs = [("forward", y, bars(Wd, xd, s_w, s_x, "nk,bkp->bnp")),
            ("dgrad", x.grad, bars(Wd.t(), dy, s_w, s_dy, "nk,bkp->bnp")),
            ("wgrad", W.grad, bars(xd, dy, s_x, channel_scales(dy)[None, :, None], "bip,bop->oi"))]
    for what, got, (y16, b16, yy, b) in refs:
        fmax = float(np.finfo(np.float32).max) / 2
        ok = yy.abs() < fmax
        assert bool(torch.isfinite(got.double())[ok].all()), "%s %s 2^%d: non-finite" % (what, operand, e)
        check(got.double()[ok], y16[ok], b16[ok], yy[ok], b[ok], "range %s %s 2^%d" % (what, operand, e))


@gpu
@pytest.mark.parametrize("where,val", [("x", math.inf), ("x", -math.inf), ("x", math.nan),
                                       ("dy", math.inf), ("dy", -math.inf), ("dy", math.nan)])
def test_f16_nonfinite_as_split(where, val):
    """One +-inf or NaN in x or dy: the fp16 twins give non-finite results wherever the split
    entries do, and the forward keeps the split's saturation rule (an infinite x stays finite)."""
    from sonet_b200 import train_ops
    B, cin, cout, P = 2, 64, 128, 300
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(B, cin, P, generator=g)
    W0 = torch.randn(cout, cin, generator=g) * 0.1
    dy0 = torch.randn(B, cout, P, generator=g)
    (x0 if where == "x" else dy0)[1, 5, 17] = val
    outs = {}
    for mode in (None, "fp16"):
        x, W = x0.to(DEV).requires_grad_(True), W0.to(DEV).requires_grad_(True)
        with train_tc(mode):
            y = train_ops.ConvTC.apply(x, W, None)
        y.backward(dy0.to(DEV))
        outs[mode] = (y.detach(), x.grad, W.grad)
    for n, a, b in zip(("y", "dx", "dW"), outs[None], outs["fp16"]):
        nf_split, nf16 = ~torch.isfinite(a), ~torch.isfinite(b)
        assert bool(nf16[nf_split].all()), "%s: finite in fp16 mode where the split is not" % n
        assert torch.equal(nf_split, nf16), "%s: non-finite pattern differs (%d vs %d)" % (
            n, int(nf_split.sum()), int(nf16.sum()))


# ---- 1b. the grouped twin: UpConvTC's forward at every route, tile edge and K split --------------
# (B, Cin, H, W, Cout): the conv route (Cin % 64 == 0, H*W % 64 == 0) and both im2col routes, rows
# below, at and past the 128-row tile, Cout tails of the 64-column tiles
GROUPED_CASES = [
    (2, 64, 8, 8, 64),         # conv: 2 row tiles per group, 4 K chunks
    (3, 128, 16, 4, 192),      # conv on a non-square map: 8 K chunks, Cout 192 (n-tile of 64)
    (1, 64, 32, 32, 130),      # conv, 8 row tiles per group, Cout tail of 2
    (2, 48, 4, 16, 64),        # im2col vec4, 3 K chunks
    (2, 32, 5, 7, 65),         # im2col scalar: 70 rows, below one tile; Cout tail of 1
    (1, 16, 3, 5, 64),         # im2col scalar, one K chunk
    (3, 32, 9, 5, 96),         # im2col scalar: 135 rows, one past a tile
]


def _grouped_splits(Cin):
    kch = (4 * Cin + 63) // 64
    return sorted({1, kch} | ({2} if kch % 2 == 0 else set()))


def upconv_ref(Wg, x, s_w, s_x):
    """Per parity group g: bars() of Wg[g] against the 2x2 neighbourhoods of x (im2col), as the
    parity planes [4][B, Cout, H*W]."""
    from test_gpu_upconv_envelope import im2col_ref
    B = x.shape[0]
    cols = im2col_ref(x)
    return [bars(Wg[g], cols[g * B:(g + 1) * B], s_w, s_x, "nk,bkp->bnp") for g in range(4)]


def parity_planes(z, H, W):
    """z [B, Cout, 2H, 2W] (or [B, Cout, 4HW]) -> [4][B, Cout, H*W], plane g = (py, px)."""
    B, Cout = z.shape[:2]
    v = z.reshape(B, Cout, H, 2, W, 2)
    return [v[:, :, :, g >> 1, :, g & 1].reshape(B, Cout, H * W) for g in range(4)]


def run_grouped16(B, Cin, H, W, Cout, splits, x=None, seed=0):
    """sonet_pointwise_tc_grouped_forward_dev_f16 called as UpConvTC.forward calls it, at `splits`."""
    from sonet_b200 import _C, ops, train_ops
    g = torch.Generator().manual_seed(seed)
    if x is None:
        x = torch.randn(B, Cin, H, W, generator=g).to(DEV)
    W4 = (torch.randn(Cout, Cin, 3, 3, generator=g) * (1.0 / (9 * Cin)) ** 0.5).to(DEV)
    P = H * W
    Wg = torch.empty(4, Cout, 4 * Cin, device=DEV)
    train_ops._fold(W4, Cout, Cin, False, Wg)
    blob, per, scale2 = train_ops._pack_groups_device(Wg)
    conv = ops.upconv_conv_mode(Cin, H, W)
    xin = ops.upconv_hshift(x) if conv else ops.upconv_im2col(x)
    inv, act = train_ops._forward_scales(scale2, x)
    z = torch.empty(B, Cout, 4 * P, device=DEV)
    scratch = torch.empty(4 * splits * B * Cout * P, device=DEV) if splits > 1 else None
    ops._call("sonet_pointwise_tc_grouped_forward_dev_f16", _C.ptr(xin), xin.shape[1], B, P,
              _C.ptr(blob), per, _C.ptr(inv), _C.ptr(act), None, Cout, ops.ACT_NONE, 4, splits, W,
              W if conv else 0, 4 * P, 0, _C.ptr(z), _C.ptr(scratch), ops._stream(x))
    return z, Wg, x, conv


@gpu
@pytest.mark.parametrize("case", GROUPED_CASES, ids=lambda c: "B%d-C%d-%dx%d-O%d" % c)
def test_grouped_f16_routes_and_splits(case):
    """Every route, K split (1, 2, every chunk its own split) and tile edge against the rounded and
    the exact operands; each split's run repeated bit for bit."""
    from sonet_b200 import ops
    B, Cin, H, W, Cout = case
    routes = set()
    for splits in _grouped_splits(Cin):
        z, Wg, x, conv = run_grouped16(*case, splits, seed=sum(case))
        again = run_grouped16(*case, splits, seed=sum(case))[0]
        assert torch.equal(z, again), "re-run changed the output (splits=%d)" % splits
        routes.add(conv)
        refs = upconv_ref(Wg, x, pow2(Wg.abs().max()), pow2(x.abs().max()))
        for gi, (got, ref) in enumerate(zip(parity_planes(z, H, W), refs)):
            check(got, *ref, "grouped %s splits=%d parity %d" % (case, splits, gi))
    assert routes == {ops.upconv_conv_mode(Cin, H, W)}


def test_grouped_cases_reach_every_route():
    """Host-only: the cases reach the conv route and both im2col routes, split and unsplit, and
    rows below, at the edge of and past a 128-row tile."""
    from sonet_b200 import ops
    routes = {("conv" if ops.upconv_conv_mode(c[1], c[2], c[3]) else
               "vec4" if c[3] % 4 == 0 else "scalar", len(_grouped_splits(c[1])) > 1)
              for c in GROUPED_CASES}
    assert {r for r, _ in routes} == {"conv", "vec4", "scalar"}
    assert {s for _, s in routes} == {True, False}
    rows = {c[0] * c[2] * c[3] for c in GROUPED_CASES}
    assert min(rows) < 128 and 128 in rows and any(r % 128 and r > 128 for r in rows)


UPCONV_RANGE = (1, 64, 8, 8, 64)


@gpu
@pytest.mark.parametrize("e", EXPONENTS)
@pytest.mark.parametrize("route", ["conv", "im2col"])
def test_upconv_f16_exponent_range(route, e):
    """UpConvTC's forward with max|x| = 2^e: the activation pre-scale keeps every magnitude off
    fp16's saturation, within the bars wherever the output is below FLT_MAX / 2."""
    from sonet_b200 import train_ops
    B, Cin, H, W, Cout = UPCONV_RANGE if route == "conv" else (1, 32, 5, 7, 64)
    g = torch.Generator().manual_seed(11 + e)
    x = _to_max(torch.randn(B, Cin, H, W, generator=g), e).to(DEV)
    W4 = (torch.randn(Cout, Cin, 3, 3, generator=g) * 0.05).to(DEV)
    with train_tc("fp16"), profiled() as calls:
        z = train_ops.UpConvTC.apply(x, W4, None)
    assert "sonet_pointwise_tc_grouped_forward_dev_f16" in names(calls)
    Wg = torch.empty(4, Cout, 4 * Cin, device=DEV)
    train_ops._fold(W4, Cout, Cin, False, Wg)
    refs = upconv_ref(Wg, x, pow2(Wg.abs().max()), pow2(x.abs().max()))
    fmax = float(np.finfo(np.float32).max) / 2
    for gi, (got, (y16, b16, yy, b)) in enumerate(zip(parity_planes(z, H, W), refs)):
        ok = yy.abs() < fmax
        assert bool(torch.isfinite(got.double())[ok].all()), "parity %d at 2^%d: non-finite" % (gi, e)
        check(got.double()[ok], y16[ok], b16[ok], yy[ok], b[ok],
              "upconv-range %s 2^%d parity %d" % (route, e, gi))


@gpu
@pytest.mark.parametrize("where,val", [("x", math.inf), ("x", -math.inf), ("x", math.nan),
                                       ("dz", math.inf), ("dz", math.nan)])
def test_upconv_f16_nonfinite_as_split(where, val):
    """One +-inf or NaN pixel in UpConvTC's x or dz: z, dx and dW are non-finite exactly where the
    split entries make them so (an infinite x saturates in both forwards)."""
    from sonet_b200 import train_ops
    B, Cin, H, W, Cout = 2, 64, 32, 32, 64
    g = torch.Generator().manual_seed(17)
    x0 = torch.randn(B, Cin, H, W, generator=g)
    W0 = torch.randn(Cout, Cin, 3, 3, generator=g) * 0.05
    dz0 = torch.randn(B, Cout, 2 * H, 2 * W, generator=g)
    (x0 if where == "x" else dz0)[1, 3, 7, 9] = val
    outs = {}
    for mode in (None, "fp16"):
        x, Wt = x0.to(DEV).requires_grad_(True), W0.to(DEV).requires_grad_(True)
        with train_tc(mode):
            z = train_ops.UpConvTC.apply(x, Wt, None)
        z.backward(dz0.to(DEV))
        outs[mode] = (z.detach(), x.grad, Wt.grad)
    for n, a, b in zip(("z", "dx", "dW"), outs[None], outs["fp16"]):
        assert torch.equal(~torch.isfinite(a), ~torch.isfinite(b)), "%s: non-finite pattern differs" % n
    if where == "x" and math.isinf(val):
        assert bool(torch.isfinite(outs["fp16"][0]).all())


# ---- 2. every train-layer kind against fp64 -------------------------------------------------------
# The fp16 mode's error relative to each tensor's largest value may be LAYER_RATIO x the TF32
# composition's plus
# LAYER_FLOOR. cuDNN does not round every convolution of that composition to TF32 (the 3x3 and the
# 4-D 1x1 convolutions came out within 2e-5 of fp64 with the flag on, torch 2.11 on one H100 80GB
# HBM3 at 700 W), so the floor stands for fp16's own rounding (the run prints both errors).
LAYER_RATIO = 4.0
LAYER_FLOOR = 1e-2
# A composition error below NO_TF32 means cuDNN did not round that tensor's convolutions to TF32
# (it kept the 4-D 1x1 layers, the 3x3 and the up-convolutions in fp32 with the flag on, torch 2.11).
# There is then no TF32 error to scale, and the bars are about 2x the largest errors of the fp16
# mode measured over three runs on one H100 80GB HBM3 (700 W), which vary from run to run: dx up to
# 0.17 of max|dx| (the 4-D 1x1 layer, where the sum over the output channels cancels to a small
# fraction of its terms), every other tensor up to 6.6e-2. Where the composition did run TF32 (the
# Conv1d layers) the two errors were equal.
NO_TF32 = 1e-4
NO_TF32_DX = 0.35
NO_TF32_REST = 0.15


def _layer_cases():
    from sonet_b200 import layers
    from test_gpu_train_parity import _layer_cases as base
    cases = dict(base())
    g = torch.Generator().manual_seed(13)
    r = lambda *s: torch.randn(*s, generator=g)
    for act in ("elu", None):
        cases["equivariant_64_128_%s" % act] = (
            lambda act=act: layers.EquivariantLayer(64, 128, act, 'batch'), lambda: (r(8, 64, 1000),))
    cases["upconv_32x32"] = (lambda: layers.UpConv(64, 64, activation='relu', normalization='batch'),
                             lambda: (r(2, 64, 32, 32),))
    cases["upconv_32x32_elu"] = (lambda: layers.UpConv(32, 64, activation='elu',
                                                       normalization='batch'),
                                 lambda: (r(2, 32, 32, 48),))
    return cases


LAYER_CASES = ["equivariant_6_64_thin", "equivariant_64_128_wgmma", "equivariant_64_128_200rows",
               "equivariant_64_128_elu", "equivariant_64_128_None", "myconv2d_1x1_knn",
               "convtopc_128_3", "upconv_3x3", "upconv_32x32", "upconv_32x32_elu", "pointresnet",
               "knn_module"]


@gpu
@pytest.mark.parametrize("case", LAYER_CASES)
def test_train_layer_f16_vs_fp64(case):
    from test_gpu_train_parity import (_analytically_zero, _first, _layer_run, _rows,
                                       precision_flags, train_kernels)
    make, inputs = _layer_cases()[case]
    torch.manual_seed(0)
    mod = make()
    mod.load_state_dict(trained_like_state_dict(mod, seed=len(case)))
    inp = inputs()
    with torch.no_grad():
        y_shape = _first(copy.deepcopy(mod).to(DEV).train()(*[a.to(DEV) if torch.is_tensor(a) else a
                                                              for a in inp])).shape
    w = torch.randn(y_shape, generator=torch.Generator().manual_seed(5)).to(DEV)
    with precision_flags(cudnn_tf32=False), train_kernels(True), train_tc("fp16"), profiled() as calls:
        got = _layer_run(mod, inp, torch.float32, w)
    with precision_flags(cudnn_tf32=True), train_kernels(False):
        tf32 = _layer_run(mod, inp, torch.float32, w)
    ref = _layer_run(mod, inp, torch.float64, w)
    gemm = [n for n in names(calls) if n.startswith(("sonet_pointwise_tc_forward_dev",
                                                     "sonet_pointwise_tc_grouped_forward_dev",
                                                     "sonet_wgrad_tc"))]
    assert all(n in TWINS for n in gemm), gemm
    worst = {}
    for n, r64 in ref.items():
        if _analytically_zero(ref, n):
            assert float(got[n].abs().max()) < 1e-3 * float(ref[n[:-4] + "weight"].abs().max()), n
            continue
        # relative to each tensor's largest value: a row (channel) 2^-10 .. 2^-24 below it keeps
        # fewer of fp16's bits under the tensor's one pre-scale
        e = float(row_rel_err(got[n].reshape(1, -1), r64.reshape(1, -1)))
        et = float(row_rel_err(tf32[n].reshape(1, -1), r64.reshape(1, -1)))
        worst[n] = (e, et)
        # where cuDNN ran the composition in full fp32 there is no TF32 error to scale
        lim = LAYER_RATIO * et + LAYER_FLOOR
        if et < NO_TF32:
            lim = max(lim, NO_TF32_DX if n == "dx" else NO_TF32_REST)
        assert e <= lim, "%s %s: error %.3e, TF32 composition %.3e" % (case, n, e, et)
    print("\n[train-fp16-layer] %s (%d fp16 GEMMs): " % (case, len(gemm)) + ", ".join(
        "%s %.2e (tf32 %.2e, ratio %.2f)" % (n, a, b, a / b if b else float("inf"))
        for n, (a, b) in worst.items()))


# ---- 3. one optimize() of each model -------------------------------------------------------------
# The loss and the whole gradient (every tensor concatenated) may be MODEL_RATIO x the TF32
# composition's relative distance plus MODEL_FLOOR, fp16's own rounding through one step: measured
# on one H100 80GB HBM3 (700 W), the classifier's loss moved 6.4e-3 against 8.5e-4 with TF32.
MODEL_RATIO = 2.0
MODEL_FLOOR = 2e-2
SHAPES = {"classifier": (4, 512), "segmenter": (4, 256), "autoencoder": (4, 512)}


def _model_step(task, enabled, tf32, mode, seed=41):
    """One optimize() step: (loss, {param: grad})."""
    from sonet_b200 import autoencoder, classifier, segmenter, synth
    from test_gpu_train_parity import precision_flags, train_kernels
    B, N = SHAPES[task]
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, device=DEV)
    opt.device = torch.device(DEV)
    st = build_states(task, opt, seed=seed)
    inp = synth.synth_inputs(B, N, seed=seed)
    mod = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}[task]
    with precision_flags(tf32), train_kernels(enabled), train_tc(mode):
        m = mod.Model(opt)
        m.encoder.load_state_dict(st["encoder"])
        head = {"classifier": "classifier", "segmenter": "segmenter", "autoencoder": "decoder"}[task]
        getattr(m, head).load_state_dict(st["head"])
        args = [inp["pc"], inp["sn"], inp["label"]]
        if task == "segmenter":
            args.append(torch.from_numpy(np.random.RandomState(seed).randint(0, 50, size=(B, N))))
        m.set_input(*args, inp["node"], inp["node_knn_I"])
        torch.manual_seed(0)
        m.optimize(epoch=2)
        torch.cuda.synchronize()
    grads = {"%s.%s" % (h, k): p.grad.detach().double().clone() for h in ("encoder", head)
             for k, p in getattr(m, h).named_parameters() if p.grad is not None}
    loss = m.loss_segmenter if task == "segmenter" else m.loss
    return float(loss), grads


def _rel(a, b):
    d = float((a - b).norm())
    n = float(b.norm())
    return d / n if n > 0 else d


@gpu
@pytest.mark.parametrize("task", ["classifier", "segmenter", "autoencoder"])
def test_model_step_f16(task):
    """The loss and every gradient (relative L2) of one optimize() under the fp16 mode are within
    MODEL_RATIO x the TF32 composition's distance from the strict reference plus MODEL_FLOOR. The
    reference is the default train path with strict fp32 flags, which the parity tests hold within
    1e-4 of fp64 (test_gpu_train_parity.py): both distances measured here are of order 1e-3."""
    l_ref, g_ref = _model_step(task, True, False, None)
    l16, g16 = _model_step(task, True, False, "fp16")
    lt, gt = _model_step(task, False, True, None)
    assert g16.keys() == g_ref.keys() == gt.keys()
    dl16, dlt = abs(l16 - l_ref) / abs(l_ref), abs(lt - l_ref) / abs(l_ref)
    assert dl16 <= MODEL_RATIO * dlt + MODEL_FLOOR, "loss: %.3e vs TF32 %.3e" % (dl16, dlt)
    cat = lambda g: torch.cat([g[k].reshape(-1) for k in sorted(g)])
    a, b = _rel(cat(g16), cat(g_ref)), _rel(cat(gt), cat(g_ref))
    per = sorted(((_rel(g16[k], g_ref[k]), k, _rel(gt[k], g_ref[k])) for k in g_ref
                  if float(g_ref[k].norm()) > 0), reverse=True)
    print("\n[train-fp16-model] %s: loss %.2e (tf32 %.2e); gradient %.2e (tf32 %.2e); worst tensor "
          "%s %.2e (tf32 %.2e)" % (task, dl16, dlt, a, b, per[0][1], per[0][0], per[0][2]))
    assert a <= MODEL_RATIO * b + MODEL_FLOOR, "%s gradient: %.3e vs TF32 %.3e" % (task, a, b)


# ---- 4. a short training run ---------------------------------------------------------------------
def _shapes_dataset(n, N, M, seed):
    """Four classes of clouds in [-1,1]^3 a classifier learns in a few steps: a cube, a flat box,
    a rod and a sphere's surface, each randomly rotated about z."""
    rs = np.random.RandomState(seed)
    label = np.arange(n) % 4
    rs.shuffle(label)
    pc = rs.uniform(-1, 1, size=(n, 3, N))
    pc[label == 1, 2] *= 0.1
    pc[label == 2, :2] *= 0.1
    s = pc[label == 3]
    pc[label == 3] = s / np.linalg.norm(s, axis=1, keepdims=True)
    t = rs.uniform(0, 2 * np.pi, n)
    c, sn_ = np.cos(t)[:, None], np.sin(t)[:, None]
    x, y = pc[:, 0].copy(), pc[:, 1].copy()
    pc[:, 0], pc[:, 1] = c * x - sn_ * y, sn_ * x + c * y
    pc = pc.astype(np.float32)
    sn = rs.normal(size=pc.shape).astype(np.float32)
    sn /= np.linalg.norm(sn, axis=1, keepdims=True)
    node = np.stack([pc[b][:, rs.permutation(N)[:M]] for b in range(n)]).astype(np.float32)
    d = ((node[:, :, :, None].astype(np.float64) - node[:, :, None, :]) ** 2).sum(axis=1)
    knn = np.argsort(d, axis=2, kind="stable")[:, :, :9].astype(np.int64)
    return [torch.from_numpy(a) for a in (pc, sn, label.astype(np.int64), node, knn)]


TRAIN_STEPS = 80
LOSS_TOL = 0.1             # |final loss (fp16) - final loss (default)|, averaged over the last steps
ACC_TOL = 4 / 64           # held-out accuracy: at most 4 of the 64 test clouds below the default's


def _train(mode):
    from sonet_b200 import classifier, synth
    B, N, M = 16, 256, 64
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device=DEV, node_num=M,
                         classes=4)
    opt.device = torch.device(DEV)
    train = _shapes_dataset(B * 8, N, M, 0)
    test = _shapes_dataset(64, N, M, 1)
    torch.manual_seed(0)
    with train_tc(mode):
        m = classifier.Model(opt)
        losses = []
        for step in range(TRAIN_STEPS):
            i = (step % 8) * B
            pc, sn, label, node, knn = (t[i:i + B] for t in train)
            m.set_input(pc, sn, label, node, knn)
            m.optimize(epoch=0)
            losses.append(float(m.loss))
    m.encoder.eval()
    m.classifier.eval()
    correct = 0
    for i in range(0, 64, B):
        m.set_input(*(t[i:i + B] for t in test))
        m.test_model()
        correct += int((m.score.argmax(1).cpu() == test[2][i:i + B]).sum())
    return losses, correct / 64


@gpu
def test_short_training_run_matches_default():
    l0, a0 = _train(None)
    l16, a16 = _train("fp16")
    f0, f16 = float(np.mean(l0[-5:])), float(np.mean(l16[-5:]))
    print("\n[train-fp16-run] %d Adam steps: held-out accuracy %.3f (default) %.3f (fp16); "
          "final loss %.4f / %.4f" % (TRAIN_STEPS, a0, a16, f0, f16))
    assert a0 >= 0.75, "the default run does not learn the task (%.3f)" % a0
    assert a16 >= a0 - ACC_TOL
    assert abs(f16 - f0) <= LOSS_TOL


# ---- 5. isolation --------------------------------------------------------------------------------
@gpu
def test_other_values_run_the_default_bits():
    """Unset and any value but fp16 give the default ConvTC / UpConvTC bits and calls."""
    from sonet_b200 import train_ops
    g = torch.Generator().manual_seed(2)
    x0, W0 = torch.randn(2, 64, 500, generator=g), torch.randn(128, 64, generator=g) * 0.1
    u0, V0 = torch.randn(1, 64, 32, 32, generator=g), torch.randn(64, 64, 3, 3, generator=g) * 0.05
    out = {}
    for mode in (None, "1", "bf16", "fp16"):
        x, W = x0.to(DEV).requires_grad_(True), W0.to(DEV).requires_grad_(True)
        u, V = u0.to(DEV).requires_grad_(True), V0.to(DEV).requires_grad_(True)
        with train_tc(mode), profiled() as calls:
            y = train_ops.ConvTC.apply(x, W, None)
            z = train_ops.UpConvTC.apply(u, V, None)
            (y.square().sum() + z.square().sum()).backward()
        out[mode] = ([y.detach(), x.grad, W.grad, z.detach(), u.grad, V.grad], names(calls))
    for mode in ("1", "bf16"):
        assert out[mode][1] == out[None][1]
        for a, b in zip(out[mode][0], out[None][0]):
            assert torch.equal(a, b)
    assert not any(n.endswith("_f16") for n in out[None][1])
    assert {n for n in out["fp16"][1] if n.endswith("_f16")} == set(TWINS)
    assert not any(torch.equal(a, b) for a, b in zip(out["fp16"][0], out[None][0]))


@gpu
@pytest.mark.parametrize("task", ["classifier", "autoencoder"])
def test_eval_forward_ignores_the_mode(task):
    from sonet_b200 import autoencoder, classifier, synth
    B, N = 2, 512
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, device=DEV)
    opt.device = torch.device(DEV)
    st = build_states(task, opt, seed=5)
    inp = synth.synth_inputs(B, N, seed=5)
    m = {"classifier": classifier, "autoencoder": autoencoder}[task].Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    head = "classifier" if task == "classifier" else "decoder"
    getattr(m, head).load_state_dict(st["head"])
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    outs = []
    for mode in (None, "fp16"):
        with train_tc(mode), profiled() as calls:
            m.test_model()
            torch.cuda.synchronize()
        assert not any(n.endswith("_f16") for n in names(calls))
        out = m.score if task == "classifier" else m.predicted_pc
        outs.append(out.detach().clone())
    assert torch.equal(outs[0], outs[1])


@gpu
def test_mode_switch_applies_at_the_next_step():
    """The mode is read at each step's forward; a step's backward keeps its forward's mode."""
    from sonet_b200 import classifier, synth
    B, N = 4, 512
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device=DEV)
    opt.device = torch.device(DEV)
    inp = synth.synth_inputs(B, N, seed=9)
    m = classifier.Model(opt)
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    seen = []
    for mode in (None, "fp16", None, "fp16"):
        with train_tc(mode), profiled() as calls:
            m.optimize(epoch=0)
            torch.cuda.synchronize()
        f16 = [n for n in names(calls) if n.endswith("_f16")]
        seen.append(bool(f16))
        if mode == "fp16":
            assert set(f16) == {"sonet_pointwise_tc_forward_dev_f16", "sonet_wgrad_tc_f16"}
            assert not any(n in TWINS.values() for n in names(calls))
    assert seen == [False, True, False, True]
    with train_tc("fp16"):
        m.encoder.train()
        m.classifier.train()
        m.forward(is_train=True, epoch=0)
        loss = m.softmax_criteria(m.score, m.label)
    with profiled() as calls:          # the variable unset before backward: still fp16
        loss.backward()
    assert "sonet_wgrad_tc_f16" in names(calls) and "sonet_wgrad_tc_f32" not in names(calls)


@gpu
def test_data_parallel_training_accepts_the_mode():
    """DataParallelTraining wraps a model under the mode; its step runs the twins, and the
    BatchNorm route is the per-cloud one (the exchange is untouched)."""
    from sonet_b200 import classifier, dist, synth
    B, N = 4, 512
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device=DEV)
    opt.device = torch.device(DEV)
    inp = synth.synth_inputs(B, N, seed=4)
    with train_tc("fp16"):
        m = classifier.Model(opt)
        dp = dist.DataParallelTraining(m, B)
        try:
            m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
            with profiled() as calls:
                m.optimize(epoch=0)
                torch.cuda.synchronize()
        finally:
            dp.close()
    n = names(calls)
    assert "sonet_wgrad_tc_f16" in n and "sonet_bn_cloud_partials_f32" in n
    assert all(torch.isfinite(p).all() for p in m.encoder.parameters())


@gpu
def test_report_worst_bar_fractions():
    print("\n[train-fp16] worst bar fraction per family: " + ", ".join(
        "%s %.3f" % kv for kv in sorted(WORST.items())))
