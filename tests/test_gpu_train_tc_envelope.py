"""The train-mode wgmma convolution (train_ops.ConvTC, and UpConvTC's dgrad) at every tile edge,
across the fp32 exponent range and on non-finite gradients.

ConvTC runs three GEMMs on the generic wgmma layer (csrc/pointwise_tc.cu), each fed differently:

    forward  y  = W x + b   blob W, packed on the device, one pre-scale per W; x unscaled
    dgrad    dx = W^T dy    blob W^T (N = Cin, K = Cout); dy pre-scaled by one power of two per
                            tensor (sonet_absmax_scale_f32)
    wgrad    dW = dy x^T    sonet_wgrad_tc_f32: blob x [Cin][k = (b, p)], K padded to 64 * splits;
                            activation dy^T (rows = Cout), pre-scaled per dy channel

Error bar. helpers.tc_reference states the bar of the eval layer, whose activations are not
pre-scaled: |err| <= TC_R * m + TC_F * (sum_k |w_k| + sum_k |x_k| / s_w). An activation pre-scaled
by s_a carries its 2^-25 absolute split floor in scaled units, 2^-25 / s_a in its own, so the
activation-side floor term becomes TC_F * sum_k |w_k| / s_a: the same formula with the pre-scale
moved. s_a and s_w are the CAPPED pre-scales (at most 2^126, tc::pow2_scale), and 2^-148 absolute
covers the rounding of a result in the subnormal range.

Non-finite gradients. The gradient scalers give a NaN pre-scale when the tensor (dgrad, x of the
wgrad) or the dy channel (wgrad) holds an infinity, so an infinite gradient never comes back
finite through the saturating fp16 conversion: one +-inf in dy makes all of dx non-finite and the
dW rows of the channels that hold it; one +-inf in x makes all of dW non-finite. A NaN passes the
conversions and reaches exactly the outputs fp64 makes NaN, as -inf (the bare epilogue's fmaxf).
"""
import contextlib
import math

import numpy as np
import pytest
import torch

from helpers import TC_F, TC_FP32_FACTOR, TC_R, assert_rows_close, row_rel_err
from test_gpu_tc_envelope import _spread_dy, _strict_fp32, pw_config

DEV = "cuda:0"
gpu = pytest.mark.gpu

CAP = 126                    # tc::pow2_scale's exponent cap: 1/s stays a normal float
WGRAD_MAX_KPI = 32           # train_ops.WGRAD_MAX_KPI: K chunks per wgrad accumulator
SUB = 2.0 ** -148            # absolute rounding allowance of results in the subnormal range
FLT_MAX = float(np.finfo(np.float32).max)

# largest error seen per family, in units of its bar (printed by test_report_worst_bar_fractions)
WORST = {}


def _note(family, units):
    WORST[family] = max(WORST.get(family, 0.0), float(units))


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


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---- host mirrors of the train-mode routing (train_ops.py) -------------------------------------
def tc_eligible(cin, cout, rows):
    """conv_bn_act_train: ConvTC, else ConvStrict (cuDNN)."""
    return cin >= 32 and cout >= 32 and rows >= 256


def wgrad_on_tc(cin, cout):
    """ConvTC.backward: sonet_wgrad_tc_f32, else the strict-fp32 einsum."""
    return cout % 64 == 0 and cin >= 16


def wgrad_plan(B, P, cin, cout):
    """train_ops.wgrad_tc's K split and sonet_wgrad_kpad: (splits, Kpad, chunks per split)."""
    base = ((cout + 127) // 128) * (((cin + 63) // 64 * 64 + 255) // 256)
    kch = (B * P + 63) // 64
    splits = max(1, min(64, 296 // base, kch))
    if -(-kch // splits) > WGRAD_MAX_KPI:                     # train_ops.WGRAD_MAX_KPI
        splits = min(64, -(-kch // WGRAD_MAX_KPI))
    q = 64 * splits
    kpad = (B * P + q - 1) // q * q
    return splits, kpad, kpad // q


def pow2(m, cap=CAP):
    """tc::pow2_scale of a max |.| (finite, or 0)."""
    m = float(m)
    if not m > 0:
        return 1.0
    return math.ldexp(1.0, min(9 - math.frexp(m)[1], cap))


def grad_scale(values):
    """The gradient pre-scale (sonet_absmax_scale_f32, and one dy channel of the wgrad): NaN
    elements are ignored, an infinite max gives NaN."""
    v = np.abs(np.asarray(values, np.float32).ravel())
    v = v[~np.isnan(v)]
    m = float(v.max()) if v.size else 0.0
    return float("nan") if math.isinf(m) else pow2(m)


def pow2_t(m):
    """pow2 of every element of a tensor of finite maxima (float64 result)."""
    m = m.double()
    e = torch.frexp(m.clamp(min=1e-300))[1].double()
    return torch.where(m > 0, torch.pow(2.0, torch.clamp(9 - e, max=CAP)), torch.ones_like(m))


def tile_widths(N):
    """(n-tile >= 1, width) of every weight-blob n-tile of an N-row blob (tc::wblob)."""
    npad = (N + 63) // 64 * 64
    return {(nt >= 1, min(256, npad - 256 * nt)) for nt in range((npad + 255) // 256)}


def row_kind(rows):
    last = rows - 128 * ((rows + 127) // 128 - 1)
    if rows < 128:
        return "below"
    return {128: "exact", 1: "+1", 127: "-1"}.get(last, "ragged")


# ---- 1. route and tile coverage -------------------------------------------------------------------
# ConvTC cases (B, Cin, Cout, P), called directly (any shape runs; conv_bn_act_train's own choice is
# ROUTES below). The comment gives what each adds: forward blob N = Cout, dgrad blob N = Cin with
# K = Cout, wgrad rows = Cout with N = Cin and K = B*P padded to 64 * splits.
SWEEP = [
    (1, 16, 64, 100),       # Cin 16; rows < 128; wgrad splits 2 over 100 points: B*P < 64*splits
    (2, 40, 128, 128),      # Cin 40; rows exactly 2 tiles; dgrad K 128 (rem 64, 2 chunks)
    (3, 63, 192, 43),       # Cin 63; rows 129; wgrad row tiles 128 + 64
    (3, 64, 320, 85),       # rows 255; forward widths 256 + 64 (nt 1)
    (1, 65, 1024, 300),     # Cout 1024: forward nt 3 width 256, wgrad 8 row tiles
    (2, 255, 64, 700),      # dgrad N 255 -> width 256; wgrad splits 22, K tail 8
    (4, 256, 128, 512),     # rows 2048 (exact); wgrad splits 32, empty K tail
    (1, 257, 192, 1000),    # dgrad widths 256 + 64 (nt 1); wgrad splits 16
    (2, 387, 320, 640),     # dgrad nt 1 width 192; wgrad splits 20, empty K tail
    (1, 387, 1024, 1153),   # wgrad splits 18 of 2 chunks over 1153 points: the last splits are padding
    (1, 64, 128, 50),       # wgrad splits 1, one chunk with a tail of 14
    (1, 64, 64, 64),        # wgrad splits 1, no tail
    (2, 300, 448, 129),     # forward nt 1 width 192; dgrad nt 1 width 64
    (1, 128, 512, 333),     # forward nt 1 width 256; dgrad K rem 64 over 8 chunks
    (2, 100, 80, 150),      # Cout 80: einsum wgrad, dgrad K rem 16
    (1, 50, 96, 333),       # Cout 96: dgrad K rem 32
    (3, 200, 100, 99),      # Cout 100 (not a multiple of 16): dgrad K rem 48 (padded)
    (2, 130, 112, 256),     # Cout 112: dgrad K rem 48
    (1, 400, 384, 127),     # rows 127; forward nt 1 width 128; dgrad nt 1 width 192
    (1, 512, 32, 300),      # Cout 32: dgrad K rem 32, one chunk; dgrad nt 1 width 256
]

# conv_bn_act_train's choice at both sides of each tc_eligible bound: (B, Cin, Cout, P)
ROUTES = [
    (1, 31, 64, 300), (1, 32, 64, 300),           # Cin 31 / 32
    (1, 64, 31, 300), (1, 64, 32, 300),           # Cout 31 / 32 (32: einsum wgrad)
    (3, 64, 64, 85), (1, 64, 64, 256),            # rows 255 / 256
]

WGRAD_COUTS = {64, 128, 192, 320, 1024}
WGRAD_CINS = {16, 40, 63, 64, 65, 255, 256, 257, 387}


def _case_id(c):
    return "B%d-Cin%d-Cout%d-P%d" % c


def test_case_lists_reach_every_route_and_tile_edge():
    """Host-only: the cases reach both sides of every routing bound, both wgrad routes, every K
    split kind, every K remainder of the dgrad blob and every tile width and row-tile edge of the
    forward and dgrad GEMMs, and the wgrad's Cout and Cin sets."""
    from sonet_b200 import train_ops
    assert train_ops.WGRAD_MAX_KPI == WGRAD_MAX_KPI
    routes = {(tc_eligible(cin, cout, B * P), cin, cout, B * P) for B, cin, cout, P in ROUTES}
    assert {r[0] for r in routes} == {True, False}
    assert {(r[0], r[1]) for r in routes if r[2] >= 32 and r[3] >= 256} >= {(False, 31), (True, 32)}
    assert {(r[0], r[2]) for r in routes if r[1] >= 32 and r[3] >= 256} >= {(False, 31), (True, 32)}
    assert {(r[0], r[3]) for r in routes if r[1] >= 32 and r[2] >= 32} >= {(False, 255), (True, 256)}
    assert any(not wgrad_on_tc(cin, cout) and tc_eligible(cin, cout, B * P) for B, cin, cout, P in ROUTES)

    splits, tails, dg_rem, widths, rows = set(), set(), set(), set(), set()
    w_couts, w_cins, einsum = set(), set(), False
    for B, cin, cout, P in SWEEP:
        for N, K in ((cout, cin), (cin, cout)):             # forward, dgrad
            widths |= tile_widths(N)
        dg = pw_config(cout, cin, B * P)                      # dgrad: K = Cout
        dg_rem.add(dg["rem"])
        rows.add(row_kind(B * P))
        if cout % 16:
            dg_rem.add("Cout%16")
        if not wgrad_on_tc(cin, cout):
            einsum = einsum or cout % 64 != 0
            continue
        w_couts.add(cout)
        w_cins.add(cin)
        s, kpad, kpi = wgrad_plan(B, P, cin, cout)
        splits.add(s > 1)
        tail = kpad - B * P
        tails.add("empty" if tail == 0 else "tail")
        if B * P < 64 * s and s > 1:
            tails.add("B*P < 64*splits")
        if tail >= 64 * kpi and s > 1:
            tails.add("padding split")
    assert splits == {True, False}
    assert tails == {"empty", "tail", "B*P < 64*splits", "padding split"}
    assert dg_rem == {16, 32, 48, 64, "Cout%16"}
    assert widths == {(nt, w) for nt in (False, True) for w in (64, 128, 192, 256)}
    assert rows == {"below", "exact", "+1", "-1", "ragged"}
    assert einsum
    assert w_couts >= WGRAD_COUTS and w_cins >= WGRAD_CINS
    # the wgrad's row tiles over Cout: full tiles and a last tile of 64
    assert {c % 128 for c in w_couts} == {0, 64}


def _expected_calls(B, cin, cout, P):
    fwd = ["sonet_pointwise_tc_pack_device", "sonet_pointwise_tc_forward_dev"]
    bwd = ["sonet_pointwise_tc_pack_device", "sonet_absmax_scale_f32", "sonet_pointwise_tc_forward_dev"]
    if wgrad_on_tc(cin, cout):
        bwd.append("sonet_wgrad_tc_f32")
    return fwd, bwd


@gpu
@pytest.mark.parametrize("case", ROUTES, ids=_case_id)
def test_conv_bn_act_train_route(case):
    """conv_bn_act_train runs ConvTC exactly where tc_eligible says, and cuDNN (no call of the
    library) elsewhere."""
    from sonet_b200 import train_ops
    B, cin, cout, P = case
    g = _gen(sum(case))
    x = torch.randn(B, cin, P, generator=g).to(DEV).requires_grad_(True)
    W = (torch.randn(cout, cin, generator=g) * 0.1).to(DEV).requires_grad_(True)
    b = torch.randn(cout, generator=g).to(DEV).requires_grad_(True)
    with profiled() as fc:
        y = train_ops.conv_bn_act_train(x, W, b, None, None)
    with profiled() as bc:
        y.backward(torch.randn(B, cout, P, generator=g).to(DEV))
    if tc_eligible(cin, cout, B * P):
        fwd, bwd = _expected_calls(B, cin, cout, P)
        assert names(fc) == fwd and names(bc) == bwd
    else:
        assert names(fc) == [] and names(bc) == []


# ---- 2. shape sweep against fp64 ----------------------------------------------------------------
def gemm_bar(A, X, s_a, s_x):
    """fp64 out[b, n, p] = sum_k A[n, k] X[b, k, p] of the wgmma layer with blob A (pre-scale s_a)
    and activation X (pre-scale s_x: a number, or a [B, K, P]-broadcastable tensor) and its bar."""
    A64, X64 = A.double(), X.double()
    y = torch.einsum("nk,bkp->bnp", A64, X64)
    m = torch.einsum("nk,bkp->bnp", A64.abs(), X64.abs())
    floor = A64.abs().sum(1)[None, :, None] / s_x + X64.abs().sum(1, keepdim=True) / s_a
    return y, TC_R * m + TC_F * floor + SUB


def wgrad_bar(dy, x, s_o, s_x):
    """fp64 dW [Cout, Cin] = sum_{b,p} dy x^T and its bar: activation dy^T pre-scaled per channel
    by s_o [Cout], blob x pre-scaled by s_x."""
    d64, x64 = dy.double(), x.double()
    y = torch.einsum("bop,bip->oi", d64, x64)
    m = torch.einsum("bop,bip->oi", d64.abs(), x64.abs())
    floor = x64.abs().sum((0, 2))[None, :] / s_o.double()[:, None] + \
        d64.abs().sum((0, 2))[:, None] / s_x
    return y, TC_R * m + TC_F * floor + SUB


def in_bar(got, y, bar, what, family):
    """Every output whose fp64 value is below FLT_MAX / 2 is finite and inside the bar."""
    got = got.detach().double()
    ok = y.abs() < FLT_MAX / 2
    fin = torch.isfinite(got)
    assert bool(fin[ok].all()), "%s: %d non-finite outputs where fp64 is finite" % (
        what, int((~fin & ok).sum()))
    units = float(((got - y).abs() / bar)[ok].max()) if bool(ok.any()) else 0.0
    _note(family, units)
    assert units <= 1.0, "%s: error is %.3g x the bar" % (what, units)
    return units


def run_convtc(B, cin, cout, P, seed, family="shape"):
    """One ConvTC forward + backward against fp64: routes and splits against the mirror, a re-run
    bit for bit, y and dx inside the bar, rows of dx and dW within TC_FP32_FACTOR of strict fp32."""
    from sonet_b200 import train_ops
    g = _gen(seed)
    x0 = torch.randn(B, cin, P, generator=g).clamp(-3.5, 3.5)
    W0 = torch.randn(cout, cin, generator=g) * (2.0 / cin) ** 0.5
    b0 = torch.randn(cout, generator=g) * 0.1
    dy = _spread_dy(B, cout, P, g).to(DEV)

    def step(calls=None):
        x, W, b = (t.to(DEV).requires_grad_(True) for t in (x0, W0, b0))
        with profiled() as fc:
            y = train_ops.ConvTC.apply(x, W, b)
        with profiled() as bc:
            y.backward(dy)
        return (y.detach(), x.grad, W.grad, b.grad), fc, bc

    (y, dx, dW, db), fc, bc = step()
    fwd, bwd = _expected_calls(B, cin, cout, P)
    assert names(fc) == fwd and names(bc) == bwd
    assert fc[1][3][10] == 1 and bc[2][3][10] == 1                 # forward_dev: unsplit
    if wgrad_on_tc(cin, cout):
        a = bc[3][3]
        assert (a[2], a[3], a[4], a[5], a[6]) == (B, cout, cin, P, wgrad_plan(B, P, cin, cout)[0])
    again, _, _ = step()
    for t, u, n in zip((y, dx, dW, db), again, ("y", "dx", "dW", "db")):
        assert torch.equal(t, u), "re-run changed %s" % n

    x, W, b = x0.to(DEV), W0.to(DEV), b0.to(DEV)
    what = "ConvTC B=%d Cin=%d Cout=%d P=%d" % (B, cin, cout, P)
    s_w = pow2(W.abs().max())
    yf, bar = gemm_bar(W, x, s_w, 1.0)
    yf = yf + b.double()[None, :, None]
    in_bar(y, yf, bar + TC_R * b.double().abs()[None, :, None], what + " y", family)
    s_dy = pow2(dy.abs().max())
    dxf, bar = gemm_bar(W.t(), dy, s_w, s_dy)
    in_bar(dx, dxf, bar, what + " dx", family)

    rows = lambda t: t.permute(1, 0, 2)                            # rows = input channels
    ref32 = _strict_fp32(lambda: torch.einsum("oi,bop->bip", W, dy))
    e32 = float(row_rel_err(rows(ref32), rows(dxf)).max())
    assert_rows_close(rows(dx), rows(dxf), what + " dx rows", max(TC_FP32_FACTOR * e32, 1e-5))
    dWf = torch.einsum("bop,bip->oi", dy.double(), x.double())
    ref32 = _strict_fp32(lambda: torch.einsum("bop,bip->oi", dy, x))
    e32 = float(row_rel_err(ref32, dWf).max())
    assert_rows_close(dW, dWf, what + " dW rows", max(TC_FP32_FACTOR * e32, 1e-5))
    # db is PyTorch's fp32 sum: within 1e-6 of the sum of magnitudes
    d64 = dy.double()
    assert bool(((db.double() - d64.sum((0, 2))).abs() <= 1e-6 * d64.abs().sum((0, 2))).all())


@gpu
@pytest.mark.parametrize("case", SWEEP, ids=_case_id)
def test_convtc_shape_sweep(case):
    run_convtc(*case, seed=sum(case))


def _record_training_shapes(task):
    """Every distinct (Cin, Cout, B*P) -> (B, P) one optimize() step of `task` at the defaults sends
    to ConvTC."""
    from sonet_b200 import autoencoder, classifier, segmenter, synth, train_ops
    from helpers import build_states
    opt = synth.make_opt(task, device=DEV)
    opt.device = torch.device(DEV)
    B, N = opt.batch_size, opt.input_pc_num
    st = build_states(task, opt, seed=3)
    inp = synth.synth_inputs(B, N, seed=3)
    mod = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}[task]
    head = {"classifier": "classifier", "segmenter": "segmenter", "autoencoder": "decoder"}[task]
    seen = {}
    apply = train_ops.ConvTC.apply

    def spy(x, W, b):
        Bx, cin, P = x.shape
        seen.setdefault((cin, W.shape[0], Bx * P), (Bx, P))
        return apply(x, W, b)

    m = mod.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    getattr(m, head).load_state_dict(st["head"])
    if task == "segmenter":
        seg = torch.from_numpy(np.random.RandomState(3).randint(0, 50, size=(B, N)))
        m.set_input(inp["pc"], inp["sn"], inp["label"], seg, inp["node"], inp["node_knn_I"])
    else:
        m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    train_ops.ConvTC.apply = spy
    try:
        m.optimize(epoch=None)
    finally:
        train_ops.ConvTC.apply = apply
    return seen


_TRAINING_SHAPES_RUN = set()


@gpu
@pytest.mark.parametrize("task", ["classifier", "segmenter", "autoencoder"])
def test_convtc_training_shapes(task):
    """Each distinct ConvTC shape of one default optimize() step, once, as the shape sweep."""
    seen = _record_training_shapes(task)
    assert seen, "no ConvTC call in a %s step" % task
    print("\n[train-envelope] %s ConvTC shapes (Cin, Cout, B*P): %s" % (task, sorted(seen)))
    for key, (B, P) in sorted(seen.items()):
        if key in _TRAINING_SHAPES_RUN:                           # run by an earlier task
            continue
        _TRAINING_SHAPES_RUN.add(key)
        cin, cout, _ = key
        run_convtc(B, cin, cout, P, seed=cin + cout + P, family="training shape")


# ---- 3. exact scale-equivariance -------------------------------------------------------------------
def _exact_input(t, lo):
    """t with |t| < 2^lo set to zero, so that every power-of-two scaling below stays exact."""
    return torch.where(t.abs() < 2.0 ** lo, torch.zeros_like(t), t)


def assert_scaled(got, base, e, what):
    """got == 2^e * base bit for bit wherever 2^e * base is a normal float or zero."""
    want = base.double() * 2.0 ** e
    normal = (want.abs() >= 2.0 ** -126) | (want == 0)
    assert bool(normal.float().mean() > 0.5), what
    assert torch.equal(got.double()[normal], want[normal]), "%s: %d outputs differ" % (
        what, int((got.double() != want)[normal].sum()))


def _dgrad(W, dy):
    from sonet_b200 import train_ops
    x = torch.zeros(dy.shape[0], W.shape[1], dy.shape[2], device=DEV, requires_grad=True)
    y = train_ops.ConvTC.apply(x, W, None)
    return torch.autograd.grad(y, x, dy)[0]


EQ_B, EQ_CIN, EQ_COUT, EQ_P = 2, 96, 192, 300


@gpu
@pytest.mark.parametrize("e", [-116, -100, -64, -17, 5, 64, 100, 118])
def test_dgrad_scale_equivariance(e):
    """dgrad(W, 2^e dy) == 2^e dgrad(W, dy): the pre-scale of 2^e dy is 2^-e times dy's, so the
    GEMM sees the same fp16 operands and the epilogue's inverse absorbs 2^e exactly."""
    g = _gen(50)
    W = (torch.randn(EQ_COUT, EQ_CIN, generator=g) * 0.1).to(DEV)
    dy = _exact_input(torch.randn(EQ_B, EQ_COUT, EQ_P, generator=g), -8).to(DEV)
    dys = dy * 2.0 ** e
    assert torch.equal(dys * 2.0 ** -e, dy) and float(dys.abs().max()) >= 2.0 ** -118
    assert_scaled(_dgrad(W, dys), _dgrad(W, dy), e, "dgrad 2^%d" % e)


@gpu
@pytest.mark.parametrize("a,b", [(-100, 0), (0, -110), (-50, -60), (60, 50), (110, 0), (0, 110),
                                 (-100, 100), (7, -3)])
def test_wgrad_scale_equivariance(a, b):
    """wgrad(2^a dy, 2^b x) == 2^(a+b) wgrad(dy, x)."""
    from sonet_b200 import train_ops
    g = _gen(51)
    x = _exact_input(torch.randn(EQ_B, EQ_CIN, EQ_P, generator=g), -8).to(DEV)
    dy = _exact_input(_spread_dy(EQ_B, 128, EQ_P, g, lo=-3.0), -20).to(DEV)
    xs, dys = x * 2.0 ** b, dy * 2.0 ** a
    assert torch.equal(xs * 2.0 ** -b, x) and torch.equal(dys * 2.0 ** -a, dy)
    assert float(dy.abs().amax((0, 2)).min()) * 2.0 ** a >= 2.0 ** -118
    assert_scaled(train_ops.wgrad_tc(dys, xs), train_ops.wgrad_tc(dy, x), a + b,
                  "wgrad 2^%d dy, 2^%d x" % (a, b))


@gpu
@pytest.mark.parametrize("e", [-90, -30, 30, 100])
def test_wgrad_one_channel_scaled(e):
    """Scaling dy channel c by 2^e changes row c of dW alone, by exactly 2^e (its own pre-scale)."""
    from sonet_b200 import train_ops
    g = _gen(52)
    x = torch.randn(EQ_B, EQ_CIN, EQ_P, generator=g).to(DEV)
    dy = _exact_input(torch.randn(EQ_B, 128, EQ_P, generator=g), -10).to(DEV)
    c = 77
    dys = dy.clone()
    dys[:, c] *= 2.0 ** e
    base, got = train_ops.wgrad_tc(dy, x), train_ops.wgrad_tc(dys, x)
    keep = torch.ones(128, dtype=torch.bool, device=DEV)
    keep[c] = False
    assert torch.equal(got[keep], base[keep])
    assert_scaled(got[c], base[c], e, "dW row of a channel scaled by 2^%d" % e)


@gpu
@pytest.mark.parametrize("e", [-110, -60, -9, 60, 110])
def test_forward_scale_equivariance(e):
    """forward(2^e W, x, 2^e b) == 2^e forward(W, x, b)."""
    from sonet_b200 import train_ops
    g = _gen(53)
    x = torch.randn(EQ_B, EQ_CIN, EQ_P, generator=g).to(DEV)
    W = _exact_input(torch.randn(EQ_COUT, EQ_CIN, generator=g) * 0.1, -12).to(DEV)
    b = _exact_input(torch.randn(EQ_COUT, generator=g), -12).to(DEV)
    Ws, bs = W * 2.0 ** e, b * 2.0 ** e
    assert torch.equal(Ws * 2.0 ** -e, W) and torch.equal(bs * 2.0 ** -e, b)
    with torch.no_grad():
        assert_scaled(train_ops.ConvTC.apply(x, Ws, bs), train_ops.ConvTC.apply(x, W, b), e,
                      "forward 2^%d W" % e)


# ---- 4. the whole fp32 exponent range ------------------------------------------------------------
EXPONENTS = [-149, -140, -130, -126, -121, -120, -119, -118, -100, -64, 0, 64, 100, 127]
OPERANDS = ["dgrad-dy", "dgrad-W", "forward-W", "wgrad-dy", "wgrad-x", "upconv-dy"]


def _to_max(t, e):
    """t scaled so that max |t| == 2^e (in fp64, then rounded to fp32: tiny exponents flush most
    elements to subnormals or zero, and the references use the rounded tensor)."""
    t64 = t.double()
    return (t64 / t64.abs().max() * 2.0 ** e).float()


def _upconv_dgrad_range(e):
    from sonet_b200 import _C, ops, train_ops
    g = _gen(60)
    B, cin, cout, H, Wd = 2, 64, 64, 5, 6
    P = H * Wd
    x = torch.randn(B, cin, H, Wd, generator=g).to(DEV).requires_grad_(True)
    W = (torch.randn(cout, cin, 3, 3, generator=g) * 0.05).to(DEV)
    dz = _to_max(torch.randn(B, cout, 2 * H, 2 * Wd, generator=g), e).to(DEV)
    z = train_ops.UpConvTC.apply(x, W, None)
    with profiled() as calls:
        dx = torch.autograd.grad(z, x, dz)[0]
    assert names(calls)[:2] == ["sonet_upconv_fold_weights_f32", "sonet_pointwise_tc_pack_device"]
    assert "sonet_absmax_scale_f32" in names(calls)
    # the GEMM dx = Wdg D of the kernel's own operands: the folded weights and the gathered dz
    Wdg = torch.empty(cin, 16 * cout, device=DEV)
    train_ops._fold(W, cout, cin, False, None, Wdg)
    D = torch.empty(B, 16 * cout, P, device=DEV)
    ops._call("sonet_upconv_dgrad_im2col_f32", _C.ptr(dz), B, cout, H, Wd, _C.ptr(D), ops._stream(dz))
    y, bar = gemm_bar(Wdg, D, pow2(Wdg.abs().max()), pow2(dz.abs().max()))
    return dx.view(B, cin, P), y, bar


@gpu
@pytest.mark.parametrize("e", EXPONENTS)
@pytest.mark.parametrize("operand", OPERANDS)
def test_exponent_range(operand, e):
    """One operand scaled so its max is 2^e, the others O(1): every output finite wherever fp64 is
    below FLT_MAX / 2, and inside the bar of the capped pre-scales."""
    from sonet_b200 import train_ops
    what = "%s at 2^%d" % (operand, e)
    if operand == "upconv-dy":
        in_bar(*_upconv_dgrad_range(e), what, "range")
        return
    g = _gen(61)
    B, cin, cout, P = 2, 96, 128, 150
    x = torch.randn(B, cin, P, generator=g).clamp(-3.5, 3.5).to(DEV)
    W = (torch.randn(cout, cin, generator=g) * 0.15).to(DEV)
    dy = torch.randn(B, cout, P, generator=g).to(DEV)
    if operand.endswith("-W"):
        W = _to_max(W, e)
    elif operand.endswith("-x"):
        x = _to_max(x, e)
    else:
        dy = _to_max(dy, e)
    if operand == "forward-W":
        with torch.no_grad():
            got = train_ops.ConvTC.apply(x, W, None)
        in_bar(got, *gemm_bar(W, x, pow2(W.abs().max()), 1.0), what, "range")
    elif operand.startswith("dgrad"):
        in_bar(_dgrad(W, dy), *gemm_bar(W.t(), dy, pow2(W.abs().max()), pow2(dy.abs().max())),
               what, "range")
    else:
        with profiled() as calls:
            got = train_ops.wgrad_tc(dy, x)
        assert names(calls) == ["sonet_wgrad_tc_f32"]
        in_bar(got, *wgrad_bar(dy, x, pow2_t(dy.abs().amax((0, 2))), pow2(x.abs().max())), what,
               "range")


def _absmax_scale(t):
    from sonet_b200 import train_ops
    with profiled() as calls:
        s = train_ops._absmax_scale(t)
    assert names(calls) == ["sonet_absmax_scale_f32"]
    return s.cpu().numpy()


def _same_scale(got, want, what):
    want = np.array([want, 1.0 / want], np.float32)
    assert np.array_equal(got, want, equal_nan=True), "%s: got %s, want %s" % (what, got, want)


@gpu
@pytest.mark.parametrize("n", [1, 255, 256, 257, 2048 * 256 + 1])
def test_absmax_scale_grid_stride(n):
    """sonet_absmax_scale_f32 against the numpy mirror: the max at the first or the last element
    (the grid-stride loop's ends), positive or negative, at magnitudes across the range."""
    g = _gen(n)
    base = torch.rand(n, generator=g) * 2 - 1
    for pos in (0, n - 1):
        for v in (3.0, -3.0, -2.0 ** -119, 2.0 ** -130, 2.0 ** 100):
            t = base * abs(v) * 0.25
            t[pos] = v
            _same_scale(_absmax_scale(t.to(DEV)), grad_scale(t.numpy()), "n=%d max %g at %d" % (n, v, pos))


@gpu
@pytest.mark.parametrize("kind", ["-0", "subnormal", "nan-mixed", "all-nan", "+inf", "-inf",
                                  "inf-and-nan", "2^-118", "2^-125", "2^127"])
def test_absmax_scale_special_values(kind):
    """-0.0 scales like zero (1), a lone subnormal gets the capped 2^126, NaN elements are ignored,
    an infinite max gives a NaN scale, and 2^-118 is the smallest max the cap leaves alone."""
    n = 3000
    t = torch.zeros(n)
    if kind == "-0":
        t[:] = -0.0
    elif kind == "subnormal":
        t[1234] = -2.0 ** -140
    elif kind == "nan-mixed":
        t = torch.randn(n, generator=_gen(1)) * 1e-3
        t[::7] = float("nan")
    elif kind == "all-nan":
        t[:] = float("nan")
    elif kind in ("+inf", "-inf"):
        t = torch.randn(n, generator=_gen(2))
        t[2999] = float(kind)
    elif kind == "inf-and-nan":
        t[5] = float("nan")
        t[6] = float("inf")
    else:
        t = torch.rand(n, generator=_gen(3)) * 2.0 ** int(kind[2:])
        t[17] = 2.0 ** int(kind[2:])
    want = grad_scale(t.numpy())
    got = _absmax_scale(t.to(DEV))
    _same_scale(got, want, kind)
    if kind in ("+inf", "-inf", "inf-and-nan"):
        assert np.isnan(got).all()
    else:
        assert np.isfinite(got).all() and got[0] <= 2.0 ** CAP


@gpu
@pytest.mark.parametrize("e", [-149, -140, -125, -120, -119, -118])
@pytest.mark.parametrize("transpose", [0, 1])
def test_pack_device_tiny_matches_host_pack(e, transpose):
    """The device pack of a matrix with max 2^e equals the host pack bit for bit, with a finite,
    capped scale."""
    from sonet_b200 import ops, train_ops
    W = _to_max(torch.randn(100, 72, generator=_gen(70 - e)), e)
    blob, scale2 = train_ops._pack_device(W.to(DEV), bool(transpose))
    hblob, inv = ops.pointwise_tc_pack(W.t().contiguous() if transpose else W)
    s = scale2.cpu().numpy()
    assert np.isfinite(s).all() and s[0] == np.float32(pow2(W.abs().max()))
    assert s[1] == np.float32(inv)
    assert torch.equal(blob.cpu(), hblob)


# ---- 5. non-finite gradients ------------------------------------------------------------------------
NF_B, NF_CIN, NF_COUT, NF_P = 2, 64, 128, 150
NONFINITE = [(where, val, pattern) for where, pattern in (("dy", "element"), ("dy", "channel"),
                                                          ("dy", "cloud"), ("x", "element"))
             for val in ("nan", "+inf", "-inf")]


@gpu
@pytest.mark.parametrize("case", NONFINITE, ids=lambda c: "%s-%s-%s" % c)
def test_nonfinite_gradients(case):
    """No entry of dx, dW or db is finite where fp64 is not. What the kernels make of it: a NaN
    reaches exactly the outputs fp64 makes non-finite; an infinity in dy makes all of dx and the dW
    rows of its channels non-finite; an infinity in x all of dW."""
    from sonet_b200 import train_ops
    where, val, pattern = case
    g = _gen(80)
    x0 = torch.randn(NF_B, NF_CIN, NF_P, generator=g)
    W0 = torch.randn(NF_COUT, NF_CIN, generator=g) * 0.1
    b0 = torch.randn(NF_COUT, generator=g) * 0.1
    dy0 = torch.randn(NF_B, NF_COUT, NF_P, generator=g)
    bad = float(val)
    t = dy0 if where == "dy" else x0
    if pattern == "element":
        t[1, 37, 99] = bad
    elif pattern == "channel":
        t[:, 37, :] = bad
    else:
        t[1] = bad
    x, W, b = (u.to(DEV).requires_grad_(True) for u in (x0, W0, b0))
    y = train_ops.ConvTC.apply(x, W, b)
    with profiled() as calls:
        y.backward(dy0.to(DEV))
    assert "sonet_wgrad_tc_f32" in names(calls)
    # fp64 on the host: the pattern of non-finite results
    x64, W64, dy64 = x0.double(), W0.double(), dy0.double()
    ref = {"dx": torch.einsum("oi,bop->bip", W64, dy64),
           "dW": torch.einsum("bop,bip->oi", dy64, x64), "db": dy64.sum((0, 2))}
    got = {"dx": x.grad.cpu(), "dW": W.grad.cpu(), "db": b.grad.cpu()}
    for k in ref:
        bad_ref = ~torch.isfinite(ref[k])
        assert bool((~torch.isfinite(got[k]))[bad_ref].all()), "%s: finite where fp64 is not" % k
    nf = {k: ~torch.isfinite(v) for k, v in got.items()}
    nf_ref = {k: ~torch.isfinite(v) for k, v in ref.items()}
    if where == "dy":
        rows = (~torch.isfinite(dy0)).any(2).any(0)                # dy channels holding it
        assert torch.equal(nf["dW"], rows[:, None].expand(NF_COUT, NF_CIN))
        if val == "nan":
            assert torch.equal(nf["dx"], nf_ref["dx"])
        else:
            assert bool(nf["dx"].all())
    else:
        assert not bool(nf["dx"].any())
        if val == "nan":
            assert torch.equal(nf["dW"], nf_ref["dW"])
        else:
            assert bool(nf["dW"].all())


@gpu
@pytest.mark.parametrize("val", ["+inf", "-inf", "nan"])
def test_nonfinite_upstream_gradient_through_batchnorm(val):
    """An EquivariantLayer with BatchNorm and ReLU in train mode: with one non-finite element in the
    upstream gradient, every gradient that PyTorch's composition (kernels off) makes non-finite is
    non-finite with the kernels on too."""
    from sonet_b200 import layers, train_ops
    B, cin, cout, P = 2, 64, 128, 300
    g = _gen(90)
    x0 = torch.randn(B, cin, P, generator=g)
    up = torch.randn(B, cout, P, generator=g)
    up[1, 5, 17] = float(val)
    torch.manual_seed(90)
    layer = layers.EquivariantLayer(cin, cout, 'relu', 'batch').to(DEV).train()
    grads = {}
    for on in (False, True):
        prev = train_ops.ENABLED
        train_ops.ENABLED = on
        try:
            layer.zero_grad(set_to_none=True)
            x = x0.to(DEV).requires_grad_(True)
            with profiled() as calls:
                y = layer(x)
                y.backward(up.to(DEV))
            assert ("sonet_pointwise_tc_forward_dev" in names(calls)) == on
        finally:
            train_ops.ENABLED = prev
        grads[on] = {"x": x.grad.clone()}
        grads[on].update({n: p.grad.clone() for n, p in layer.named_parameters()})
    assert set(grads[True]) == set(grads[False])
    print("\n[train-envelope] upstream %s: non-finite fraction (kernels off / on) %s" % (val, ", ".join(
        "%s %.3f/%.3f" % (n, float((~torch.isfinite(grads[False][n])).float().mean()),
                          float((~torch.isfinite(grads[True][n])).float().mean())) for n in sorted(grads[True]))))
    assert not bool(torch.isfinite(grads[False]["x"]).all())
    for n in grads[False]:
        off = ~torch.isfinite(grads[False][n])
        assert bool((~torch.isfinite(grads[True][n]))[off].all()), \
            "%s: finite with the kernels where PyTorch is not" % n


@gpu
def test_forward_keeps_the_eval_saturation_rule():
    """ConvTC's forward gives the eval generic layer's bits on saturating and non-finite inputs:
    |x| >= 131008 acts as +-131008 (inf included) and NaN comes out as -inf."""
    from sonet_b200 import ops, train_ops
    g = _gen(95)
    B, cin, cout, P = 2, 96, 192, 300
    x = torch.randn(B, cin, P, generator=g)
    x[0, 3, ::5] = float("nan")
    x[1, 7, :] = float("inf")
    x[0, 9, 1::4] = float("-inf")
    x[1, 11, 2::3] = 1e6
    x[0, 13, :50] = -3e38
    x[1, 15, 5] = 131008.0
    W = torch.randn(cout, cin, generator=g) * 0.1
    b = torch.randn(cout, generator=g)
    xd, Wd, bd = x.to(DEV), W.to(DEV), b.to(DEV)
    with torch.no_grad():
        got = train_ops.ConvTC.apply(xd, Wd, bd)
    blob, inv = ops.pointwise_tc_pack(W)
    want = ops.pointwise_layer_tc(xd, blob.to(DEV), inv, bd, cout, False)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    assert bool(torch.isneginf(got[0, :, ::5][:, :10]).all())
    assert not bool(torch.isnan(got).any())


# ---- 6. summary -----------------------------------------------------------------------------------
@gpu
def test_report_worst_bar_fractions():
    """The largest error of each family of this run, in units of its bar."""
    for fam in sorted(WORST):
        print("\n[train-envelope] worst %s: %.3f of the bar" % (fam, WORST[fam]))
    assert all(v <= 1.0 for v in WORST.values())
