"""-m gpu: the fp32 CUDA-core kernels (csrc/pointwise.cu) at every dispatch edge, against plain
fp64 references.

Kernels under test: the register-tiled point-wise layer (64x64 and 128x128 tiles, vector and
scalar loads), the four MyLinear kernels (tiled, blocked with 4 / 2 / 1 channels per block, warp
per output) and the three row-max kernels (vector, small rows, warp per row). The host functions
below mirror the launchers' dispatch from the device's SM count and opt-in shared memory; one test
checks that the case lists reach every branch and that each case runs the kernel the mirror names.

Three kinds of reference:
- exact inputs: x, W multiples of 1/16 in [-1, 1], shift and addend multiples of 1/256, scale a
  power of two in {1/2, 1, 2}. Every partial sum of Cin <= 12288 such products is exact in fp32,
  so the result does not depend on the summation order and must equal the fp64 evaluation bit for
  bit (ReLU and no activation; ELU within 2 ulp of expm1).
- random inputs: |got - y| <= gamma(Cin + 3) * (|scale| sum|w x| + |shift| + |addend|), the bound
  of recursive fma summation in any order (gamma(n) = n u / (1 - n u), u = 2^-24). Derived, not
  measured: it cannot be flaky.
- invariances, bit for bit: both point-wise tile configurations and both load paths accumulate
  fmaf in ascending input-channel order, and every MyLinear row is independent of the batch.

Non-finite inputs: NaN and +-inf must come out where the fp64 PyTorch evaluation of the same
expression has them; ReLU and the row max propagate NaN as torch.relu and torch.amax do.
"""
import contextlib
import json
import os
import re
import tempfile

import pytest
import torch
import torch.nn.functional as F

DEV = "cuda:0"
gpu = pytest.mark.gpu
U = 2.0 ** -24
ACTS = (None, "relu", "elu")


# ---- dispatch mirrors (csrc/pointwise.cu: sonet_pointwise_layer_f32, launch_linear, sonet_rowmax_f32)
def _aligned(*ts):
    return all(t is None or t.data_ptr() % 16 == 0 for t in ts)


def pw_route(P, Cout, vec_ok, w_ok):
    """(tile, VECP, 128-bit weight loads); vec_ok: x0 / x1 / out 16-byte aligned, w_ok: Wt is."""
    tile = 128 if P >= 1024 and Cout >= 128 else 64
    return tile, P % 4 == 0 and vec_ok, Cout % 4 == 0 and w_ok


def device_limits():
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.shared_memory_per_block_optin


def linear_route(B, Cin, Cout, aligned, sms, optin):
    if Cin % 4 == 0 and aligned:
        if (16 + 16) * (Cin // 4 + 1) * 16 <= optin and (B + 15) // 16 <= 65535:
            return "tile"
        ct = 4
        while ct > 1 and (-(-Cout // ct) < (sms * 3) // 4 or ct * Cin * 4 > 48 * 1024):
            ct //= 2
        if ct * Cin * 4 <= 48 * 1024:
            return "block%d" % ct
    return "warp"


def rowmax_route(L, aligned):
    G = L // 4
    if L % 4 == 0 and 1 <= G <= 32 and G & (G - 1) == 0 and L > 32 and aligned:
        return "vec"
    return "small" if L <= 32 else "warp"


def tile_cin_max(optin):
    """The largest Cin the tiled MyLinear kernel takes: 32 rows of Cin + 4 floats in shared memory."""
    return 4 * (optin // 512 - 1)


def ct_threshold(ct, sms):
    """The smallest Cout at which launch_linear keeps ct channels per block (shared memory allowing)."""
    return ct * ((sms * 3) // 4 - 1) + 1


def resolve(v, sms, optin):
    """Case dimensions may name a device-dependent edge: TILE (tile_cin_max), CT4 / CT2
    (ct_threshold), with an optional signed offset ("CT4-1", "TILE+4")."""
    if isinstance(v, int):
        return v
    m = re.fullmatch(r"(TILE|CT4|CT2)([+-]\d+)?", v)
    base = {"TILE": tile_cin_max(optin), "CT4": ct_threshold(4, sms), "CT2": ct_threshold(2, sms)}
    return base[m.group(1)] + int(m.group(2) or 0)


_KERNEL = re.compile(r"sonet::(pointwise_kernel|linear_tile_kernel|linear_block_kernel|linear_kernel|"
                     r"rowmax_vec_kernel|rowmax_small_kernel|rowmax_warp_kernel)(<[^>]*>)?")


@contextlib.contextmanager
def kernels_launched():
    """The sonet kernels launched inside the block, in launch order, as (name, template args)."""
    from torch.profiler import ProfilerActivity, profile
    out = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        yield out
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    evs = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    for e in evs:
        m = _KERNEL.search(e["name"])
        if m:
            args = tuple(a.strip() for a in (m.group(2) or "<>")[1:-1].split(",") if a.strip())
            out.append((m.group(1), args))


# ---- input generators ------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def exact_vals(shape, g, denom, span=1):
    """Multiples of 1/denom in [-span, span]."""
    return (torch.randint(-span * denom, span * denom + 1, shape, generator=g).double() / denom).float()


def pow2_scale(n, g):
    return torch.pow(2.0, torch.randint(-1, 2, (n,), generator=g).float())


def offset_copy(t, off):
    """A contiguous view of t's values starting `off` floats into a fresh buffer (off = 1: only
    4-byte aligned)."""
    base = torch.zeros(t.numel() + off, dtype=t.dtype, device=DEV)
    v = base[off:].view(t.shape)
    v.copy_(t)
    return v


def gamma(n):
    return n * U / (1 - n * U)


def ulp32(v):
    v = v.float().abs()
    return (torch.nextafter(v, torch.full_like(v, float("inf"))) - v).double()


def apply_act(y, act):
    if act == "relu":
        return torch.relu(y)
    if act == "elu":
        return F.elu(y)
    return y


def assert_exact(got, y, act, what):
    """got (fp32) == act(y) (fp64, exact) bit for bit; ELU within 2 ulp of expm1."""
    want = apply_act(y, act)
    got = got.double().to(want.device)
    if act == "elu":
        err = (got - want).abs()
        lim = 2 * ulp32(want)
        bad = err > lim
        assert not bool(bad.any()), "%s: ELU off by %.3g ulp" % (what, float((err / lim * 2).max()))
    else:
        assert torch.equal(got, want.float().double()), "%s: %d entries differ from the exact result" % (
            what, int((got != want).sum()))


def assert_in_bound(got, y, bar, act, what):
    """|got - act(y)| <= bar (+ 2 ulp of expm1 for ELU); act is 1-Lipschitz."""
    want = apply_act(y, act)
    lim = bar + (2 * ulp32(want) if act == "elu" else 0)
    u = float(((got.double().to(want.device) - want).abs() / lim.clamp(min=1e-300)).max())
    assert u <= 1.0, "%s: error is %.3g x the fp32 summation bound" % (what, u)
    return u


# ---- point-wise layer ----------------------------------------------------------------------------------
def pw_reference(x, W, scale, shift, add, gidx):
    """fp64 y = scale * (W x) + shift + addend[gidx clamped]; and sum |w x| terms for the bound.
    x [B,Cin,P], W [Cout,Cin] on any device; returns on DEV."""
    x64, W64 = x.to(DEV, torch.float64), W.to(DEV, torch.float64)
    y = torch.einsum("oc,bcp->bop", W64, x64)
    m = torch.einsum("oc,bcp->bop", W64.abs(), x64.abs())
    if scale is not None:
        s = scale.to(DEV, torch.float64)[None, :, None]
        y, m = y * s, m * s.abs()
    if shift is not None:
        s = shift.to(DEV, torch.float64)[None, :, None]
        y, m = y + s, m + s.abs()
    if add is not None:
        B, Cout, G = add.shape
        idx = gidx.to(DEV).long().clamp(0, G - 1)[:, None, :].expand(B, Cout, -1)
        a = torch.gather(add.to(DEV, torch.float64), 2, idx)
        y, m = y + a, m + a.abs()
    return y, m


# (B, C0, C1, P, Cout, G, scale, shift, view): view "" aligned, "x" x0 / x1 / out offset by one
# float (scalar path), "w" Wt offset by one float (scalar weight loads)
PW = [
    (2, 3, 0, 1024, 128, 0, True, True, ""),        # 128x128 VECP; one K slab; Cout = 128
    (1, 64, 0, 1027, 129, 0, False, True, ""),      # 128x128 scalar; Cin % 8 = 0; Cout 128 + 1
    (2, 13, 0, 1100, 130, 7, True, False, ""),      # 128x128 VECP; Cin % 8 = 5; Cout % 4 = 2; G = 7
    (1, 38, 41, 1025, 255, 0, True, True, ""),      # 128x128 scalar; split inside a slab; 256 - 1
    (2, 16, 32, 2048, 256, 1, False, True, ""),     # 128x128 VECP; split at a slab edge; G = 1
    (1, 100, 0, 1030, 257, 64, True, True, ""),     # 128x128 scalar; Cin % 8 = 4; 256 + 1; G = 64
    (2, 387, 0, 1024, 512, 0, False, True, ""),     # 128x128 VECP; the KNN module's first layer
    (1, 15, 0, 1024, 1000, 0, True, False, ""),     # 128x128 VECP; Cin % 8 = 7; Cout 1000
    (3, 6, 0, 256, 64, 0, False, False, ""),        # 64x64 VECP; Cout = 64; neither scale nor shift
    (2, 1, 0, 63, 63, 0, True, True, ""),           # 64x64 scalar; Cin 1; Cout 64 - 1; P < 64
    (1, 2, 0, 1023, 65, 0, True, True, ""),         # 64x64 scalar (P 1024 - 1); Cout 64 + 1
    (2, 200, 10, 512, 127, 5, False, True, ""),     # 64x64 VECP; split at a slab edge; 128 - 1
    (1, 21, 0, 4096, 100, 0, True, True, ""),       # 64x64 at large P (Cout < 128)
    (1, 300, 9, 777, 192, 3, True, False, ""),      # 64x64 scalar; split inside a slab; 3 x 64
    (2, 1, 0, 5, 1, 0, True, True, ""),             # Cout 1, P 5
    (2, 41, 0, 1024, 128, 0, True, True, "w"),      # 128x128, offset Wt with Cout % 4 == 0
    (1, 40, 0, 300, 64, 2, False, True, "w"),       # 64x64, offset Wt with Cout % 4 == 0
    (2, 12, 10, 1024, 132, 0, True, True, "x"),     # 128x128 scalar through offset views, P % 4 == 0
    (1, 33, 0, 512, 68, 0, True, False, "x"),       # 64x64 scalar through offset views
]


def _pw_id(c):
    return "B%d-C%d+%d-P%d-O%d%s%s%s%s" % (c[0], c[1], c[2], c[3], c[4], "-G%d" % c[5] if c[5] else "",
                                           "" if c[6] else "-noscale", "" if c[7] else "-noshift",
                                           "-off" + c[8] if c[8] else "")


def pw_inputs(case, g, exact):
    B, C0, C1, P, Cout, G, sc, sh, _ = case
    Cin = C0 + C1
    if exact:
        x, W = exact_vals((B, Cin, P), g, 16), exact_vals((Cout, Cin), g, 16)
        scale = pow2_scale(Cout, g) if sc else None
        shift = exact_vals((Cout,), g, 256, 4) if sh else None
        add = exact_vals((B, Cout, G), g, 256, 4) if G else None
    else:
        x = torch.randn(B, Cin, P, generator=g)
        W = torch.randn(Cout, Cin, generator=g) * (2.0 / Cin) ** 0.5
        scale = torch.rand(Cout, generator=g) * 1.5 + 0.25 if sc else None
        shift = torch.randn(Cout, generator=g) if sh else None
        add = torch.randn(B, Cout, G, generator=g) if G else None
    gidx = None
    if G:
        gidx = torch.randint(0, G, (B, P), generator=g).int()
        gidx[:, ::7] = -3                           # out of range: the kernel clamps to 0 / G - 1
        gidx[:, 3::11] = G + 5
    return x, W, scale, shift, add, gidx


def run_pw(case, x, W, scale, shift, add, gidx, act):
    """One ops.pointwise_layer call laid out as the case says; returns (out, route)."""
    from sonet_b200 import ops
    B, C0, C1, P, Cout, G, _, _, view = case
    xd = x.to(DEV)
    x0, x1 = xd[:, :C0].contiguous(), (xd[:, C0:].contiguous() if C1 else None)
    Wt = W.t().contiguous().to(DEV)
    out = None
    if view == "x":
        x0 = offset_copy(x0, 1)
        x1 = offset_copy(x1, 1) if x1 is not None else None
        out = offset_copy(torch.empty(B, Cout, P, device=DEV), 1)
    elif view == "w":
        Wt = offset_copy(Wt, 1)
    dv = lambda t: None if t is None else t.to(DEV)        # noqa: E731
    got = ops.pointwise_layer(x0, Wt, dv(scale), dv(shift), act, x1=x1, addend=dv(add), gidx=dv(gidx),
                              out=out)
    return got, pw_route(P, Cout, _aligned(x0, x1, got), _aligned(Wt))


@gpu
@pytest.mark.parametrize("case", PW, ids=_pw_id)
def test_pointwise_exact_inputs(case):
    g = _gen(sum(case[:6]))
    x, W, scale, shift, add, gidx = pw_inputs(case, g, exact=True)
    y, _ = pw_reference(x, W, scale, shift, add, gidx)
    for act in ACTS:
        got, route = run_pw(case, x, W, scale, shift, add, gidx, act)
        assert_exact(got, y, act, "%s %s %s" % (_pw_id(case), act, route))


@gpu
@pytest.mark.parametrize("case", PW, ids=_pw_id)
def test_pointwise_random_inputs_within_bound(case):
    g = _gen(7 + sum(case[:6]))
    x, W, scale, shift, add, gidx = pw_inputs(case, g, exact=False)
    y, m = pw_reference(x, W, scale, shift, add, gidx)
    bar = gamma(case[1] + case[2] + 3) * m
    for act in ACTS:
        got, route = run_pw(case, x, W, scale, shift, add, gidx, act)
        assert_in_bound(got, y, bar, act, "%s %s %s" % (_pw_id(case), act, route))


@gpu
def test_pointwise_tile_configs_and_load_paths_agree_bitwise():
    """Columns 0..1022 of a P = 1024 run (128x128, VECP) == a P = 1023 run (64x64, scalar), and an
    offset view of x0 / x1 / out (128x128, scalar) == the aligned run: all accumulate fmaf in
    ascending input-channel order."""
    from sonet_b200 import ops
    g = _gen(3)
    B, C0, C1, Cout, G = 2, 45, 30, 200, 9
    x = torch.randn(B, C0 + C1, 1024, generator=g).to(DEV)
    Wt = (torch.randn(C0 + C1, Cout, generator=g) * 0.15).to(DEV)
    shift = torch.randn(Cout, generator=g).to(DEV)
    add = torch.randn(B, Cout, G, generator=g).to(DEV)
    gidx = torch.randint(-2, G + 2, (B, 1024), generator=g).int().to(DEV)
    for act in ACTS:
        x0, x1 = x[:, :C0].contiguous(), x[:, C0:].contiguous()
        full = ops.pointwise_layer(x0, Wt, None, shift, act, x1=x1, addend=add, gidx=gidx)
        assert pw_route(1024, Cout, True, True)[:2] == (128, True)
        short = ops.pointwise_layer(x0[:, :, :1023].contiguous(), Wt, None, shift, act,
                                    x1=x1[:, :, :1023].contiguous(), addend=add,
                                    gidx=gidx[:, :1023].contiguous())
        assert pw_route(1023, Cout, True, True)[:2] == (64, False)
        assert torch.equal(full[:, :, :1023], short), act
        o0, o1 = offset_copy(x0, 1), offset_copy(x1, 1)
        out = offset_copy(torch.empty_like(full), 1)
        off = ops.pointwise_layer(o0, Wt, None, shift, act, x1=o1, addend=add, gidx=gidx, out=out)
        assert not _aligned(o0, o1, off)
        assert torch.equal(off, full), act


# ---- MyLinear ------------------------------------------------------------------------------------------
# (B, Cin, Cout, view): Cin / Cout may name a device-dependent edge (resolve); view "x" / "w": that
# operand as a view one float into its buffer (not 16-byte aligned), "x4": four floats (aligned)
LINEAR = [
    (1, 4, 1, ""),                  # tile: smallest
    (17, 64, 3, ""),                # tile: odd B, Cout < 16
    (16, 1024, 512, ""),            # tile: the classifier's fc2
    (129, "TILE", 17, ""),          # tile: largest Cin, Cout 16 + 1, 9 row tiles
    (33, "TILE", 16, "x4"),         # tile: largest Cin, offset but aligned x
    (15, 260, 15, ""),              # tile: Cout 16 - 1
    (17, "TILE+4", "CT4", ""),      # block<4>: one past the tile kernel, smallest Cout for 4
    (33, 3072, "CT4+15", ""),       # block<4>: largest Cin for 4 channels in 48 KB
    (1, "TILE+4", 1024, ""),        # block<4>: B = 1
    (15, "TILE+4", "CT4-1", ""),    # block<2>: Cout one below the 4-channel threshold
    (129, 3076, "CT4", ""),         # block<2>: Cin one step past 4 channels in 48 KB
    (16, 6144, "CT2", ""),          # block<2>: largest Cin for 2 channels, smallest Cout for 2
    (17, "TILE+4", "CT2-1", ""),    # block<1>: Cout one below the 2-channel threshold
    (33, 6148, 512, ""),            # block<1>: Cin one step past 2 channels in 48 KB
    (4, 12288, 8, ""),              # block<1>: largest Cin in 48 KB
    (16, 12292, 33, ""),            # warp: Cin past every shared-memory kernel
    (129, 1030, 17, ""),            # warp: Cin % 4 = 2
    (15, 3, 5, ""),                 # warp: Cin % 4 = 3
    (33, 1023, 130, ""),            # warp: Cin % 4 = 3
    (17, 1024, 40, "x"),            # warp: offset x
    (16, 2048, 100, "w"),           # warp: offset W
]


def _lin_id(c):
    return "B%d-Cin%s-Cout%s%s" % (c[0], c[1], c[2], "-off" + c[3] if c[3] else "")


def lin_case(case):
    sms, optin = device_limits()
    B, Cin, Cout, view = case
    return B, resolve(Cin, sms, optin), resolve(Cout, sms, optin), view


def lin_operands(x, W, view):
    xd, Wd = x.to(DEV), W.to(DEV)
    if view in ("x", "x4"):
        xd = offset_copy(xd, 1 if view == "x" else 4)
    elif view == "w":
        Wd = offset_copy(Wd, 1)
    return xd, Wd


def lin_reference(x, W, scale, shift):
    x64, W64 = x.to(DEV, torch.float64), W.to(DEV, torch.float64)
    y, m = x64 @ W64.t(), x64.abs() @ W64.abs().t()
    if scale is not None:
        s = scale.to(DEV, torch.float64)
        y, m = y * s, m * s.abs()
    if shift is not None:
        s = shift.to(DEV, torch.float64)
        y, m = y + s, m + s.abs()
    return y, m


@gpu
@pytest.mark.parametrize("case", LINEAR, ids=_lin_id)
def test_linear_exact_random_and_batch_invariant(case):
    from sonet_b200 import ops
    B, Cin, Cout, view = lin_case(case)
    g = _gen(B + Cin + Cout)
    # exact inputs, bit for bit
    x, W = exact_vals((B, Cin), g, 16), exact_vals((Cout, Cin), g, 16)
    for k, act in enumerate(ACTS):
        scale = pow2_scale(Cout, g) if k != 1 else None
        shift = exact_vals((Cout,), g, 256, 4) if k != 2 else None
        xd, Wd = lin_operands(x, W, view)
        got = ops.linear(xd, Wd, None if scale is None else scale.to(DEV),
                         None if shift is None else shift.to(DEV), act)
        y, _ = lin_reference(x, W, scale, shift)
        assert_exact(got, y, act, "%s %s" % (_lin_id(case), act))
    # random inputs, rigorous bound; rows do not depend on the batch
    x = torch.randn(B, Cin, generator=g)
    W = torch.randn(Cout, Cin, generator=g) * (2.0 / Cin) ** 0.5
    scale = torch.rand(Cout, generator=g) + 0.5
    shift = torch.randn(Cout, generator=g)
    y, m = lin_reference(x, W, scale, shift)
    xd, Wd = lin_operands(x, W, view)
    sd, hd = scale.to(DEV), shift.to(DEV)
    for act in ACTS:
        got = ops.linear(xd, Wd, sd, hd, act)
        assert_in_bound(got, y, gamma(Cin + 3) * m, act, "%s %s" % (_lin_id(case), act))
        for lo, hi in ((0, 1), (B - 1, B), (B // 3, B // 3 + 2), (1, B)):
            if hi <= B and lo < hi:
                sub = ops.linear(lin_operands(x[lo:hi], W, view)[0], Wd, sd, hd, act)
                assert torch.equal(sub, got[lo:hi]), (lo, hi, act)


# ---- row max ----------------------------------------------------------------------------------------
# (R, L, view): the vector kernel handles 4 * (32 / G) rows per warp (8 at L = 64, 4 at L = 128)
ROWMAX = [
    (7, 64, ""), (8, 64, ""), (9, 64, ""), (37, 64, ""),
    (3, 128, ""), (4, 128, ""), (5, 128, ""), (300, 128, ""),
    (19, 1, ""), (300, 4, ""), (40, 31, ""), (257, 32, ""),
    (20, 33, ""), (9, 40, ""), (33, 256, ""), (12, 1000, ""), (21, 64, "x"),
]


def _special_rows(L):
    """(positions, values) written into rows 0, 1, ... in turn: +-inf, an all -inf row, NaN at the
    first, last and a middle position, NaN beside +inf."""
    inf, nan = float("inf"), float("nan")
    mid = L // 2
    rows = [([0], [inf]), ([L - 1], [-inf]), (list(range(L)), [-inf] * L), ([0], [nan]),
            ([L - 1], [nan]), ([mid], [nan]), ([mid], [inf])]
    if L > 1:
        rows += [([0, L - 1], [inf, nan]), ([mid, 0], [-inf, nan])]
    return rows


@gpu
@pytest.mark.parametrize("R,L,view", ROWMAX, ids=lambda v: str(v))
def test_rowmax_vs_amax_with_non_finite_rows(R, L, view):
    from sonet_b200 import ops
    t = torch.randn(R, L, generator=_gen(R * 1000 + L))
    for r, (pos, vals) in enumerate(_special_rows(L)):
        if r < R:
            t[r, pos] = torch.tensor(vals)
    if R > 12:
        t[R - 1, L // 3] = float("nan")             # the last row (a partial warp)
    td = offset_copy(t.to(DEV), 1) if view == "x" else t.to(DEV)
    got = ops.rowmax(td)
    torch.testing.assert_close(got.cpu(), torch.amax(t, dim=1), rtol=0, atol=0, equal_nan=True)


# ---- every branch is reached -----------------------------------------------------------------------
@gpu
def test_case_lists_reach_every_branch():
    """The mirrors above, applied to the case lists, reach every branch of the three launchers;
    and the kernel each case launches is the one its mirror names."""
    from sonet_b200 import ops
    sms, optin = device_limits()
    pw_expect, lin_expect, rm_expect = [], [], []
    with kernels_launched() as seen:
        for case in PW:
            x, W, scale, shift, add, gidx = pw_inputs(case, _gen(0), exact=True)
            _, route = run_pw(case, x, W, scale, shift, add, gidx, "relu")
            pw_expect.append(route)
        for case in LINEAR:
            B, Cin, Cout, view = lin_case(case)
            xd, Wd = lin_operands(torch.zeros(B, Cin), torch.zeros(Cout, Cin), view)
            ops.linear(xd, Wd, None, None, "relu")
            lin_expect.append(linear_route(B, Cin, Cout, _aligned(xd, Wd), sms, optin))
        for R, L, view in ROWMAX:
            t = torch.zeros(R, L, device=DEV)
            t = offset_copy(t, 1) if view == "x" else t
            ops.rowmax(t)
            rm_expect.append(rowmax_route(L, _aligned(t)))
    seen = list(seen)
    assert len(seen) == len(PW) + len(LINEAR) + len(ROWMAX), seen
    pw_seen, lin_seen, rm_seen = (seen[:len(PW)], seen[len(PW):len(PW) + len(LINEAR)],
                                  seen[len(PW) + len(LINEAR):])
    for (name, args), (tile, vecp, _) in zip(pw_seen, pw_expect):
        assert name == "pointwise_kernel" and args[:2] == (str(tile), str(tile))
        assert args[4] in (("true", "1") if vecp else ("false", "0")), (args, tile, vecp)
    lin_names = {"tile": ("linear_tile_kernel", ()), "block4": ("linear_block_kernel", ("4",)),
                 "block2": ("linear_block_kernel", ("2",)), "block1": ("linear_block_kernel", ("1",)),
                 "warp": ("linear_kernel", ())}
    for (name, args), want, case in zip(lin_seen, lin_expect, LINEAR):
        wn, wa = lin_names[want]
        assert name == wn and args[:len(wa)] == wa, (case, want, name, args)
    for (name, _), want in zip(rm_seen, rm_expect):
        assert name == "rowmax_%s_kernel" % want
    # coverage
    assert {(t, v, w) for t, v, w in pw_expect} >= {(128, True, True), (128, False, True),
                                                    (64, True, True), (64, False, True),
                                                    (128, True, False), (64, True, False)}
    assert set(lin_expect) == {"tile", "block4", "block2", "block1", "warp"}
    assert set(rm_expect) == {"vec", "small", "warp"}
    couts = {c[4] for c in PW}
    assert {c % 4 for c in couts} == {0, 1, 2, 3}
    assert {63, 64, 65, 127, 128, 129, 255, 256, 257} <= couts
    cins = [(c[1] + c[2], -(-(c[1] + c[2]) // 8)) for c in PW]
    assert {n % 8 for n, k in cins if k > 1} == set(range(8)) and any(k == 1 for _, k in cins)
    splits = {c[1] % 8 == 0 for c in PW if c[2]}
    assert splits == {True, False} and any(c[2] == 0 for c in PW)
    assert {c[5] for c in PW} >= {0, 1} and any(c[5] > 1 for c in PW)
    assert {c[6] for c in PW} == {True, False} and {c[7] for c in PW} == {True, False}
    assert {B for B, *_ in LINEAR} >= {1, 15, 16, 17, 33, 129}
    lin_dims = [lin_case(c) for c in LINEAR]
    tile_max = tile_cin_max(optin)
    assert {tile_max, tile_max + 4} <= {c[1] for c in lin_dims}
    assert {ct_threshold(4, sms), ct_threshold(4, sms) - 1, ct_threshold(2, sms),
            ct_threshold(2, sms) - 1} <= {c[2] for c in lin_dims}
    assert {c[2] % 16 for c in lin_dims} >= {0, 1, 15}
    assert {c[3] for c in LINEAR} >= {"x", "w"}
    assert any(B % 2 for (B, _, _, _), r in zip(lin_dims, lin_expect) if r.startswith("block"))
    assert {L for _, L, _ in ROWMAX} >= {1, 4, 31, 32, 33, 40, 64, 128, 256, 1000}


# ---- non-finite inputs through the kernels ----------------------------------------------------------
def _poison(t, g, n, vals):
    flat = t.view(-1)
    idx = torch.randperm(flat.numel(), generator=g)[:n * len(vals)]
    for i, v in enumerate(vals):
        flat[idx[i * n:(i + 1) * n]] = v
    return t


def _elementwise_ref(W, x, scale, shift):
    """fp64 y[b,o,p] = scale[o] * sum_c W[o,c] x[b,c,p] + shift[o] from explicit products, so that
    inf * 0 and inf - inf give NaN exactly as IEEE arithmetic does."""
    prod = W.double()[None, :, :, None] * x.double()[:, None, :, :]
    y = prod.sum(2)
    m = prod.abs().sum(2)
    if scale is not None:
        y, m = y * scale.double()[None, :, None], m * scale.double().abs()[None, :, None]
    if shift is not None:
        y, m = y + shift.double()[None, :, None], m + shift.double().abs()[None, :, None]
    return y, m


def assert_nonfinite_pattern(got, y, bar, act, what):
    """NaN, +inf and -inf exactly where act(y) has them; finite entries within the bound."""
    want = apply_act(y, act)
    got = got.double().cpu()
    assert torch.equal(torch.isnan(got), torch.isnan(want)), "%s: NaN pattern" % what
    inf = torch.isinf(want)
    assert torch.equal(torch.isinf(got), inf) and torch.equal(got[inf], want[inf]), "%s: inf pattern" % what
    fin = torch.isfinite(want)
    assert bool(fin.any()) and bool((~fin).any())
    lim = bar + (2 * ulp32(want) if act == "elu" else 0)
    assert bool(((got[fin] - want[fin]).abs() <= lim[fin]).all()), "%s: finite entries" % what


NONFINITE = [("x", [float("nan"), float("inf"), float("-inf")]), ("W", [float("nan"), float("inf")]),
             ("shift", [float("nan"), float("-inf"), float("inf")])]


@gpu
@pytest.mark.parametrize("where,vals", NONFINITE, ids=[w for w, _ in NONFINITE])
@pytest.mark.parametrize("B,C0,C1,P,Cout", [(2, 7, 5, 1030, 130), (1, 20, 0, 70, 20)])
def test_pointwise_non_finite_inputs(where, vals, B, C0, C1, P, Cout):
    from sonet_b200 import ops
    g = _gen(B + C0 + P)
    x = torch.randn(B, C0 + C1, P, generator=g)
    W = torch.randn(Cout, C0 + C1, generator=g) * 0.3
    scale = torch.rand(Cout, generator=g) + 0.5
    shift = torch.randn(Cout, generator=g)
    _poison({"x": x, "W": W, "shift": shift}[where], g, 2, vals)
    y, m = _elementwise_ref(W, x, scale, shift)
    bar = gamma(C0 + C1 + 3) * m
    xd = x.to(DEV)
    for act in ACTS:
        got = ops.pointwise_layer(xd[:, :C0].contiguous(), W.t().contiguous().to(DEV), scale.to(DEV),
                                  shift.to(DEV), act, x1=xd[:, C0:].contiguous() if C1 else None)
        assert_nonfinite_pattern(got, y, bar, act, "pointwise %s %s" % (where, act))


@gpu
@pytest.mark.parametrize("where,vals", NONFINITE, ids=[w for w, _ in NONFINITE])
@pytest.mark.parametrize("B,Cin,Cout", [(17, 64, 33), (5, "TILE+4", "CT4"), (3, "TILE+4", "CT2"),
                                        (4, 8192, 9), (9, 30, 20)])
def test_linear_non_finite_inputs(where, vals, B, Cin, Cout):
    from sonet_b200 import ops
    sms, optin = device_limits()
    Cin, Cout = resolve(Cin, sms, optin), resolve(Cout, sms, optin)
    g = _gen(B + Cin + Cout)
    x = torch.randn(B, Cin, generator=g)
    W = torch.randn(Cout, Cin, generator=g) * Cin ** -0.5
    shift = torch.randn(Cout, generator=g)
    _poison({"x": x[:-1], "W": W, "shift": shift}[where], g, 2, vals)      # the last row stays finite
    y, m = _elementwise_ref(W, x.t()[None], None, shift)                  # [1, Cout, B]
    y, m = y[0].t(), m[0].t()
    bar = gamma(Cin + 3) * m
    for act in ACTS:
        got = ops.linear(x.to(DEV), W.to(DEV), None, shift.to(DEV), act)
        assert_nonfinite_pattern(got, y, bar, act, "linear %s %s" % (where, act))


# ---- modules under SONET_TC=0: NaN as PyTorch has it -------------------------------------------------
def _nan_masks_match(got, want, what):
    got, want = got.detach().cpu(), want.detach().cpu()
    nan = torch.isnan(want)
    assert bool(nan.any()) and bool((~nan).any()), what
    assert torch.equal(torch.isnan(got), nan), "%s: NaN pattern differs from PyTorch's" % what
    err = float(((got[~nan] - want[~nan]).abs() / want[~nan].abs().clamp(min=1)).max())
    assert err <= 1e-4, "%s: finite entries off by %.3g" % (what, err)


def _seeded(module, seed):
    from sonet_b200 import synth
    module.load_state_dict(synth.synth_state_dict(module, seed=seed))
    return module.eval()


@gpu
@pytest.mark.parametrize("act", ACTS)
def test_modules_propagate_nan_under_fp32_mode(act, monkeypatch):
    from sonet_b200 import layers
    monkeypatch.setenv("SONET_TC", "0")
    g = _gen(17)
    nan = float("nan")
    # EquivariantLayer, thin and wide (both tile configurations)
    for cin, cout, P in ((40, 70, 300), (64, 192, 1100)):
        lay = _seeded(layers.EquivariantLayer(cin, cout, act, "batch"), cin)
        x = torch.randn(2, cin, P, generator=g)
        x[0, 3, 17] = x[1, cin - 1, P - 1] = nan
        with torch.no_grad():
            want = lay(x)
            got = lay.to(DEV)(x.to(DEV))
        _nan_masks_match(got, want, "EquivariantLayer %d->%d %s" % (cin, cout, act))
    # MyLinear
    lin = _seeded(layers.MyLinear(256, 40, act, "batch"), 3)
    x = torch.randn(9, 256, generator=g)
    x[2, 5] = x[7, 255] = nan
    with torch.no_grad():
        want = lin(x)
        got = lin.to(DEV)(x.to(DEV))
    _nan_masks_match(got, want, "MyLinear %s" % act)
    # KNNModule: unfused layers, then the row max over each node's K neighbours
    B, C, M, K = 2, 24, 16, 5
    knn = _seeded(layers.KNNModule(3 + C, (64, 48), act, "batch"), 5)
    coord = torch.randn(B, 3, M, generator=g)
    feat = torch.randn(B, C, M, generator=g)
    feat[0, 4, 6] = feat[1, 0, 15] = nan
    d = ((coord[:, :, :, None] - coord[:, :, None, :]) ** 2).sum(1)
    knn_I = torch.topk(d, K, dim=2, largest=False)[1]
    with torch.no_grad():
        wc, wf = knn(coord, feat, knn_I, K, "avg")
        gc, gf = knn.to(DEV)(coord.to(DEV), feat.to(DEV), knn_I.to(DEV), K, "avg")
    torch.testing.assert_close(gc.cpu(), wc, rtol=1e-6, atol=1e-6)
    _nan_masks_match(gf, wf, "KNNModule %s" % act)


@gpu
def test_encoder_final_max_propagates_nan(monkeypatch):
    """Under SONET_TC=0, with +-inf weights in the final PointNet's last layer, final_pn_out has rows
    that are NaN at some nodes only; the encoder's feature is torch.amax of final_pn_out."""
    from sonet_b200 import networks, synth
    monkeypatch.setenv("SONET_TC", "0")
    B, N = 2, 256
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device=DEV)
    cpu_opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N)
    enc = networks.Encoder(opt).to(DEV)
    enc.load_state_dict(synth.synth_state_dict(networks.Encoder(cpu_opt), seed=4))
    enc.eval()
    # output 100 + r = +-inf * (ReLU output r of the layer before): +-inf where that is positive,
    # NaN (inf * 0) where it is zero
    w = enc.final_pointnet.layers[-1].conv.weight
    with torch.no_grad():
        for r in range(32):
            w[100 + r, r] = float("inf") if r % 2 else float("-inf")
    inp = synth.synth_inputs(B, N, seed=4)
    with torch.no_grad():
        feat = enc(inp["pc"].to(DEV), inp["sn"].to(DEV), inp["node"].to(DEV),
                   inp["node_knn_I"].to(DEV))
    fpo = enc.final_pn_out
    rows = torch.isnan(fpo).any(2) & ~torch.isnan(fpo).all(2)
    assert bool(rows.any()), "no row is NaN at some nodes only"
    torch.testing.assert_close(feat, torch.amax(fpo, dim=2), rtol=0, atol=0, equal_nan=True)
    assert bool(torch.isnan(feat).any()) and bool(torch.isfinite(feat).any())


# ---- a NaN stays in its cloud -------------------------------------------------------------------------
def _snapshot(m):
    enc = m.encoder
    out = {"score": m.score, "feature": m.feature}
    for n in ("som_node", "first_pn_out_masked_max", "knn_center_1", "knn_feature_1", "final_pn_out",
              "feature", "min_idx", "mask", "centers", "x_decentered", "first_pn_out"):
        out["encoder." + n] = getattr(enc, n)
    for n, t in enc._assign.items():
        if t is not None:
            out["encoder._assign." + n] = t
    return {k: v.detach().clone() for k, v in out.items()}


@gpu
@pytest.mark.parametrize("mode", ["default", "fp32"])
def test_nan_point_stays_in_its_cloud(mode, monkeypatch):
    """One NaN coordinate in cloud 0 of a B = 4 eval batch: every output and encoder attribute of
    clouds 1-3 is bit-identical to a clean run (eval only: batch-statistics BN mixes clouds)."""
    from sonet_b200 import classifier, networks, synth
    if mode == "fp32":
        monkeypatch.setenv("SONET_TC", "0")
    B, N = 4, 256
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device=DEV)
    cpu_opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N)
    st_e = synth.synth_state_dict(networks.Encoder(cpu_opt), seed=11)
    st_c = synth.synth_state_dict(networks.Classifier(cpu_opt), seed=12)
    inp = synth.synth_inputs(B, N, seed=11)

    def run(pc):
        m = classifier.Model(opt)
        m.encoder.load_state_dict(st_e)
        m.classifier.load_state_dict(st_c)
        m.set_input(pc, inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
        m.test_model()
        return _snapshot(m)

    clean = run(inp["pc"])
    pc = inp["pc"].clone()
    pc[0, 1, 37] = float("nan")
    dirty = run(pc)
    for k in clean:
        assert torch.equal(dirty[k][1:], clean[k][1:]), k
