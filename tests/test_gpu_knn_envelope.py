"""The fused KNN kernel (csrc/knn_tc.cu) across its envelope: every K from 2 to 16 at the node-block
edges (partial blocks, blocks straddling clouds, blocks spanning many clouds, the module's route
ceiling), its M and K limits, several work items per CTA, operand magnitudes from 2^-14 to 2^14,
saturation, non-finite inputs and out-of-range neighbour ids; in both activations, both precision
modes and both Y layouts, which must agree bit for bit.

Two oracles:
  * exact: a node's K rows are independent wgmma rows and the epilogue act(fmaf(., inv2 > 0,
    shift2)) is monotone, so the K-neighbour result equals, bit for bit, the max over j of K = 2
    runs whose two neighbours are both column j (the max of two equal rows is that row). This pins
    the blocking, padding, pass and key logic with no tolerance;
  * fp64, with the tensor-core bars of test_gpu_knn_tc.py (split) and test_gpu_fp16_mode.py
    (fp16), layer 1's fp32 error carried through layer 2 and saturation at +-131008 (split) or
    +-65504 (fp16).
"""
import pytest
import torch

from helpers import tc_reference
from test_gpu_fp16_mode import F16_C, check, gemm16, r16, w16
from test_gpu_knn_tc import C, DEV, _check, _inputs, _module, _profile, _reference
from test_gpu_knn_tc_sched import _items, _sm_count

pytestmark = pytest.mark.gpu
ACTS = ["relu", "elu"]
MODES = pytest.mark.parametrize("f16", [False, True], ids=["split", "fp16"])
SAT = 131008.0                 # hi and lo of the split each saturate at 65504
# NaN bit patterns with the sign bit clear and set; 0xffffffff's max key is POOL_KEY_INIT itself
NAN_BITS = (0x7fc00000, 0x7fffffff, 0xffc00000 - 2 ** 32, -1)
# The worst case of layer 2's fp32 accumulation in fp16 mode: one truncating ulp (2^-23) of the
# running sum per k16 step, 32 steps. F16_C is calibrated on sums that no few terms dominate; where
# saturated channels (65504 |w|) dominate every partial sum from the first step on, the error
# approaches this bound (2.5e-6 of m measured on one H100 80GB HBM3, 700 W power limit), and it
# replaces F16_C for those cases.
ACC_WORST = 32 * 2.0 ** -23
_WORST = {}


def _nan_bits(n):
    """n NaNs cycling through NAN_BITS, as int32 (written through an int32 view, bits intact)."""
    return torch.tensor([NAN_BITS[i % 4] for i in range(n)], dtype=torch.int32, device=DEV)


def _params(seed, scale=1.0, ch_scale=None, w2_decades=0.0, s2_shift=0.0):
    """The kernel's operands from the folded KNNModule _module(seed), in fp32: w1 = (W1d | shift1)
    [512,4], W2 [512,512], shift2 [512], W2's blob and inverse pre-scale. scale (a power of two)
    multiplies shift1 and shift2; ch_scale [512] multiplies row c of w1; W2's rows are spread over
    w2_decades decades; s2_shift is added to shift2."""
    from sonet_b200 import ops
    mod = _module(seed)
    pk = mod._tc_params()
    w1 = pk["w1"].clone()
    w1[:, 3] *= scale
    if ch_scale is not None:
        w1 *= ch_scale.to(DEV)[:, None]
    W2 = mod.layers[1].folded()[0].detach().clone()
    if w2_decades:
        W2 *= torch.logspace(0, -w2_decades, 512, device=DEV)[:, None]
    blob, inv = ops.knn_mlp_tc_pack(W2)
    return dict(mod=mod, w1=w1.contiguous(), W2=W2, s2=(pk["shift2"] * scale + s2_shift).contiguous(),
                blob=blob.to(DEV), inv=inv)


def _case(B, M, K, seed, center_is_coord=False, kstride=None, yscale=3.0):
    """coord, center [B,3,M] in [-1, 1), neighbour ids [B,M,kstride or K] (column 0 the node
    itself, the rest uniform, so duplicates occur), Y [B,512,M] channel-major."""
    g = torch.Generator(DEV).manual_seed(seed)
    coord = torch.rand(B, 3, M, device=DEV, generator=g) * 2 - 1
    center = coord if center_is_coord else torch.rand(B, 3, M, device=DEV, generator=g) * 2 - 1
    idx = torch.randint(0, M, (B, M, kstride or K), device=DEV, generator=g)
    idx[:, :, 0] = torch.arange(M, device=DEV)
    Y = torch.randn(B, 512, M, device=DEV, generator=g) * yscale
    return coord, center, idx, Y


def _same(a, b):
    """torch.equal, with NaN equal to NaN."""
    n = torch.isnan(a)
    return torch.equal(n, torch.isnan(b)) and torch.equal(a.masked_fill(n, 0), b.masked_fill(n, 0))


def _run(p, coord, center, idx, K, y, act, f16):
    from sonet_b200 import ops
    return ops.knn_mlp_tc(coord, center, idx, K, y, p["w1"], p["blob"], p["inv"], p["s2"], f16=f16,
                          act=act)


def _both_layouts(p, coord, center, idx, K, Y, act, f16):
    """The kernel on node-major Y (the module's layout) and on channel-major Y: the same bits.
    Returns (output, node-major Y)."""
    ynm = Y.transpose(1, 2).contiguous().transpose(1, 2)
    out = _run(p, coord, center, idx, K, ynm, act, f16)
    assert _same(out, _run(p, coord, center, idx, K, Y.contiguous(), act, f16)), \
        "node-major and channel-major Y differ"
    return out, ynm


def _exact(p, coord, center, idx, K, y, act, f16, out, what):
    """out == max over j of the K = 2 run whose neighbours are both column j, bit for bit."""
    B, M = idx.shape[:2]
    rows = [_run(p, coord, center, idx[:, :, j:j + 1].expand(B, M, 2).contiguous(), 2, y, act, f16)
            for j in range(K)]
    assert _same(out, torch.stack(rows).max(0)[0]), "%s: not the max of its rows run alone" % what


def _act64(z, act):
    return z.clamp(min=0) if act == "relu" else torch.where(z > 0, z, torch.expm1(z))


def _fp64(p, coord, center, idx, K, Y, act, f16, dominated=False):
    """fp64 knn_feature of the nodes of center [B,3,M'] and idx [B,M',K'] (ids into coord and Y,
    clamped to [0, M-1] as the kernel does) and its bar: (y, bar) in split mode, (y, m) for
    test_gpu_fp16_mode.check in fp16 mode.

    Layer 1: the fp32 epilogue's error e1 (4 roundings of at most 2^-24 of the magnitudes, as
    test_gpu_knn_tc._reference; expm1f's ulp under ELU) is carried through the activation and the
    saturation of layer 2's input (+-131008 split, rn16sat fp16) as the interval it can move h1 by;
    an input that is already +-inf moves nothing. Layer 2: split, the tensor-core bar plus the
    saturated lo term of test_gpu_tc_envelope.py (2^-11 |W2| lo(h1)); fp16, gemm16 with F16_C.
    dominated: in fp16 mode, the accumulation bar is ACC_WORST instead of F16_C.
    ReLU, ELU and the max over K are 1-Lipschitz."""
    B, Mq = idx.shape[:2]
    M = coord.shape[2]
    nb = idx[:, :, :K].clamp(0, M - 1)
    bi = torch.arange(B, device=DEV)[:, None, None]
    dec = torch.stack([coord[:, c][bi, nb] - center[:, c][:, :, None] for c in range(3)], 1)
    dec = dec.double().reshape(B, 3, Mq * K)                       # fp32 differences, as __fsub_rn
    yg = Y.transpose(1, 2)[bi, nb].double().reshape(B, Mq * K, 512).transpose(1, 2)
    w1 = p["w1"].double()
    pre = torch.einsum("oc,bcp->bop", w1[:, :3], dec) + yg + w1[:, 3, None]
    mag = torch.einsum("oc,bcp->bop", w1[:, :3].abs(), dec.abs()) + yg.abs() + w1[:, 3, None].abs()
    e1 = 4 * 2.0 ** -24 * (mag + yg.abs())
    e1 = torch.where(torch.isfinite(e1), e1, torch.zeros_like(e1))
    h1 = _act64(pre, act)
    ulp = torch.where(h1 < 0, 2.0 ** -23 * h1.abs(), torch.zeros_like(h1)) if act == "elu" else 0.0
    sat = r16 if f16 else (lambda t: t.clamp(-SAT, SAT))
    hs = sat(h1)
    eh = torch.maximum((sat(_act64(pre + e1, act) + ulp) - hs).abs(),
                       (sat(_act64(pre - e1, act) - ulp) - hs).abs())
    s2 = p["s2"].double()[None, :, None]
    if f16:
        W16 = w16(p["W2"], p["inv"])
        y2, m = gemm16(W16, p["inv"], hs)
        y2, m = y2 + s2, m + s2.abs()
        bar = m * (ACC_WORST / F16_C if dominated else 1.0) \
            + torch.einsum("ok,bkp->bop", W16.abs(), eh) * p["inv"] / F16_C
    else:
        y2, bar = tc_reference(p["W2"], hs, shift=p["s2"], w_scale=1.0 / p["inv"])
        lo = (hs.abs() - 65504.0).clamp(min=0)
        bar = bar + torch.einsum("ok,bkp->bop", p["W2"].double().abs(), 2.0 ** -11 * lo + eh)
    out = _act64(y2, act).view(B, 512, Mq, K).amax(3)
    bar = bar.view(B, 512, Mq, K).amax(3)
    if act == "elu":                                                # the output's expm1f
        ulp = torch.where(out < 0, 2.0 ** -23 * out.abs(), torch.zeros_like(out))
        bar = bar + ulp / (F16_C if f16 else 1.0)
    return out, bar


def _verify(got, ref, f16, group, what):
    """got within the fp64 bar; records the worst error in bar units per group."""
    y, b = ref
    u = float(((got.double() - y).abs() / ((F16_C if f16 else 1.0) * b).clamp(min=1e-300)).max())
    key = "%s, %s" % (group, "fp16" if f16 else "split")
    _WORST[key] = max(_WORST.get(key, 0.0), u)
    if f16:
        check(got, y, b, what)
    else:
        _check(got, y, b, what)


def _both_oracles(p, coord, center, idx, K, Y, act, f16, group, what, dominated=False):
    out, ynm = _both_layouts(p, coord, center, idx, K, Y, act, f16)
    _exact(p, coord, center, idx, K, ynm, act, f16, out, what)
    _verify(out, _fp64(p, coord, center, idx, K, Y, act, f16, dominated), f16, group, what)
    return out


# ---- every K at the node-block edges ---------------------------------------------------------------
@MODES
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("K", range(2, 17))
def test_every_k(K, act, f16):
    """A warpgroup owns npb = 64 // K whole nodes, so 64 % K of its rows are padding (12 at
    K = 13). Shapes: B*M not a multiple of npb; every block straddling two clouds; M = 1 (and
    M = 5 at K = 2), so one block spans many clouds; the module's route ceiling M = 2304 // K."""
    npb = 64 // K
    shapes = [(3, 2 * npb + 1), (npb, npb + 1), (7, 1), (2, 2304 // K)] + ([(9, 5)] if K == 2 else [])
    p = _params(K)
    for B, M in shapes:
        coord, center, idx, Y = _case(B, M, K, seed=1000 * K + 10 * B + M, center_is_coord=True)
        what = "K=%d B=%d M=%d %s %s" % (K, B, M, act, "fp16" if f16 else "split")
        out = _both_oracles(p, coord, center, idx, K, Y, act, f16, "every K", what)
        if act == "relu" and not f16:
            _, f_ref, f_bar = _reference(p["mod"], coord, None, idx, K, "center", y_exact=Y)
            _check(out, f_ref, f_bar, what + " (_reference)")


# ---- the kernel's limits ------------------------------------------------------------------------------
@MODES
@pytest.mark.parametrize("act", ACTS)
def test_largest_m(act, f16):
    """M = 65535, one cloud, K = 2: the exact oracle everywhere, fp64 on 2050 nodes (first and
    last among them)."""
    B, M, K = 1, 65535, 2
    p = _params(21)
    coord, center, idx, Y = _case(B, M, K, seed=21)
    out, ynm = _both_layouts(p, coord, center, idx, K, Y, act, f16)
    what = "M=65535 %s %s" % (act, "fp16" if f16 else "split")
    _exact(p, coord, center, idx, K, ynm, act, f16, out, what)
    sel = torch.cat((torch.tensor([0, M - 1]),
                     torch.randperm(M, generator=torch.Generator().manual_seed(21))[:2048])).to(DEV)
    ref = _fp64(p, coord, center[:, :, sel], idx[:, sel], K, Y, act, f16)
    _verify(out[:, :, sel], ref, f16, "M = 65535", what)


def test_rejects_beyond_limits_and_empty_batch():
    """M = 65536 and K outside [2, 16] raise before any launch; B = 0 is a no-op."""
    p = _params(22)
    for M, K, msg in ((65536, 2, "too large"), (40, 1, "out of range"), (40, 17, "out of range")):
        coord, center, idx, Y = _case(1, M, K, seed=M + K)
        with pytest.raises(RuntimeError, match=msg):
            _run(p, coord, center, idx, K, Y, "relu", False)
    coord, center, idx, Y = _case(0, 40, 9, seed=0)
    for act in ACTS:
        for f16 in (False, True):
            assert _run(p, coord, center, idx, 9, Y, act, f16).shape == (0, 512, 40)


# ---- several items per CTA: the keys are reset between them --------------------------------------
@MODES
@pytest.mark.parametrize("act", ACTS)
def test_key_reset_between_items(act, f16):
    """>= 3 items per CTA (item i + grid runs on the CTA of item i). The clouds inside the first
    round get a large positive spike in Y, so maxima a missed key reset carried over would show in
    every later item."""
    K, M = 9, 200
    npb, sm = 64 // K, _sm_count()
    B = 3 * sm * npb // M + 2
    items = _items(B, M, K)
    assert items >= 3 * sm
    spiked = min(items, sm) * npb // M                  # whole clouds of the first round
    assert spiked >= 1
    p = _params(31)
    coord, center, idx, Y = _case(B, M, K, seed=31)
    Y[:spiked] += 1000.0
    _both_oracles(p, coord, center, idx, K, Y, act, f16, "rounds",
                  "rounds B=%d %s %s" % (B, act, "fp16" if f16 else "split"))


# ---- magnitudes --------------------------------------------------------------------------------------
@MODES
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("e", [-14, -8, 0, 8, 14])
def test_operand_scale(e, act, f16):
    """Y, coordinates, centres, shift1 and shift2 scaled together by 2^e (a ReLU module's output
    scales with them): at 2^-14 the split's subnormal floor rules, at 2^14 h1 nears 65504."""
    s = 2.0 ** e
    B, M, K = 3, 50, 9
    p = _params(7, scale=s)
    coord, center, idx, Y = _case(B, M, K, seed=70, yscale=0.5)
    Y = Y.clamp(-1.5, 1.5) * s
    _both_oracles(p, coord * s, center * s, idx, K, Y, act, f16, "scale 2^e",
                  "scale 2^%d %s %s" % (e, act, "fp16" if f16 else "split"))


@MODES
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("kind", ["channel-scales", "w2-rows"])
def test_mixed_scales(kind, act, f16):
    """channel-scales: layer 1's channels (Y and w1's row) each scaled by 2^-14 .. 2^14;
    w2-rows: W2's rows spread over 4 decades under one power-of-two pre-scale (pow2_scale, inv2:
    the weight-side floor of the bar)."""
    B, M, K = 2, 60, 11
    coord, center, idx, Y = _case(B, M, K, seed=80, yscale=0.5)
    if kind == "channel-scales":
        g = torch.Generator().manual_seed(8)
        ch = torch.pow(2.0, torch.randint(-14, 15, (512,), generator=g).float())
        p = _params(8, ch_scale=ch)
        Y = Y.clamp(-1.5, 1.5) * ch.to(DEV)[None, :, None]
    else:
        p = _params(9, w2_decades=4.0)
    _both_oracles(p, coord, center, idx, K, Y, act, f16, kind,
                  "%s %s %s" % (kind, act, "fp16" if f16 else "split"))


@MODES
@pytest.mark.parametrize("act", ACTS)
def test_saturation(act, f16):
    """Y channels at 65520 (rn16 would round it to inf), 131008, 1e6, -3e38, +inf and -inf: layer 1
    saturates at +-131008 (split) or +-65504 (fp16) before layer 2, -inf gives h1 = 0 under ReLU
    and -1 under ELU, and every output is finite."""
    B, M, K = 2, 90, 7
    p = _params(41)
    coord, center, idx, Y = _case(B, M, K, seed=41)
    for c, v in ((5, 65520.0), (9, SAT), (11, 1e6), (17, -3e38), (23, float("inf")), (31, float("-inf"))):
        Y[:, c] = v
    Y[:, 40, ::3] = float("inf")
    Y[:, 41, 1::3] = float("-inf")
    out = _both_oracles(p, coord, center, idx, K, Y, act, f16, "saturation",
                        "saturation %s %s" % (act, "fp16" if f16 else "split"), dominated=True)
    assert bool(torch.isfinite(out).all())


@MODES
def test_elu_negative_dominant(f16):
    """shift2 lowered until most node maxima are below 0: ELU's negative branch after the max."""
    B, M, K = 3, 80, 6
    coord, center, idx, Y = _case(B, M, K, seed=51)
    y0, _ = _fp64(_params(51), coord, center, idx, K, Y, "elu", False)
    z = torch.where(y0 > 0, y0, torch.log1p(y0))                  # the maxima before ELU
    p = _params(51, s2_shift=-float(torch.quantile(z.flatten(), 0.6)))
    out = _both_oracles(p, coord, center, idx, K, Y, "elu", f16, "ELU negative",
                        "ELU negative %s" % ("fp16" if f16 else "split"))
    share = float((out < 0).double().mean())
    assert share >= 0.3, "only %.2f of the outputs are negative" % share


# ---- non-finite inputs -------------------------------------------------------------------------------
@MODES
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("where", ["Y-nan", "Y-inf", "coord-nan", "coord-inf", "center-nan",
                                   "center-inf", "Y-node-0"])
def test_non_finite(where, act, f16):
    """NaN and +-inf in Y at four neighbour nodes of cloud 2, in their coordinates, or in four nodes'
    centres. K = 13 (12 padding rows per warpgroup) over > 2 items per CTA. Only the nodes that
    gather a bad value (or own the bad centre) change: every other node, cloud, later item on the
    same CTA, and (Y-node-0: NaN and inf in Y node (0, 0), which padding rows read and no node
    gathers) everything, is bit-identical to the clean run.
    The rule: under ELU a NaN in any of a node's rows makes the node NaN in all 512 channels,
    whatever the NaN's sign bit; under ReLU layer 1 maps a NaN to 0, which is what -inf in the
    same place gives. +-inf saturates: the result is finite and inside the fp64 bar."""
    B, M, K = 6, 200, 13
    assert _items(B, M, K) > 2 * _sm_count()
    p = _params(13)
    coord, center, idx, Y = _case(B, M, K, seed=13)
    idx[0] = idx[0].clamp(min=1)                        # nobody gathers node (0, 0)
    clean, _ = _both_layouts(p, coord, center, idx, K, Y, act, f16)
    b0, ns = 2, [3, 50, 101, 160]
    coord2, center2, Y2 = coord.clone(), center.clone(), Y.clone()
    inf = float("inf")
    hit = torch.zeros(B, M, dtype=torch.bool, device=DEV)
    gathers = torch.isin(idx[b0, :, :K], torch.tensor(ns, device=DEV)).any(1)
    if where == "Y-nan":
        for i, n in enumerate(ns):
            Y2.view(torch.int32)[b0, 7::64, n] = NAN_BITS[i]
        hit[b0] = gathers
    elif where == "Y-inf":
        Y2[b0, 7::64, ns[0]] = inf
        Y2[b0, 7::64, ns[1]] = -inf
        Y2[b0, 7::128, ns[2]] = inf
        Y2[b0, 71::128, ns[2]] = -inf
        Y2[b0, :, ns[3]] = -inf
        hit[b0] = gathers
    elif where == "coord-nan":
        for i, n in enumerate(ns):
            coord2.view(torch.int32)[b0, i % 3, n] = NAN_BITS[i]
        hit[b0] = gathers
    elif where == "coord-inf":
        for i, n in enumerate(ns):
            coord2[b0, i % 3, n] = inf if i % 2 else -inf
        hit[b0] = gathers
    elif where == "center-nan":
        for i, n in enumerate(ns):
            center2.view(torch.int32)[b0, i % 3, n] = NAN_BITS[i]
        hit[b0, ns] = True
    elif where == "center-inf":
        for i, n in enumerate(ns):
            center2[b0, i % 3, n] = inf if i % 2 else -inf
        hit[b0, ns] = True
    else:
        Y2.view(torch.int32)[0, ::4, 0] = _nan_bits(128)
        Y2[0, 1::4, 0] = inf
        Y2[0, 2::4, 0] = -inf
    what = "%s %s %s" % (where, act, "fp16" if f16 else "split")
    out, ynm = _both_layouts(p, coord2, center2, idx, K, Y2, act, f16)
    assert bool(hit.any()) == (where != "Y-node-0")
    keep = ~hit[:, None, :].expand_as(out)
    assert _same(out[keep], clean[keep]), "%s: a node that gathers no bad value changed" % what
    _exact(p, coord2, center2, idx, K, ynm, act, f16, out, what)
    bad = hit[:, None, :].expand_as(out)
    if where.endswith("inf"):
        assert bool(torch.isfinite(out).all()), what
        _verify(out, _fp64(p, coord2, center2, idx, K, Y2, act, f16, dominated=True), f16, "+-inf",
                what)
    elif where.endswith("nan") and act == "elu":
        assert bool(torch.isnan(out[bad]).all()), "%s: a node with a NaN row is not NaN" % what
    elif where == "center-nan":                          # ReLU: every h1 of the node is 0
        want = p["s2"].clamp(min=0)[None, :, None].expand_as(out)
        assert torch.equal(out[bad], want[bad]), what
    elif where.endswith("nan"):                          # ReLU: the NaN acts as -inf
        Y3 = Y2.masked_fill(torch.isnan(Y2), -inf)
        if where == "coord-nan":
            Y3, coord2 = Y.clone(), coord
            Y3[b0, :, ns] = -inf
        ref, _ = _both_layouts(p, coord2, center2, idx, K, Y3, act, f16)
        assert torch.equal(out, ref), "%s: NaN does not act as -inf" % what
        _verify(ref, _fp64(p, coord2, center2, idx, K, Y3, act, f16), f16, "+-inf", what + " as -inf")
    else:
        assert _same(out, clean), "%s: a padding row reached the output" % what


# ---- neighbour ids -----------------------------------------------------------------------------------
@MODES
@pytest.mark.parametrize("act", ACTS)
def test_neighbour_ids(act, f16):
    """Duplicate neighbours and the node itself twice (both oracles); ids -1, M, 2^40 and -2^40
    give the bits of the clamped ids; garbage in columns K..Kstride-1 is never read."""
    B, M, K, S = 3, 37, 5, 8
    p = _params(5)
    coord, center, idx, Y = _case(B, M, K, seed=55, kstride=S)
    idx[:, :, 1] = idx[:, :, 2]
    idx[:, ::3, 3] = torch.arange(0, M, 3, device=DEV)
    base = idx[:, :, :K].contiguous()
    what = "ids %s %s" % (act, "fp16" if f16 else "split")
    out = _both_oracles(p, coord, center, base, K, Y, act, f16, "ids", what)
    wide = idx.clone()
    wide[:, :, K:] = torch.randint(-2 ** 62, 2 ** 62, (B, M, S - K), device=DEV)
    assert torch.equal(_run(p, coord, center, wide, K, Y, act, f16), out), what + ": Kstride > K"
    odd = base.clone()
    odd[:, 0::4, 1] = -1
    odd[:, 1::4, 2] = M
    odd[:, 2::4, 3] = 2 ** 40
    odd[:, 3::4, 4] = -2 ** 40
    got = _run(p, coord, center, odd, K, Y, act, f16)
    assert torch.equal(got, _run(p, coord, center, odd.clamp(0, M - 1), K, Y, act, f16)), what


# ---- the module's routes at their boundaries ------------------------------------------------------
@pytest.mark.parametrize("K", [2, 13, 16])
def test_forward_route_boundary(K):
    """KNNModule.forward fuses up to M*K = 2304 and falls back to the layer stack + rowmax just
    above; at the last fused M the fallback route on the same inputs agrees within the fp64 bar."""
    from sonet_b200 import ops
    top = 2304 // K
    for M in (top, top + 1):
        mod = _module(K + M)
        coord, x, knn_I = _inputs(1, M, K, seed=M)
        (_, feat), names = _profile(lambda: mod(coord, x, knn_I, K, "center"))
        fused = M == top
        assert mod._tc_fused(K, M) == fused
        assert ("sonet_knn_mlp_tc_forward" in names) == fused, names
        assert ("sonet_rowmax_f32" in names) != fused, names
        _, f_ref, f_bar = _reference(mod, coord, x, knn_I, K, "center")
        _check(feat, f_ref, f_bar if fused else 2 * f_bar, "forward M=%d K=%d" % (M, K))
        if fused:
            _, h = ops.knn_assemble(coord, x.contiguous(), knn_I, K, "center")
            _check(mod._layers_max(h, 1, M, K), f_ref, 2 * f_bar, "fallback M=%d K=%d" % (M, K))


@pytest.mark.parametrize("K", [2, 9])
def test_forward_pooled_route_boundary(K):
    """forward_pooled fuses at M = 256 and returns None (before any launch) at M = 257."""
    for M in (256, 257):
        mod = _module(M + K)
        coord, x, knn_I = _inputs(2, M, K, seed=M * K)
        bits = x.view(torch.int32)
        keys = (bits ^ ((bits >> 31) & 0x7fffffff)).contiguous()
        p0 = (torch.rand(2, C, device=DEV) * 2).contiguous()
        res, names = _profile(lambda: mod.forward_pooled(coord, (keys, p0), knn_I, K, "center"))
        if M == 257:
            assert res is None and names == [], names
            continue
        _, feat, mm = res
        assert "sonet_knn_mlp_tc_forward" in names, names
        assert torch.equal(mm, x)
        _, f_ref, f_bar = _reference(mod, coord, x, knn_I, K, "center")
        _check(feat, f_ref, f_bar, "forward_pooled M=%d K=%d" % (M, K))


@pytest.mark.parametrize("act", ACTS)
def test_module_nan_feature_fused_and_unfused(act):
    """A NaN in one node's feature at module level. The fused route's per-node Y comes from a bare
    generic layer, whose epilogue turns the NaN into -inf in all 512 channels, so the rows that
    gather the node see h1 = act(-inf) (0 under ReLU, -1 under ELU) and the output stays finite.
    The unfused route (layer stack + rowmax) carries the NaN through ELU to every channel of those
    nodes; under ReLU its first layer maps it to 0. Other nodes keep their bits on both routes."""
    from sonet_b200 import ops
    from sonet_b200.layers import KNNModule
    B, M, K, n = 2, 64, 9, 10
    mod = _module(61)
    if act == "elu":
        elu = KNNModule(3 + C, (512, 512), "elu", "batch").to(DEV).eval()
        elu.load_state_dict(mod.state_dict())
        mod = elu
    coord, x, knn_I = _inputs(B, M, K, seed=61)
    dirty = x.clone()
    dirty[1, 5, n] = float("nan")
    runs = {}
    for name, xx in (("clean", x), ("dirty", dirty)):
        (_, fused), names = _profile(lambda: mod(coord, xx, knn_I, K, "center"))
        assert any(s.startswith("sonet_knn_mlp_tc_forward") for s in names), names
        _, h = ops.knn_assemble(coord, xx.contiguous(), knn_I, K, "center")
        runs[name] = (fused, mod._layers_max(h, B, M, K))
    hit = torch.zeros(B, 1, M, dtype=torch.bool, device=DEV)
    hit[1, 0] = (knn_I[1, :, :K] == n).any(1)
    keep, bad = (~hit).expand(B, 512, M), hit.expand(B, 512, M)
    for i, route in enumerate(("fused", "unfused")):
        assert torch.equal(runs["dirty"][i][keep], runs["clean"][i][keep]), route
    assert bool(torch.isfinite(runs["dirty"][0]).all())
    unfused = runs["dirty"][1]
    if act == "elu":
        assert bool(torch.isnan(unfused[bad]).all())
    else:
        assert bool(torch.isfinite(unfused).all())


def test_report_worst_bar_units():
    """Last in the file: the worst error of each group in units of its bar."""
    for k in sorted(_WORST):
        print("\n[knn envelope] %-28s %.3f bar units" % (k, _WORST[k]))
