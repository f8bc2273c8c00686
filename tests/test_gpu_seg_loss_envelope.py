"""The segmentation loss kernel (csrc/seg_loss.cu: per-point log-softmax NLL, fp64 reduction)
against F.cross_entropy in fp64 and a numpy fp64 log-sum-exp restatement of the per-point term, at N around
the 256-thread block, B up to the 65535 grid limit, C from 1 to 1000, logits spread to +-1e30 or
packed a few ulp apart near +-1e6, non-finite scores, ignored and out-of-range targets.

Bar. Per point the kernel computes, in fp32, m = max_c s_c, e_c = expf(fl(s_c - m)), the
sequential sum S of the e_c, then l = fl(fl(s_t - m) - logf(S)) negated. With u = 2^-24 and
g(n) = n u / (1 - n u):
  - rounding s_c - m moves e_c by |s_c - m| u relative; weighted by e_c / S this adds at most
    C u / e to the relative error of S (x e^-x <= 1/e, and S >= 1);
  - expf is within 2 ulp (4 u relative) of exp, the sum of C positive terms within g(C - 1);
    so S is within g(2C + 3) relative, and log S within g(2C + 4) absolute plus logf's 1 ulp
    (2 u log S);
  - fl(s_t - m) and the last subtraction add u |s_t - m| and u (|s_t - m| + log S).
So per point  |l - l_exact| <= bar_i = g(2C + 8) (1 + |s_t - m| + log S).
The reduction runs in fp64 (2^-52 P sum |l_i| for P points) and rounds once to fp32, so
  |loss - exact| <= (sum_i bar_i + 2^-52 P sum_i |l_i|) / count + ulp32(exact).
Every case reports its error as a fraction of that bar."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
U = 2.0 ** -24
WORST = []          # (fraction of the bar, case) of every finite comparison, for the report


def gamma(n):
    return n * U / (1 - n * U)


def restated(score, target):
    """numpy fp64 per-point terms l_i [B,N] (NaN for an out-of-range target), their bars, and the
    mask of counted points."""
    s = score.astype(np.float64)
    B, C, N = s.shape
    t = target.astype(np.int64)
    counted = t != -100
    ok = (t >= 0) & (t < C)
    with np.errstate(all="ignore"):
        m = s.max(1)
        S = np.exp(s - m[:, None, :]).sum(1)
        st = np.take_along_axis(s, np.clip(t, 0, C - 1)[:, None, :], 1)[:, 0, :]
        ell = np.log(S) - (st - m)
        ell = np.where(ok, ell, np.nan)
        bar = gamma(2 * C + 8) * (1.0 + np.abs(st - m) + np.log(S))
    return ell, bar, counted


def check(score, target, what, reductions=(True, False)):
    """Kernel vs fp64 torch (and the restatement) for both reductions; returns the losses."""
    from sonet_b200 import ops
    sc, tg = torch.from_numpy(score).to(DEV), torch.from_numpy(target).to(DEV)
    ell, bar, counted = restated(score, target)
    out = []
    for avg in reductions:
        got = float(ops.seg_loss(sc, tg, size_average=avg))
        cnt = int(counted.sum())
        if (target[counted] >= 0).all() and (target[counted] < score.shape[1]).all():
            want = float(F.cross_entropy(sc.double(), tg, reduction="mean" if avg else "sum"))
        else:
            want = float("nan")             # torch raises on such targets; the kernel says NaN
        tot = float(ell[counted].sum()) if cnt else 0.0
        mine = (tot / cnt if cnt else float("nan")) if avg else tot
        if not np.isfinite(want):
            assert np.isnan(want) == np.isnan(got) and (np.isnan(want) or got == want), \
                (what, avg, got, want)
            assert np.isnan(mine) == np.isnan(want) and (np.isnan(mine) or mine == want)
        else:
            P = ell.size
            e = bar[counted].sum() + 2.0 ** -52 * P * np.abs(ell[counted]).sum()
            e = e / (cnt if avg else 1) + float(np.spacing(np.float32(abs(want))))
            assert abs(mine - want) <= 1e-12 * max(1.0, abs(want)), (what, mine, want)
            frac = abs(got - want) / e
            WORST.append((frac, "%s %s" % (what, "mean" if avg else "sum")))
            assert frac <= 1.0, "%s: |%r - %r| is %.3g x the bar" % (what, got, want, frac)
        out.append(got)
    return out


def normal_case(B, C, N, seed, scale=4.0):
    rs = np.random.RandomState(seed)
    score = (rs.standard_normal((B, C, N)) * scale).astype(np.float32)
    target = rs.randint(0, C, (B, N)).astype(np.int64)
    return score, target


@pytest.mark.parametrize("N", (1, 255, 256, 257, 4097))
@pytest.mark.parametrize("C", (1, 2, 50, 1000))
@pytest.mark.parametrize("B", (1, 7))
def test_shapes(B, C, N):
    check(*normal_case(B, C, N, seed=B * 10007 + C * 31 + N), "B=%d C=%d N=%d" % (B, C, N))


@pytest.mark.parametrize("C,N", ((2, 257), (1, 3), (50, 1)))
def test_grid_limit_batch(C, N):
    check(*normal_case(65535, C, N, seed=C + N), "B=65535 C=%d N=%d" % (C, N))


def test_batch_beyond_grid_is_rejected_before_launch():
    from sonet_b200 import _C
    lib = _C.lib()
    score = torch.zeros(65536, 1, 1, device=DEV)
    target = torch.zeros(65536, 1, dtype=torch.int64, device=DEV)
    scratch = torch.empty(int(lib.sonet_seg_loss_scratch_bytes(65536, 1)), dtype=torch.uint8,
                          device=DEV)
    loss = torch.full((), 12345.0, device=DEV)
    rc = lib.sonet_seg_loss_f32(score.data_ptr(), target.data_ptr(), 65536, 1, 1, 1,
                                scratch.data_ptr(), loss.data_ptr(), None)
    assert rc == -1 and "65536" in _C.last_error()
    torch.cuda.synchronize()
    assert float(loss) == 12345.0
    from sonet_b200 import ops
    with pytest.raises(RuntimeError):
        ops.seg_loss(score, target)


@pytest.mark.parametrize("C", (2, 50, 1000))
def test_spread_to_1e30(C):
    rs = np.random.RandomState(C)
    B, N = 3, 300
    score = (rs.uniform(-1, 1, (B, C, N)) * 10.0 ** rs.uniform(0, 30, (B, C, N))).astype(np.float32)
    target = rs.randint(0, C, (B, N)).astype(np.int64)
    check(score, target, "spread 1e30 C=%d" % C)


@pytest.mark.parametrize("sign", (1, -1))
@pytest.mark.parametrize("C", (2, 50, 1000))
def test_packed_near_1e6(sign, C):
    """All logits within a few ulp (0.0625) of +-1e6: the max must be taken before any exp."""
    rs = np.random.RandomState(C + (sign > 0))
    B, N = 2, 257
    base = np.float32(sign * 1e6)
    score = (base + np.float32(0.0625) * rs.randint(-4, 5, (B, C, N))).astype(np.float32)
    target = rs.randint(0, C, (B, N)).astype(np.int64)
    check(score, target, "near %+.0e C=%d" % (sign * 1e6, C))


def test_one_point_dominates():
    """One point's loss is ~1e4 times every other's."""
    score, target = normal_case(2, 50, 300, seed=3, scale=1.0)
    ell, _, _ = restated(score, target)
    score[1, target[1, 17], 17] -= np.float32(1e5)
    ell2, _, _ = restated(score, target)
    assert ell2[1, 17] > 1e4 * np.median(ell)
    check(score, target, "one dominant point")


@pytest.mark.parametrize("kind", ("ninf_other", "ninf_target", "ninf_all", "pinf_other",
                                  "pinf_target", "nan_other", "nan_target"))
def test_non_finite_scores(kind):
    """One point (a column of its block's last warp) carries the non-finite score; the result must
    follow fp64 torch in both reductions."""
    score, target = normal_case(2, 5, 300, seed=11)
    b, n = 1, 250
    t = target[b, n]
    other = (t + 2) % 5
    v = {"ninf": -np.inf, "pinf": np.inf, "nan": np.nan}[kind.split("_")[0]]
    if kind.endswith("_all"):
        score[b, :, n] = v
    else:
        score[b, t if kind.endswith("target") else other, n] = v
    got = check(score, target, kind)
    if kind == "ninf_other":
        assert np.isfinite(got).all()
    elif kind == "ninf_target":
        assert got == [np.inf, np.inf]
    else:
        assert np.isnan(got).all()


def test_ignored_targets():
    score, target = normal_case(3, 50, 257, seed=5)
    allign = np.full_like(target, -100)
    mean, total = check(score, allign, "all ignored")
    assert np.isnan(mean) and total == 0.0
    third = target.copy()
    third[:, ::3] = -100
    check(score, third, "every third ignored")
    third[:, 1::3] = -100
    third[0, 256] = 7                                  # one counted point, at a block's last lane
    check(score, third, "one counted point")


@pytest.mark.parametrize("bad", (-1, 50, 1 << 40))
def test_out_of_range_targets_give_nan(bad):
    score, target = normal_case(2, 50, 257, seed=6)
    target[1, 200] = bad
    mean, total = check(score, target, "target %d" % bad)
    assert np.isnan(mean) and np.isnan(total)


def test_repeated_calls_are_bit_identical():
    from sonet_b200 import ops
    score, target = normal_case(7, 1000, 4097, seed=9)
    sc, tg = torch.from_numpy(score).to(DEV), torch.from_numpy(target).to(DEV)
    for avg in (True, False):
        a = ops.seg_loss(sc, tg, size_average=avg)
        for _ in range(3):
            assert torch.equal(ops.seg_loss(sc, tg, size_average=avg).view(torch.int32),
                               a.view(torch.int32))


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    """After the module: the largest error of its finite comparisons, as a fraction of the bar."""
    yield
    if WORST:
        frac, what = max(WORST)
        print("\nseg_loss: worst %.3g of the bar (%s) over %d comparisons" % (frac, what, len(WORST)))
