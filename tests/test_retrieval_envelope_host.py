"""The retrieval restatement (tests/retrieval_emu.py) proven against the host entry
sonet_retrieval_rank_cpu_f32 without a GPU, on the same grid the kernel is held to in
test_gpu_retrieval_envelope.py: every dim-chunk edge, every tile edge with k around n, each digit at
which the radix select can stop, tie runs, identical, NaN, overflowing and subnormal rows, the group
kernel's item counts and label patterns, and argmax labels. Then the distances against exact
arithmetic, and the formatter against Python's '%f' over dense sweeps."""
import numpy as np
import pytest
import torch

import retrieval_emu as emu

BUDGET = 2e7        # restatement cost per case (group size x D summed over the checked queries)


def host(f, lab, L, k):
    from sonet_b200 import ops
    out = ops.retrieval_rank(torch.from_numpy(f), None if lab is None else torch.from_numpy(lab),
                             None if lab is None else L, k=k)
    return [t.numpy() for t in out]


def check(f, lab, L, k, what, seed=0):
    got = host(f, lab, L, k)
    qs = emu.pick_queries(f, lab, L, BUDGET, seed)
    emu.assert_equal_rank(got, emu.rank(f, lab, L, k, qs), qs, what)
    return got


@pytest.mark.parametrize("D", emu.DIMS)
def test_restatement_dim_chunk(D):
    check(*emu.dim_case(D, seed=D), "D=%d" % D)


@pytest.mark.parametrize("n,k", emu.tile_grid())
def test_restatement_tiles(n, k):
    check(*emu.tile_case(n, k, seed=n * 7 + k), "n=%d k=%d" % (n, k))


@pytest.mark.parametrize("kind", emu.EXITS)
def test_restatement_select_exits(kind):
    """The builder puts the k-th / (k+1)-th key split of the origin item at the intended digit, and
    the host entry keeps exactly the contract's keys there."""
    f, lab, L, k, o = emu.exit_case(kind, seed=31)
    keys = emu.dist_keys(f[o:o + 1], f)[0]
    assert emu.exit_shift(keys, k) == kind
    got = check(f, lab, L, k, "exit %s" % kind)
    assert got[2][o] == k
    if kind == "tie":
        v = np.sort(keys)[k - 1]
        tied = np.flatnonzero(keys == v)
        taken = got[0][o][got[1][o].view(np.uint32) == v]
        assert len(tied) > len(taken) > 0
        assert np.array_equal(taken, tied[:len(taken)])       # the lowest positions of the run


@pytest.mark.parametrize("kind", emu.SPECIALS)
def test_restatement_special_rows(kind):
    f, lab, L, k = emu.special_case(kind, seed=5)
    got = check(f, lab, L, k, kind)
    g = np.flatnonzero(lab == 1)
    d = got[1][g]
    if kind == "zero":
        assert np.all(d == 0) and np.array_equal(got[0][g[0]], g[:k])
    elif kind == "nan":
        assert np.all(d.view(np.uint32) == emu.NAN_KEY) and np.array_equal(got[0][g[-1]], g[:k])
    elif kind in ("inf_diff", "inf_round"):
        assert np.isinf(d).any()
        if kind == "inf_round":      # a finite fp64 sum whose rounding overflows, and one that fits
            assert (d.view(np.uint32) == 0x7f7fffff).any() or (d > 3e38).any()
    elif kind == "tiny":
        assert ((d > 0) & (d < np.float32(2.0 ** -126))).any()


@pytest.mark.parametrize("Q", emu.GROUP_Q)
@pytest.mark.parametrize("pattern,L", emu.GROUP_PATTERNS)
def test_restatement_groups(Q, pattern, L):
    f, lab, L, k = emu.group_case(Q, pattern, L, seed=Q + L)
    got = check(f, lab, L, k, "Q=%d %s L=%d" % (Q, pattern, L))
    bad = lab < 0
    bad |= lab >= L
    assert np.all(got[2][bad] == -1) and not np.isin(np.flatnonzero(bad), got[0]).any()


@pytest.mark.parametrize("D", emu.ARGMAX_D)
def test_restatement_argmax_labels(D):
    f, lab, L, k = emu.argmax_case(D, seed=D)
    got = check(f, lab, L, k, "argmax D=%d" % D)
    if D >= 32:
        assert got[3][0] % 32 == 0 and len(set(got[3][:32] % 32)) == 32


def test_exact_distance_bar():
    """Every sampled distance is the correctly rounded fp32 value of the exact distance, or 1 ulp
    from it: the fp64 sum of at most 1024 exact squares is within (D - 1) 2^-53 < 2^-43 relative,
    its sqrt within 2^-44 + 2^-53, so the one rounding to fp32 (2^-24) can only land on the other
    neighbour when the exact value is that close to a midpoint. The restatement is held to it here,
    the kernel in test_gpu_retrieval_envelope.py."""
    worst = 0
    for D in emu.DIMS:
        f, lab, L, k = emu.dim_case(D, seed=D)
        idx, dist, count, _ = host(f, lab, L, k)
        w, n = emu.ulp_check(f, idx, dist, count, 200 if D < 1000 else 60, seed=D)
        assert n > 0
        worst = max(worst, w)
    for kind in ("inf_round", "tiny"):
        f, lab, L, k = emu.special_case(kind, seed=5)
        idx, dist, count, _ = host(f, lab, L, k)
        w, n = emu.ulp_check(f, idx, dist, count, 400, seed=1)
        assert n > 0
        worst = max(worst, w)
    assert worst <= 1


def test_exact_reference_rounds_correctly():
    """exact_dist_bits itself: exact cases, a half-way case rounded to even, overflow."""
    one = np.float32([1.0])
    assert emu.exact_dist_bits(np.float32([3, 4]), np.float32([0, 0])) == 0x40a00000
    assert emu.exact_dist_bits(one, one) == 0
    assert emu.exact_dist_bits(np.float32([1e-45]), np.float32([0])) == 1
    # 8192^2 + 16777215^2 = (2^24 + 1)^2: half-way between 2^24 (even) and 2^24 + 2
    assert emu.exact_dist_bits(np.float32([8192, 16777215]), np.float32([0, 0])) == 0x4b800000
    assert emu.exact_dist_bits(np.float32([8192, 16777215]), np.float32([0, 1])) == 0x4b800000
    assert emu.exact_dist_bits(np.float32([3.4e38, 3.4e38]), np.float32([0, 0])) == 0x7f800000
    big = np.float32(np.finfo(np.float32).max)
    assert emu.exact_dist_bits(np.float32([big]), np.float32([0])) == 0x7f7fffff
    assert emu.exact_dist_bits(np.float32([np.inf]), np.float32([0])) is None
    rs = np.random.RandomState(0)
    for _ in range(200):                      # against fp64 where fp64 is exact enough to decide
        a = rs.standard_normal(3).astype(np.float32)
        e = np.float32(np.sqrt((a.astype(np.float64) ** 2).sum()))
        assert abs(emu.exact_dist_bits(a, np.zeros(3, np.float32)) - int(e.view(np.uint32))) <= 1


# ---- the formatter: '%f' % float(d), dense sweeps ----------------------------------------------

def formatted(vals):
    from sonet_b200 import ops
    vals = np.asarray(vals, np.float32)
    k = 1024
    Q = (len(vals) + k - 1) // k
    dist = np.resize(vals, Q * k).reshape(Q, k)
    count = np.full(Q, k, np.int32)
    count[-1] = len(vals) - (Q - 1) * k
    ids = np.arange(Q, dtype=np.int64)
    idx = np.zeros((Q, k), np.int64)
    text, _ = ops.retrieval_format(torch.from_numpy(ids), torch.from_numpy(idx),
                                   torch.from_numpy(dist), torch.from_numpy(count), threads=4)
    lines = text.decode().split("\n")
    assert lines[-1] == ""
    return [ln.split(" ", 1)[1] for ln in lines[:-1]]


def assert_formats(vals):
    vals = np.asarray(vals, np.float32)
    got = formatted(vals)
    want = ["%f" % float(v) for v in vals]
    bad = [i for i in range(len(vals)) if got[i] != want[i]]
    assert not bad, [(float(vals[i]), got[i], want[i]) for i in bad[:5]]


def test_formatter_half_way_sweep():
    """j * 2^-7: every one with an odd j is a half-way case at the 6th decimal (the 7th decimal is
    a 5 followed by nothing), so the rounding must go to even."""
    j = np.arange(0, 6000)
    assert_formats(j * np.float32(2.0 ** -7))
    assert '%f' % (3 * 2.0 ** -7) == "0.023438" and '%f' % (5 * 2.0 ** -7) == "0.039062"


def test_formatter_fine_sweep():
    assert_formats(np.arange(0, 6000) * np.float32(2.0 ** -20))
    assert_formats(np.arange(0, 6000) * np.float32(2.0 ** -20) + np.float32(4095.0))


def test_formatter_random_bits():
    """10^5 seeded bit patterns, every exponent from subnormal to 2^40, a tenth of them negative."""
    rs = np.random.RandomState(1)
    n = 100000
    e = rs.randint(0, 127 + 41, n).astype(np.uint32)
    m = rs.randint(0, 1 << 23, n).astype(np.uint32)
    s = (rs.uniform(size=n) < 0.1).astype(np.uint32)
    vals = ((s << 31) | (e << 23) | m).view(np.float32)
    assert np.isfinite(vals).all() and (e == 0).any() and (e == 127 + 40).any()
    assert_formats(vals)
