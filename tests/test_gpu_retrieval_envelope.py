"""The retrieval kernels (csrc/retrieval.cu) against the numpy restatement of their contract
(tests/retrieval_emu.py, proven against the host entry by test_retrieval_envelope_host.py), bit for
bit in idx, the dist bits, count and label, at the shapes where the kernels' structure changes:

  dims        D around the 64-dim staged chunk (1, 2, 63..65, 127..129, 1023, 1024)
  tiles       a group of n around the 8-query and 128-candidate tiles, k at n - 1, n, n + 1 and at
              1, 2, 4095, 4096 (min(n, k) around the bitonic sort's powers of two), n = 5000
  exits       the k-th key decided by the radix select at shift 24, 16, 8 or 0, and a tie run at the
              k-th value longer than the slots left for it (the lowest positions must be kept)
  specials    identical rows, NaN rows, fp32 differences that overflow, fp64 sums whose rounding
              overflows, +-0 and subnormal features
  groups      Q around the group kernel's 32 warp segments up to 32 * 1024 + 1, L = 1, 2, 4095,
              4096, one label / own labels / even labels / zipf, invalid labels mixed in, and a
              work list longer than the rank kernel's grid
  argmax      the row maximum in every lane residue mod 32, ties across and within lanes, NaN in
              several lanes, -0 / +0 ties

Every query is checked where the restatement is cheap, a seeded subset at the large shapes. Then the
kernel's distances are held to exact arithmetic (test_exact_distance_bar)."""
import numpy as np
import pytest
import torch

import retrieval_emu as emu

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
BUDGET = 2e7


def kernel(f, lab, L, k):
    from sonet_b200 import ops
    out = ops.retrieval_rank(torch.from_numpy(f).to(DEV),
                             None if lab is None else torch.from_numpy(lab).to(DEV),
                             None if lab is None else L, k=k)
    return [t.cpu().numpy() for t in out]


def check(f, lab, L, k, what, seed=0):
    got = kernel(f, lab, L, k)
    qs = emu.pick_queries(f, lab, L, BUDGET, seed)
    emu.assert_equal_rank(got, emu.rank(f, lab, L, k, qs), qs, what)
    return got


@pytest.mark.parametrize("D", emu.DIMS)
def test_dim_chunk(D):
    check(*emu.dim_case(D, seed=D), "D=%d" % D)


@pytest.mark.parametrize("n,k", emu.tile_grid())
def test_tiles(n, k):
    check(*emu.tile_case(n, k, seed=n * 7 + k), "n=%d k=%d" % (n, k))


@pytest.mark.parametrize("kind", emu.EXITS)
def test_select_exits(kind):
    f, lab, L, k, o = emu.exit_case(kind, seed=31)
    assert emu.exit_shift(emu.dist_keys(f[o:o + 1], f)[0], k) == kind
    got = check(f, lab, L, k, "exit %s" % kind)
    assert got[2][o] == k


@pytest.mark.parametrize("kind", emu.EXITS)
def test_select_exits_many_queries(kind):
    """The same layouts for 24 origins at once, one per group, so the select's exit differs between
    the warps of a CTA and between CTAs of the grid."""
    fs, labs = [], []
    for g in range(24):
        f, _, _, k, _ = emu.exit_case(kind, seed=100 + g)
        fs.append(f)
        labs.append(np.full(len(f), g, np.int64))
    perm = np.random.RandomState(7).permutation(sum(len(f) for f in fs))
    f = np.concatenate(fs)[perm]
    lab = np.concatenate(labs)[perm]
    check(f, lab, 24, k, "exits %s x24" % kind)


@pytest.mark.parametrize("kind", emu.SPECIALS)
def test_special_rows(kind):
    check(*emu.special_case(kind, seed=5), kind)


@pytest.mark.parametrize("Q", emu.GROUP_Q)
@pytest.mark.parametrize("pattern,L", emu.GROUP_PATTERNS)
def test_groups(Q, pattern, L):
    f, lab, L, k = emu.group_case(Q, pattern, L, seed=Q + L)
    check(f, lab, L, k, "Q=%d %s L=%d" % (Q, pattern, L), seed=Q)


def test_work_list_longer_than_grid():
    """Small groups enough that the rank kernel's fixed grid (4 CTAs per SM) walks the work list
    several times."""
    Q, L = 32 * 1024 + 1, 4096
    f, lab, L, k = emu.group_case(Q, "own", L, seed=Q + L)
    items = emu.work_items(emu.labels(f, lab, L)[1], L)
    assert items > 4 * 4 * torch.cuda.get_device_properties(0).multi_processor_count
    check(f, lab, L, k, "work list of %d items" % items, seed=1)


@pytest.mark.parametrize("D", emu.ARGMAX_D)
def test_argmax_labels(D):
    check(*emu.argmax_case(D, seed=D), "argmax D=%d" % D)


def test_exact_distance_bar():
    """The kernel's d against the correctly rounded fp32 value of the exact distance of the fp32
    difference vector (integer arithmetic, retrieval_emu.exact_dist_bits), on sampled entries of the
    dim, overflow and subnormal cases. Bar: 1 ulp. The fp64 sum of D <= 1024 exact squares has a
    relative error of at most (D - 1) 2^-53 < 2^-43, its fp64 sqrt at most 2^-44 + 2^-53, so the
    final rounding to fp32 (half an ulp is 2^-24 relative) can only pick the other fp32 neighbour,
    never one further away, and only when the exact value lies within ~2^-44 of a midpoint."""
    worst, total = 0, 0
    for D in emu.DIMS:
        f, lab, L, k = emu.dim_case(D, seed=D)
        idx, dist, count, _ = kernel(f, lab, L, k)
        w, n = emu.ulp_check(f, idx, dist, count, 300 if D < 1000 else 80, seed=D)
        worst, total = max(worst, w), total + n
    for kind in ("inf_round", "tiny", "inf_diff"):
        f, lab, L, k = emu.special_case(kind, seed=5)
        idx, dist, count, _ = kernel(f, lab, L, k)
        w, n = emu.ulp_check(f, idx, dist, count, 400, seed=2)
        worst, total = max(worst, w), total + n
    print("retrieval distance: worst %d ulp over %d sampled entries (bar 1 ulp)" % (worst, total))
    assert total > 2000 and worst <= 1


def test_repeated_calls_are_bit_identical():
    f, lab, L, k, _ = emu.exit_case("tie", seed=3)
    a = kernel(f, lab, L, k)
    for _ in range(2):
        for x, y in zip(a, kernel(f, lab, L, k)):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
