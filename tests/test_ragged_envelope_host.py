"""The numpy restatements of the ragged encoder's kernels (tests/ragged_emu.py) without a GPU: the
vectorised group against the loop version bit for bit, the offsets clamp on hand-built malformed
arrays, index_max_ragged against pool_ref cloud by cloud, and the stacked-order decentring against
the sorted one."""
import numpy as np
import pytest

import ragged_emu
from test_gpu_pool_envelope import pool_ref


def _clouds(sizes, M, seed, scale=1.0, centre=0.0):
    rs = np.random.RandomState(seed)
    pts = (centre + scale * rs.uniform(-1, 1, size=(sum(sizes), 6))).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    node = rs.uniform(-1, 1, size=(len(sizes), 3, M)).astype(np.float32)
    return pts, off, node


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


# ---- the vectorised group ---------------------------------------------------------------------------
@pytest.mark.parametrize("k,M", [(1, 1), (1, 2), (2, 3), (3, 9), (4, 33), (2, 65)])
def test_group_fast_is_the_loop_version_bit_for_bit(k, M):
    sizes = [1, max(k - 1, 1), 31, 32, 33, 200, 1100]
    pts, off, node = _clouds(sizes, M, seed=M + k, scale=3.0, centre=0.5)
    idx, _ = ragged_emu.assign(pts, off, node, k)
    want = ragged_emu.group(pts, off, idx, M, k)
    got = ragged_emu.group_fast(pts, off, idx, M, k)
    for w, g, name in zip(want[:3], got[:3], ("order", "node_sorted", "pos0")):
        assert np.array_equal(w, g), name
    assert np.array_equal(_i32(want[3]), _i32(got[3]))


def test_group_fast_long_lanes_match_the_loop_version():
    """Every copy on one node: lane chains of 40 terms, far from the origin, where the order of
    the additions shows in the low bits."""
    M, k = 2, 4
    pts, off, _ = _clouds([317], M, seed=3, scale=1.0, centre=100.0)
    idx = np.zeros(k * 317, np.int32)
    idx[::7] = 1
    want = ragged_emu.group(pts, off, idx, M, k)
    got = ragged_emu.group_fast(pts, off, idx, M, k)
    assert np.array_equal(_i32(want[3]), _i32(got[3]))
    assert np.array_equal(want[1], got[1])


def test_group_fast_clamps_ids_like_the_kernel():
    M, k = 9, 2
    pts, off, _ = _clouds([50, 3], M, seed=1)
    rs = np.random.RandomState(2)
    idx = rs.randint(0, M, size=k * 53).astype(np.int32)
    idx[::5] = -1
    idx[1::5] = M
    idx[2::11] = 2 ** 31 - 1
    got = ragged_emu.group_fast(pts, off, idx, M, k)
    want = ragged_emu.group(pts, off, np.clip(idx, 0, M - 1), M, k)
    for w, g in zip(want, got):
        assert np.array_equal(np.asarray(w).view(np.int32) if w.dtype == np.float32 else w,
                              np.asarray(g).view(np.int32) if g.dtype == np.float32 else g)


def test_group_fast_hand_built_means():
    """One cloud of 3 points, k = 2, M = 3: node 1 holds copies 0, 1, 5, node 2 the rest, node 0
    none. Means are sum / (count + 1e-5) in float32; an empty node's is 0."""
    pts = np.zeros((3, 6), np.float32)
    pts[:, 0] = [1.0, 2.0, 4.0]
    idx = np.array([1, 1, 2, 2, 2, 1], np.int32)      # copy s*3 + n
    order, ns, pos0, cm = ragged_emu.group_fast(pts, np.array([0, 3]), idx, 3, 2)
    assert order.tolist() == [0, 1, 5, 2, 3, 4]
    assert ns.tolist() == [1, 1, 1, 2, 2, 2] and pos0.tolist() == [0]
    den = np.float32(np.float32(3) + np.float32(1e-5))
    assert cm[0, 0].tolist() == [0.0, np.float32(np.float32(7) / den), np.float32(np.float32(7) / den)]


# ---- the offsets clamp ---------------------------------------------------------------------------------
def test_ranges_clamp_hand_built_offsets():
    T = 10
    lo, hi = ragged_emu.ragged_ranges([-4, 3, 15, 2, 7, 30], T)
    assert lo.tolist() == [0, 3, 10, 2, 7]
    assert hi.tolist() == [3, 10, 10, 7, 10]     # past T: T; decreasing pair: empty


@pytest.mark.parametrize("offsets", [[0, 3, 3, 3, 10], [-5, 4, 10], [0, 10, 10, 10, 10, 10],
                                     [2, 5, 8], [0, 6, 2, 9, 10], [0, 7, 3, 5, 1, 10], [12, 14, 20]])
def test_find_picks_one_cloud_per_row(offsets):
    """Every row lies inside at most one cloud's range as ragged_find picks it, and inside exactly
    the one searchsorted picks when the offsets are sorted. B may exceed the non-empty clouds."""
    T = 10
    g = np.arange(T)
    b, inside = ragged_emu.ragged_find(offsets, T, g)
    lo, hi = ragged_emu.ragged_ranges(offsets, T)
    assert np.all((b >= 0) & (b < len(offsets) - 1))
    assert np.array_equal(inside, (lo[b] <= g) & (g < hi[b]))
    c = ragged_emu.clamped_offsets(offsets, T)
    if np.all(np.diff(c) >= 0):
        want = np.searchsorted(c[:-1], g, side="right") - 1
        assert np.array_equal(b[inside], want[inside])
        assert np.array_equal(inside, (g >= c[0]) & (g < c[-1]))


def test_find_follows_the_binary_search_on_unsorted_offsets():
    """[0, 7, 3, 5, 1, 10]: the search's first probe is cloud 2 (offset 3), so rows 3..4 land in
    cloud 2 [3, 5) though cloud 0 [0, 7) also spans them, and rows 5..9 run on to cloud 4 [1, 10)
    past the empty cloud 3."""
    b, inside = ragged_emu.ragged_find([0, 7, 3, 5, 1, 10], 10, np.arange(10))
    assert b.tolist() == [0, 0, 0, 2, 2, 4, 4, 4, 4, 4]
    assert inside.all()


def test_assign_rows_is_assign_on_sorted_offsets():
    M, k = 9, 3
    pts, off, node = _clouds([1, 2, 40, 7], M, seed=5)
    idx, count = ragged_emu.assign(pts, off, node, k)
    idx2, count2, writes = ragged_emu.assign_rows(pts, off, node, k)
    assert np.array_equal(idx, idx2) and np.array_equal(count, count2)
    assert np.all(writes == 1)


def test_assign_rows_counts_racing_columns():
    """Offsets [0, 5, 3, 4, 10] at k = 3: rows 0..2 land in cloud 0 [0, 5) (columns s*5 + n),
    row 3 in cloud 2 [3, 4) (columns 9..11), rows 4..9 in cloud 3 [4, 10) (columns 12..29), so
    columns 10..12 are written twice and 3, 4, 8 never."""
    pts, _, node = _clouds([10], 9, seed=6)
    _, count, writes = ragged_emu.assign_rows(pts, [0, 5, 3, 4, 10], np.repeat(node, 4, axis=0), 3)
    assert np.flatnonzero(writes == 2).tolist() == [10, 11, 12]
    assert np.flatnonzero(writes == 0).tolist() == [3, 4, 8]
    assert count.sum(1).tolist() == [9, 0, 3, 18]


# ---- decentring ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,with_sn", [(1, True), (3, False), (4, True)])
def test_decenter_is_the_sorted_copies_in_stacked_order(k, with_sn):
    M = 9
    sizes = [1, 5, 77]
    pts, off, node = _clouds(sizes, M, seed=k)
    idx, _ = ragged_emu.assign(pts, off, node, k)
    order, ns, _, cm = ragged_emu.group_fast(pts, off, idx, M, k)
    xa, writes = ragged_emu.decenter(pts, off, idx, cm, k, with_sn)
    assert np.all(writes == 1)
    cloud = ns // M
    pt_of = np.concatenate([off[b] + np.tile(np.arange(P), k) for b, P in enumerate(sizes)])
    src = pt_of[order]
    want = pts[src, :3].T - cm[cloud, :, ns % M].T
    assert np.array_equal(_i32(xa[:3, order]), _i32(want))
    if with_sn:
        assert np.array_equal(_i32(xa[3:, order]), _i32(pts[src, 3:].T))
    assert xa.shape[0] == (6 if with_sn else 3)


# ---- index_max_ragged --------------------------------------------------------------------------------------
def _pool_data(C, kT, seed):
    rs = np.random.RandomState(seed)
    d = rs.randint(-3, 4, size=(C, kT)).astype(np.float32)      # many exact ties
    d[:, ::7] = -0.0
    d[:, 1::9] = 0.0
    d[:, 2::13] = np.nan
    d[:, 3::17] = np.inf
    d[:, 4::19] = -np.inf
    d[0::2, 5::5] = -1000.0
    d[1::3] = -1000.0 - rs.randint(0, 3, size=(1, kT)).astype(np.float32)   # sentinel channels
    return d


@pytest.mark.parametrize("C", [1, 15, 16, 17])
@pytest.mark.parametrize("k,M", [(1, 1), (3, 9), (4, 256)])
def test_index_max_ragged_is_pool_ref_per_cloud(C, k, M):
    sizes = [1, 4, 0, 37, 2]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    T = int(off[-1])
    data = _pool_data(C, k * T, seed=C + M)
    rs = np.random.RandomState(M)
    index = rs.randint(0, min(M, 5), size=k * T).astype(np.int32)
    got_i, got_v = ragged_emu.index_max_ragged(data, index, off, M, k)
    for b, P in enumerate(sizes):
        blk = slice(k * off[b], k * off[b + 1])
        if P == 0:
            assert not got_i[b].any() and not _i32(got_v[b]).any()
            continue
        wi, wv = pool_ref(data[None, :, blk], index[None, blk], M)
        assert np.array_equal(got_i[b], wi[0]), b
        assert np.array_equal(_i32(got_v[b]), _i32(wv[0])), b


def test_index_max_ragged_hand_built():
    """Column values of one cloud (k = 1, M = 2, all on node 0 but the last): -0 before +0 keeps
    -0; NaN never wins; a node whose values are all <= -1000 falls back to column 0; an id above
    M-1 reads as M-1, a negative one as M-1 too (uint32)."""
    data = np.array([[-0.0, 0.0, np.nan, -5.0, 7.0],
                     [-1000.0, -1001.0, np.nan, -2000.0, -1000.0]], np.float32)
    index = np.array([0, 0, 0, 0, 1], np.int32)
    i, v = ragged_emu.index_max_ragged(data, index, [0, 5], 2, 1)
    assert i[0].tolist() == [[0, 4], [0, 0]]
    assert _i32(v[0]).tolist() == _i32([[-0.0, 7.0], [-1000.0, -1000.0]]).tolist()
    i2, _ = ragged_emu.index_max_ragged(data, np.array([0, 0, 0, -1, 7], np.int32), [0, 5], 2, 1)
    assert i2[0].tolist() == [[0, 4], [0, 0]]
    i3, v3 = ragged_emu.index_max_ragged(data, np.array([0, 0, 0, -1, 7], np.int32), [0, 2], 2, 1)
    assert i3[0].tolist() == [[0, 0], [0, 0]] and np.isnan(data[:, 2]).all()
