"""Host side of normal orientation by minimum spanning tree (sonet_point_normals_orient_f32,
pointclouds.orient_normals, estimate_normals(orient="propagate")), no GPU: the restatement in
orient_emu.py against scipy's minimum spanning tree and on hand-built graphs whose answers are known,
the C entry's argument validation before any CUDA call, its declaration and binding, and the Python
refusals."""
import ctypes

import numpy as np
import pytest
import torch
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import minimum_spanning_tree

import orient_emu

ORIENT = "sonet_point_normals_orient_f32"
SIZE = "sonet_point_normals_orient_scratch_bytes"
P_ = 256     # a non-null, 256-byte aligned placeholder pointer: validation fails before any read


def _cloud(n, rs):
    pts = rs.uniform(-1, 1, size=(n, 3)).astype(np.float32)
    nrm = rs.normal(size=(n, 3)).astype(np.float32)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return pts, nrm


def _knn(pts, K):
    d = ((pts[:, None, :].astype(np.float64) - pts[None]) ** 2).sum(-1)
    return np.argsort(d, axis=1, kind="stable")[:, :K].astype(np.int32)


# ---- the restatement ------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_restated_tree_is_scipys_minimum_spanning_tree(seed):
    """On random graphs, distinct weights almost surely: the same edge set as scipy's MST, whose
    zero-weight entries would vanish, so the weights are offset by 1 there."""
    rs = np.random.RandomState(seed)
    pts, nrm = _cloud(300, rs)
    idx = _knn(pts, 6)
    off = np.array([0, 300])
    cloud, lo, hi = orient_emu.vertices(pts, off, nrm, 300)
    ga, gb, w, flip = orient_emu.edges(idx, cloud, lo, hi, nrm)
    assert len(np.unique(w)) == len(w)
    _, _, (ta, tb) = orient_emu.orient(pts, off, idx, nrm, 1, want_tree=True)
    g = coo_matrix((w.astype(np.float64) + 1.0, (ga, gb)), shape=(300, 300))
    mst = minimum_spanning_tree(g).tocoo()
    want = {(min(a, b), max(a, b)) for a, b in zip(mst.row, mst.col)}
    assert {(int(a), int(b)) for a, b in zip(ta, tb)} == want


def test_ring_of_flips_follows_the_tree_parity():
    """A ring of 8 points whose normals alternate; the heaviest edge (the least |dot|) is left out
    of the tree, and every sign follows the anchor along the rest."""
    ang = np.arange(8) * np.pi / 4
    pts = np.stack([np.cos(ang), np.sin(ang), np.zeros(8)], 1).astype(np.float32)
    nrm = np.stack([np.cos(ang), np.sin(ang), np.zeros(8)], 1).astype(np.float32)
    nrm[1::2] *= -1                                   # every other normal points inward
    nrm[3] = [0.0, 0.6, 0.8]                          # edges 2-3 and 3-4 become the heaviest
    idx = np.array([[(i - 1) % 8, (i + 1) % 8] for i in range(8)], np.int32)
    off = np.array([0, 8])
    out, comp, (ta, tb) = orient_emu.orient(pts, off, idx, nrm, 1, want_tree=True)
    assert len(ta) == 7 and (comp == comp[0]).all()
    radial = (out[:, :2] * pts[:, :2]).sum(1)
    assert (np.delete(radial, 3) > 0).all()           # outward, away from the centroid
    assert np.array_equal(np.abs(out), np.abs(nrm))   # signs only


def test_ties_are_decided_by_the_lower_then_the_higher_index():
    """Equal weights everywhere: the tree is the one Kruskal builds in (lo, hi) order."""
    pts = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]])
    nrm = np.tile(np.float32([0, 0, 1]), (4, 1))
    idx = np.array([[1, 2, 3], [0, 2, 3], [0, 1, 3], [0, 1, 2]], np.int32)
    _, comp, (ta, tb) = orient_emu.orient(pts, np.array([0, 4]), idx, nrm, 1, want_tree=True)
    assert list(zip(ta.tolist(), tb.tolist())) == [(0, 1), (0, 2), (0, 3)]
    # all four are equally far from the centroid: the lowest index anchors
    assert (comp == 0).all()


def test_isolated_zero_and_non_finite_points_and_max_points():
    rs = np.random.RandomState(5)
    pts, nrm = _cloud(12, rs)
    nrm[2] = 0                                        # zero normal: not a vertex
    nrm[4, 1] = np.nan                                # non-finite normal
    pts[6, 0] = np.inf                                # non-finite point
    idx = _knn(np.nan_to_num(pts, posinf=9), 4)
    idx[idx == 8] = -1                                # nobody lists 8, and 8 lists only itself
    idx[8] = 8
    idx[:, 3] = -1                                    # out-of-range entries are skipped
    out, comp = orient_emu.orient(pts, np.array([0, 12]), idx, nrm, 1)
    for r in (2, 4, 6):
        assert comp[r] == -1 and np.array_equal(out[r], nrm[r], equal_nan=True)
    assert comp[8] == 8                               # its own anchor
    out2, comp2 = orient_emu.orient(pts, np.array([0, 12]), idx, nrm, 1, max_points=10)
    assert (comp2[10:] == -1).all() and np.array_equal(out2[10:], nrm[10:])


def test_viewpoint_anchor_and_nan_view():
    pts = np.float32([[0, 0, 0], [1, 0, 0], [2, 0, 0]])
    nrm = np.float32([[0, 0, 1], [0, 0, -1], [0, 0, 1]])
    idx = np.array([[1], [2], [1]], np.int32)
    out, comp = orient_emu.orient(pts, np.array([0, 3]), idx, nrm, 2, view=[[2, 0, -5]])
    assert (comp == 2).all() and (out[:, 2] == -1).all()
    out, comp = orient_emu.orient(pts, np.array([0, 3]), idx, nrm, 2, view=[[np.nan, 0, 0]])
    assert (comp == 0).all() and (out[:, 2] == 1).all()   # NaN distances: index 0, its sign kept


# ---- the C entry ----------------------------------------------------------------------------------
def _orient(lib, data=P_, T=10, stride=6, off=P_, S=1, maxp=10, idx=P_, K=16, anchor=1, view=None,
            scratch=P_, nbytes=1 << 20, out=P_, ostride=6, comp=None):
    return lib.sonet_point_normals_orient_f32(data, T, stride, off, S, maxp, idx, K, anchor, view,
                                              scratch, nbytes, out, ostride, comp, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(S=-1), "S=-1"), (dict(T=-1), "T=-1"), (dict(stride=2), "stride=2"),
    (dict(ostride=2), "normal_stride=2"), (dict(K=0), "K=0"), (dict(K=33), "K=33"),
    (dict(maxp=-1), "max_points=-1"), (dict(maxp=1 << 24), "max_points=16777216"),
    (dict(anchor=0), "anchor code 0"), (dict(anchor=3), "anchor code 3"),
    (dict(anchor=-1), "anchor code -1"), (dict(anchor=2), "view must not be null"),
    (dict(off=None), "null"), (dict(out=None), "null"), (dict(idx=None), "null"),
    (dict(data=None), "null"), (dict(scratch=None), "scratch"), (dict(nbytes=256), "scratch"),
    (dict(scratch=P_ + 8), "aligned"),
])
def test_bad_arguments_fail_before_any_cuda_call(lib_built, kw, msg):
    """Every pointer is a placeholder no CUDA call could use: the entry returns before one."""
    from sonet_b200 import _C
    rc = _orient(_C.lib(), **kw)
    assert rc == _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    assert msg in _C.last_error(), _C.last_error()


def test_empty_batches_and_the_scratch_query(lib_built):
    from sonet_b200 import _C
    lib = _C.lib()
    assert _orient(lib, S=0, scratch=None, nbytes=0) == 0
    assert _orient(lib, S=0, T=0, data=None, idx=None, scratch=None, nbytes=0) == 0
    assert _orient(lib, S=0, anchor=2, view=P_, scratch=None, nbytes=0) == 0
    assert lib.sonet_point_normals_orient_scratch_bytes(100, 0) == 0
    # flags 256 | centroids | four u64 and three 32-bit arrays of T, each rounded up to 256 bytes
    assert lib.sonet_point_normals_orient_scratch_bytes(1000, 3) == 256 + 256 + 4 * 8192 + 3 * 4096
    assert lib.sonet_point_normals_orient_scratch_bytes(0, 1) == 512
    assert lib.sonet_point_normals_orient_scratch_bytes(1 << 33, 1) == 512 + 44 * (1 << 33)
    assert lib.sonet_point_normals_orient_scratch_bytes(-1, 1) == -1
    assert lib.sonet_point_normals_orient_scratch_bytes(1, -1) == -1


def test_entry_and_constants_are_declared_exported_and_bound(lib_built):
    from sonet_b200 import _C, ops
    h = ctypes.CDLL(lib_built)
    for name in (ORIENT, SIZE):
        assert hasattr(h, name) and name in _C.EXPORTED_SYMBOLS
    assert len(_C._SIGNATURES[ORIENT]) == 16 and _C._SIGNATURES[ORIENT][1] is ctypes.c_longlong
    assert _C._RESTYPE[SIZE] is ctypes.c_longlong
    assert _C._SIGNATURES[SIZE] == [ctypes.c_longlong, ctypes.c_int]
    assert _C.CONSTANTS["SONET_POINT_ORIENT_MAX_POINTS"] == 1 << 24
    assert _C.CONSTANTS["SONET_POINT_ORIENT_MAX_ROUNDS"] == 24
    assert (ops.POINT_ORIENT_MAX_POINTS, ops.POINT_ORIENT_MAX_ROUNDS) == (1 << 24, 24)
    assert [ops.orient_rounds(p) for p in (0, 1, 2, 3, 4, 5, 10000, (1 << 24) - 1)] == \
        [0, 0, 1, 2, 2, 3, 14, 24]
    assert ORIENT not in _C.F16_ENTRIES and ORIENT not in _C.ACT_ENTRIES


# ---- the Python functions -------------------------------------------------------------------------
def _cpu_pair(counts):
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int64))
    return torch.zeros((int(off[-1]), 3)), off


@pytest.mark.parametrize("orient", ["propagate-centroid", "Propagate", "tree", 4])
def test_estimate_normals_refuses_other_orient_values(orient):
    from sonet_b200 import pointclouds
    with pytest.raises(ValueError, match="orient="):
        pointclouds.estimate_normals(*_cpu_pair([10]), orient=orient)


@pytest.mark.parametrize("anchor", ["propagate", "canonical", None, 1, "Centroid"])
def test_orient_normals_refuses_bad_anchor(anchor):
    from sonet_b200 import pointclouds
    data, off = _cpu_pair([10])
    with pytest.raises(ValueError, match="anchor="):
        pointclouds.orient_normals(data, off, data, anchor=anchor)


def test_python_refuses_missing_viewpoint_bad_idx_and_empty_clouds(monkeypatch):
    from sonet_b200 import pointclouds
    data, off = _cpu_pair([4, 4])
    with pytest.raises(ValueError, match="CUDA tensors"):
        pointclouds.orient_normals(data, off, data)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    with pytest.raises(ValueError, match="orient='propagate-viewpoint' needs viewpoint"):
        pointclouds.estimate_normals(data, off, orient="propagate-viewpoint")
    with pytest.raises(ValueError, match=r"viewpoint must be \[2, 3\]"):
        pointclouds.estimate_normals(data, off, orient="propagate-viewpoint", viewpoint=[[0, 0, 0]])
    with pytest.raises(ValueError, match="anchor='viewpoint' needs viewpoint"):
        pointclouds.orient_normals(data, off, data, anchor="viewpoint")
    with pytest.raises(ValueError, match=r"k=2 must be an integer"):
        pointclouds.orient_normals(data, off, data, k=2)
    with pytest.raises(ValueError, match=r"idx must be a CUDA i32 \[8, K\]"):
        pointclouds.orient_normals(data, off, data, idx=torch.zeros((8, 33), dtype=torch.int32))
    with pytest.raises(ValueError, match="cloud 1 has 0 points"):
        pointclouds.orient_normals(*_cpu_pair([3, 0]), torch.zeros(3, 3))
    big = torch.tensor([0, 1 << 24], dtype=torch.int64)
    with pytest.raises(ValueError, match="orientation supports at most 16777215"):
        pointclouds._max_points(big.numpy(), "orient_normals")
