"""Host side of point-cloud normal estimation (sonet_point_knn_f32, sonet_point_normals_f32,
sonet_b200.pointclouds), no GPU: the C entries' argument validation before any CUDA call, their
declaration, export and binding, the Python functions' refusals, save_npz files read back by the
reference's own loader, and the numpy restatement the GPU tests hold the kernels to, checked here on
inputs whose answers are known exactly."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

KNN = "sonet_point_knn_f32"
NORMALS = "sonet_point_normals_f32"
SIZE = "sonet_point_normals_scratch_bytes"
P_ = 256     # a non-null, 256-byte aligned placeholder pointer: validation fails before any read


# ---- the numpy restatement ------------------------------------------------------------------------
def knn_restated(pts, K, rows=None):
    """(idx [R, K] i32, dist [R, K] f32) of the queries `rows` (default all) of one cloud pts [P, 3]
    f32: d = ((dx*dx + dy*dy) + dz*dz) in fp32, ascending, NaN last, ties by index; -1 / +inf
    past P."""
    pts = np.asarray(pts, np.float32)
    P = len(pts)
    q = pts if rows is None else pts[rows]
    with np.errstate(invalid="ignore", over="ignore"):
        dx, dy, dz = (q[:, None, c] - pts[None, :, c] for c in range(3))
        d = (dx * dx + dy * dy) + dz * dz
    order = np.argsort(d, axis=1, kind="stable")[:, :K]      # NaN sorts last, stable keeps index order
    idx = np.full((len(q), K), -1, np.int32)
    dist = np.full((len(q), K), np.inf, np.float32)
    idx[:, :min(P, K)] = order
    dist[:, :min(P, K)] = np.take_along_axis(d, order, axis=1)
    return idx, dist


def pca_restated(pts, idx):
    """(w [R, 3] ascending eigenvalues, v [R, 3, 3] eigenvectors as columns, cov [R, 3, 3], ok [R])
    of the neighbour sets idx [R, K] (cloud-local, entries outside [0, P) skipped) of one cloud in
    fp64 with numpy.linalg.eigh; ok is False where the kernel's contract gives the zero vector."""
    pts = np.asarray(pts, np.float64)
    P = len(pts)
    idx = np.asarray(idx, np.int64)
    valid = (idx >= 0) & (idx < P)
    nb = pts[np.where(valid, idx, 0)]                          # [R, K, 3]
    n = valid.sum(1)
    finite = np.where(valid[..., None], np.isfinite(nb), True).all(axis=(1, 2))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        mean = np.where(valid[..., None], nb, 0).sum(1) / n[:, None]
        dev = np.where(valid[..., None], nb - mean[:, None, :], 0)
        cov = np.einsum("tki,tkj->tij", dev, dev) / n[:, None, None]
    tr = np.trace(cov, axis1=1, axis2=2)
    ok = (n >= 3) & finite & np.isfinite(tr) & (tr > 0)
    w = np.zeros((len(idx), 3))
    v = np.tile(np.eye(3), (len(idx), 1, 1))
    if ok.any():
        w[ok], v[ok] = np.linalg.eigh(cov[ok])
    wp = np.maximum(w, 0)
    ok &= wp[:, 1] > 2.0 ** -40 * wp.sum(1)
    return w, v, cov, ok


def canonical(n):
    """n [R, 3] f32 with the first component of largest magnitude made positive."""
    n = np.array(n, np.float32)
    c = np.argmax(np.abs(n), axis=1)
    flip = n[np.arange(len(n)), c] < 0
    n[flip] = -n[flip]
    return n


def centroid_restated(pts):
    """The cloud's fp64 mean in the kernel's order: lane t of 256 sums rows t, t+256, .. from +0,
    then s[i] += s[i+h] for h = 128, .., 1; c = s[0] / P."""
    x = np.asarray(pts, np.float64)
    P = len(x)
    acc = np.zeros((256, 3))
    for r in range(0, P, 256):
        blk = x[r:r + 256]
        acc[:len(blk)] = acc[:len(blk)] + blk
    h = 128
    while h:
        acc[:h] = acc[:h] + acc[h:2 * h]
        h //= 2
    return acc[0] / P


def orient_restated(n, pts, code, cen=None, view=None):
    """The normals n [R, 3] f32 (canonical or zero) of points pts [R, 3] under an orientation
    code: flipped iff ((nx*rx + ny*ry) + nz*rz) < 0 in fp64, ref = p - cen (1) or view - p (2)."""
    n = canonical(n)
    if code == 0:
        return n
    p = np.asarray(pts, np.float64)
    ref = p - np.asarray(cen, np.float64) if code == 1 else np.asarray(view, np.float32).astype(np.float64) - p
    nd = n.astype(np.float64)
    with np.errstate(invalid="ignore"):
        dot = (nd[:, 0] * ref[:, 0] + nd[:, 1] * ref[:, 1]) + nd[:, 2] * ref[:, 2]
    n[dot < 0] = -n[dot < 0]
    return n


def test_restated_knn_orders_ties_by_index_and_nan_last():
    pts = np.float32([[0, 0, 0], [1, 0, 0], [0, 0, 0], [np.nan, 0, 0], [3e30, 0, 0], [-1, 0, 0]])
    idx, dist = knn_restated(pts, 6)
    assert idx[0].tolist() == [0, 2, 1, 5, 4, 3] and dist[0, :4].tolist() == [0, 0, 1, 1]
    assert np.isinf(dist[0, 4]) and np.isnan(dist[0, 5])
    assert idx[3].tolist() == [0, 1, 2, 3, 4, 5]               # a NaN point: every distance NaN
    idx, dist = knn_restated(pts[:2], 4)
    assert idx.tolist() == [[0, 1, -1, -1], [1, 0, -1, -1]] and np.isinf(dist[:, 2:]).all()


def test_restated_normals_exact_on_a_plane_and_a_known_covariance():
    rs = np.random.RandomState(0)
    plane = np.zeros((30, 3))
    plane[:, [0, 2]] = rs.uniform(-1, 1, size=(30, 2))        # the plane y = 0
    idx = np.tile(np.arange(10), (30, 1))
    w, v, cov, ok = pca_restated(plane, idx)
    assert ok.all() and (cov[:, 1, :] == 0).all() and (w[:, 0] == 0).all()
    assert np.array_equal(canonical(v[:, :, 0].astype(np.float32)), np.tile(np.float32([0, 1, 0]), (30, 1)))
    # six points +-a e_x, +-b e_y, +-c e_z: covariance diag(a^2, b^2, c^2) / 3, normal e_z
    a, b, c = 3.0, 2.0, 0.5
    box = np.array([[a, 0, 0], [-a, 0, 0], [0, b, 0], [0, -b, 0], [0, 0, c], [0, 0, -c]])
    w, v, cov, ok = pca_restated(box, np.arange(6)[None])
    assert ok.all() and np.array_equal(cov[0], np.diag([a * a, b * b, c * c]) / 3)
    assert np.allclose(w[0], [c * c / 3, b * b / 3, a * a / 3], rtol=1e-15)
    assert np.allclose(np.abs(v[0][:, 0]), [0, 0, 1], atol=1e-15)
    # degenerate: coincident, collinear, non-finite, fewer than 3 valid indices
    line = np.arange(8)[:, None] * np.array([[1.0, 2.0, 3.0]])
    assert not pca_restated(np.ones((8, 3)), np.arange(8)[None])[3].any()
    assert not pca_restated(line, np.arange(8)[None])[3].any()
    bad = box.copy()
    bad[2, 1] = np.inf
    assert not pca_restated(bad, np.arange(6)[None])[3].any()
    assert not pca_restated(box, np.array([[0, 1, -1, 6, 7]]))[3].any()
    assert pca_restated(box, np.array([[0, 2, -1, 4, 9]]))[3].all()


def test_restated_sign_rules():
    n = np.float32([[0.6, -0.8, 0], [-0.5, 0.5, 0.1], [0, 0, -1], [0, 0, 0]])
    assert np.array_equal(canonical(n), np.float32([[-0.6, 0.8, 0], [0.5, -0.5, -0.1], [0, 0, 1], [0, 0, 0]]))
    p = np.float32([[0, 0, 0], [1, 1, 1], [0, 0, 5], [1, 2, 3]])
    got = orient_restated(n, p, 1, cen=np.array([0.0, 0.0, 6.0]))
    assert np.array_equal(got, np.float32([[-0.6, 0.8, 0], [0.5, -0.5, -0.1], [0, 0, -1], [0, 0, 0]]))
    got = orient_restated(n, p, 2, view=[np.nan, 0, 0])
    assert np.array_equal(got, canonical(n))
    assert np.allclose(centroid_restated(np.arange(3000.0).reshape(1000, 3)), [1498.5, 1499.5, 1500.5])


# ---- the C entries --------------------------------------------------------------------------------
def _knn(lib, data=P_, T=10, stride=3, off=P_, S=1, K=16, idx=P_, dist=None):
    return lib.sonet_point_knn_f32(data, T, stride, off, S, K, idx, dist, None)


def _normals(lib, data=P_, T=10, stride=6, off=P_, S=1, idx=P_, K=16, orient=0, view=None,
             scratch=None, nbytes=0, out=P_, ostride=6, curv=None):
    return lib.sonet_point_normals_f32(data, T, stride, off, S, idx, K, orient, view, scratch,
                                       nbytes, out, ostride, curv, None)


@pytest.mark.parametrize("call,kw,msg", [
    ("knn", dict(S=-1), "S=-1"), ("knn", dict(T=-1), "T=-1"), ("knn", dict(stride=2), "stride=2"),
    ("knn", dict(K=2), "K=2"), ("knn", dict(K=33), "K=33"), ("knn", dict(off=None), "null"),
    ("knn", dict(idx=None), "null"), ("knn", dict(data=None), "null"),
    ("normals", dict(S=-1), "S=-1"), ("normals", dict(T=-1), "T=-1"),
    ("normals", dict(stride=2), "stride=2"), ("normals", dict(ostride=2), "normal_stride=2"),
    ("normals", dict(K=2), "K=2"), ("normals", dict(K=33), "K=33"),
    ("normals", dict(orient=3), "orientation code 3"), ("normals", dict(orient=-1), "code -1"),
    ("normals", dict(orient=2), "view must not be null"), ("normals", dict(off=None), "null"),
    ("normals", dict(out=None), "null"), ("normals", dict(idx=None), "null"),
    ("normals", dict(data=None), "null"), ("normals", dict(orient=1), "scratch"),
    ("normals", dict(orient=1, scratch=P_, nbytes=8), "scratch"),
    ("normals", dict(orient=1, scratch=P_ + 8, nbytes=4096), "aligned"),
])
def test_bad_arguments_fail_before_any_cuda_call(lib_built, call, kw, msg):
    """Every pointer is a placeholder no CUDA call could use: the entries return before one."""
    from sonet_b200 import _C
    lib = _C.lib()
    rc = (_knn if call == "knn" else _normals)(lib, **kw)
    assert rc == _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    assert msg in _C.last_error(), _C.last_error()


def test_empty_batches_return_without_a_launch(lib_built):
    from sonet_b200 import _C
    lib = _C.lib()
    assert _knn(lib, S=0) == 0 and _knn(lib, S=0, T=0, data=None) == 0
    assert _normals(lib, S=0) == 0
    assert _normals(lib, S=0, orient=1, scratch=P_, nbytes=0) == 0
    assert _normals(lib, S=0, orient=2, view=P_) == 0
    assert lib.sonet_point_normals_scratch_bytes(0) == 0
    assert lib.sonet_point_normals_scratch_bytes(5) == 256
    assert lib.sonet_point_normals_scratch_bytes(11) == 512
    assert lib.sonet_point_normals_scratch_bytes(1 << 30) == 24 << 30      # not truncated
    assert lib.sonet_point_normals_scratch_bytes(-1) == -1


def test_entries_and_constants_are_declared_exported_and_bound(lib_built):
    from sonet_b200 import _C, ops
    h = ctypes.CDLL(lib_built)
    for name in (KNN, NORMALS, SIZE):
        assert hasattr(h, name) and name in _C.EXPORTED_SYMBOLS
    assert len(_C._SIGNATURES[KNN]) == 9 and len(_C._SIGNATURES[NORMALS]) == 15
    assert _C._RESTYPE[SIZE] is ctypes.c_longlong and _C._SIGNATURES[SIZE] == [ctypes.c_int]
    assert _C._SIGNATURES[KNN][1] is ctypes.c_longlong and _C._SIGNATURES[NORMALS][1] is ctypes.c_longlong
    want = dict(SONET_POINT_KNN_MAX_K=32, SONET_NORMALS_CANONICAL=0,
                SONET_NORMALS_AWAY_FROM_CENTROID=1, SONET_NORMALS_TOWARD_VIEWPOINT=2)
    for k, v in want.items():
        assert _C.CONSTANTS[k] == v
    assert (ops.POINT_KNN_MAX_K, ops.NORMALS_CANONICAL, ops.NORMALS_AWAY_FROM_CENTROID,
            ops.NORMALS_TOWARD_VIEWPOINT) == (32, 0, 1, 2)
    assert KNN not in _C.F16_ENTRIES and NORMALS not in _C.ACT_ENTRIES


# ---- the Python functions -------------------------------------------------------------------------
def _cpu_pair(counts):
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int64))
    return torch.zeros((int(off[-1]), 3)), off


@pytest.mark.parametrize("k", [2, 33, 0, 3.0, True, None])
def test_python_refuses_bad_k(k):
    from sonet_b200 import pointclouds
    data, off = _cpu_pair([10])
    for fn in (lambda: pointclouds.knn(data, off, k),
               lambda: pointclouds.estimate_normals(data, off, k=k)):
        with pytest.raises(ValueError, match=r"k=.* must be an integer in \[3, 32\]"):
            fn()


@pytest.mark.parametrize("orient", ["up", "Centroid", 1, "canonical"])
def test_python_refuses_bad_orient(orient):
    from sonet_b200 import pointclouds
    data, off = _cpu_pair([10])
    with pytest.raises(ValueError, match="orient="):
        pointclouds.estimate_normals(data, off, orient=orient)


def test_python_refuses_host_tensors_small_clouds_and_missing_viewpoint(monkeypatch):
    from sonet_b200 import pointclouds
    data, off = _cpu_pair([10, 2, 5])
    with pytest.raises(ValueError, match="CUDA tensors"):
        pointclouds.estimate_normals(data, off)
    # the offsets checks run on a host copy: stand the tensors in as if they were on the device
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    with pytest.raises(ValueError, match="cloud 1 has 2 points; a normal needs at least 3"):
        pointclouds.estimate_normals(data, off)
    with pytest.raises(ValueError, match="cloud 0 has 0 points"):
        pointclouds.knn(*_cpu_pair([0, 4]), 3)
    with pytest.raises(ValueError, match="cloud 1 has -1 points"):
        pointclouds.knn(torch.zeros((10, 3)), torch.tensor([0, 5, 4, 10]), 3)
    with pytest.raises(ValueError, match=r"offsets must lie in \[0, 10\]"):
        pointclouds.knn(torch.zeros((10, 3)), torch.tensor([0, 5, 11]), 3)
    with pytest.raises(ValueError, match="needs viewpoint"):
        pointclouds.estimate_normals(*_cpu_pair([4, 4]), orient="viewpoint")
    with pytest.raises(ValueError, match=r"viewpoint must be \[2, 3\]"):
        pointclouds.estimate_normals(*_cpu_pair([4, 4]), orient="viewpoint", viewpoint=[[0, 0, 0]])


def test_python_refuses_a_sample_larger_than_a_cloud(monkeypatch):
    from sonet_b200 import pointclouds
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    data, off = _cpu_pair([5000, 4000, 4096])
    with pytest.raises(ValueError, match=r"cloud 1: cannot take a larger sample \(4096\) than "
                                         r"population \(4000\) when 'replace=False'"):
        pointclouds.som_nodes(data, off, n=4096)


def test_build_dataset_refuses_bad_shapes_and_labels():
    from sonet_b200 import pointclouds
    with pytest.raises(ValueError, match=r"cloud 1 has shape \(5, 2\)"):
        pointclouds._to_device_rows([np.zeros((5, 3)), np.zeros((5, 2))], "cpu")
    with pytest.raises(ValueError, match="no clouds"):
        pointclouds._to_device_rows([], "cpu")
    rows, off = pointclouds._to_device_rows([np.ones((5, 3)), np.full((2, 3), 2.0)], "cpu")
    assert rows.shape == (7, 6) and (rows[:, 3:] == 0).all() and off.tolist() == [0, 5, 7]
    rows2, off2 = pointclouds._to_device_rows((torch.cat([rows[:, :3], rows[:, :1]], 1), off), "cpu")
    assert torch.equal(rows2, rows) and torch.equal(off2, off)


def test_save_npz_round_trip_through_the_reference_loader(tmp_path):
    """Ragged files written by save_npz, read by the reference's own ModelNet_Shrec_Loader (shrec,
    test mode, input_pc_num <= every cloud: the loader's choice is replayed)."""
    from oracle import ref_shims
    from sonet_b200 import pointclouds
    rs = np.random.RandomState(3)
    sizes, N, M = (60, 50, 75), 50, 16
    pts = [rs.uniform(-1, 1, size=(P, 6)).astype(np.float32) for P in sizes]
    nodes = [torch.from_numpy(rs.uniform(-1, 1, size=(M, 3)).astype(np.float32)) for _ in sizes]
    names = ["%06d" % (55 * (i + 1) + i) for i in range(3)]
    root = tmp_path / "shrec"
    paths = pointclouds.save_npz(str(root / "4x4" / "test"), names, (pts, nodes))
    assert [os.path.basename(p) for p in paths] == ["model_%s.npz" % n for n in names]
    for p, path in zip(pts, paths):
        z = np.load(path)
        assert sorted(z.files) == ["pc", "sn", "som_node"] and np.array_equal(z["sn"], p[:, 3:])
    with pytest.raises(ValueError, match="save_npz"):
        pointclouds.save_npz(str(tmp_path), names[:2], (pts, nodes))
    if not os.path.isdir(os.path.join(ref_shims.REF, "data")):
        pytest.skip("the reference checkout is not on this machine")
    ref_shims.install(use_ref_plugin=False)
    from data.modelnet_shrec_loader import ModelNet_Shrec_Loader
    (root / "category.txt").write_text("".join("cat%02d\n" % c for c in range(55)))
    (root / "test.txt").write_text("".join(n + "\n" for n in names))
    opt = types.SimpleNamespace(dataset="shrec", input_pc_num=N, node_num=M, som_k=1, classes=55,
                                batch_size=3, rot_horizontal=False, rot_perturbation=False,
                                translation_perturbation=False)
    loader = ModelNet_Shrec_Loader(str(root), "test", opt)
    assert len(loader) == 3
    for b in range(3):
        np.random.seed(100 + b)
        item = loader[b]
        sel = np.random.RandomState(100 + b).choice(sizes[b], N, replace=False)
        assert np.array_equal(item[0].numpy(), pts[b][sel, 0:3].T)
        assert np.array_equal(item[1].numpy(), pts[b][sel, 3:6].T)
        assert np.array_equal(item[3].numpy(), nodes[b].numpy().T)
