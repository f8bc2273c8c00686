"""-m gpu: exact k-NN within each cloud and PCA surface normals (csrc/point_normals.cu,
sonet_b200.pointclouds).

The k-NN is held bit for bit, indices and distances, to the numpy fp32 restatement in
test_point_normals_host.py at every K bucket, around every tile size the kernel uses, on ragged
batches, ties and non-finite coordinates. The normals are held to numpy.linalg.eigh in fp64 on the
kernel's own neighbour sets, to the documented sign rules, and to known geometry: planes, spheres
and the faces of convex meshes."""
import argparse
import os

import numpy as np
import pytest
import torch

from helpers import build_states
from test_point_normals_host import (canonical, centroid_restated, knn_restated, orient_restated,
                                     pca_restated)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
QTILE, CTILE = 128, 1024     # the kernel's query tile and shared-memory candidate tile


def _upload(clouds, stride=3):
    counts = [len(c) for c in clouds]
    data = np.zeros((sum(counts), stride), np.float32)
    data[:, :3] = np.concatenate(clouds) if clouds else np.zeros((0, 3), np.float32)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return torch.from_numpy(data).to(DEV), torch.from_numpy(off).to(DEV)


def _knn(clouds, K, stride=3):
    from sonet_b200 import ops
    data, off = _upload(clouds, stride)
    idx, dist = ops.point_knn(data, off, K, want_dist=True)
    torch.cuda.synchronize()
    return idx.cpu().numpy(), dist.cpu().numpy(), off.cpu().numpy()


def _check_knn(clouds, K, rows=None, stride=3):
    """Every cloud's idx and dist equal the restatement (on `rows` sampled queries of a cloud
    larger than 4096 points); returns (idx, dist, offsets)."""
    idx, dist, off = _knn(clouds, K, stride)
    rs = np.random.RandomState(K)
    for s, c in enumerate(clouds):
        q = None if len(c) <= 4096 else rs.choice(len(c), rows or 256, replace=False)
        wi, wd = knn_restated(c, K, q)
        gi, gd = idx[off[s]:off[s + 1]], dist[off[s]:off[s + 1]]
        if q is not None:
            gi, gd = gi[q], gd[q]
        assert np.array_equal(gi, wi), (s, len(c), K)
        assert np.array_equal(gd, wd, equal_nan=True), (s, len(c), K)
        assert ((gi >= 0) & (gi < len(c)) | (gi == -1)).all()
    return idx, dist, off


# ---- k-NN -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [3, 4, 16, 31, 32])
def test_knn_bit_exact_at_every_tile_edge(K):
    rs = np.random.RandomState(K)
    sizes = sorted({K - 1, K, K + 1, QTILE - 1, QTILE, QTILE + 1, CTILE - 1, CTILE, CTILE + 1,
                    2 * CTILE + 3})
    clouds = [rs.uniform(-1, 1, size=(P, 3)).astype(np.float32) for P in sizes]
    _check_knn(clouds, K)


def test_knn_ragged_with_an_empty_and_a_100k_cloud_and_strided_rows():
    rs = np.random.RandomState(1)
    clouds = [rs.normal(size=(700, 3)).astype(np.float32), np.zeros((0, 3), np.float32),
              rs.uniform(-1, 1, size=(100000, 3)).astype(np.float32),
              rs.uniform(0, 5, size=(2500, 3)).astype(np.float32)]
    _check_knn(clouds, 16, rows=512, stride=6)


def test_knn_duplicates_and_exact_ties():
    rs = np.random.RandomState(2)
    grid = rs.randint(-3, 4, size=(600, 3)).astype(np.float32)      # many exact distance ties
    dup = np.repeat(rs.uniform(-1, 1, size=(50, 3)).astype(np.float32), 7, axis=0)
    rs.shuffle(dup)
    same = np.ones((40, 3), np.float32)                              # all coincident
    idx, dist, off = _check_knn([grid, dup, same], 16)
    s = slice(off[2], off[3])
    assert (idx[s] == np.arange(16)).all() and (dist[s] == 0).all()


@pytest.mark.parametrize("K", [4, 16])
def test_knn_non_finite_coordinates_stay_in_range_and_local(K):
    rs = np.random.RandomState(3)
    bad = rs.uniform(-1, 1, size=(300, 3)).astype(np.float32)
    bad[5] = [np.nan, 0, 0]
    bad[17] = [np.inf, 1, 2]
    bad[18] = [-np.inf, 0, 0]
    bad[40:60, 2] = 3e30                   # finite points whose squared distances overflow
    bad[200] = [np.inf, np.inf, np.inf]
    small = bad[:K - 1].copy()             # P < K with a NaN point
    good = [rs.uniform(-1, 1, size=(P, 3)).astype(np.float32) for P in (130, 1030)]
    idx, dist, off = _check_knn([good[0], bad, small, good[1]], K)
    alone = [_knn([g], K)[:2] for g in good]
    for s, (ai, ad) in zip((0, 3), alone):
        assert np.array_equal(idx[off[s]:off[s + 1]], ai)
        assert np.array_equal(dist[off[s]:off[s + 1]], ad)
    assert (idx[off[2]:off[3], K - 1] == -1).all() and np.isinf(dist[off[2]:off[3], K - 1]).all()


def test_knn_results_do_not_depend_on_the_batch():
    rs = np.random.RandomState(4)
    clouds = [rs.uniform(-1, 1, size=(P, 3)).astype(np.float32) for P in (900, 131, 2000, 77)]
    i1, d1, o1 = _knn(clouds, 16)
    perm = [2, 0, 3, 1]
    i2, d2, o2 = _knn([clouds[p] for p in perm] + [clouds[0]], 16)
    for pos, s in enumerate(perm + [0]):
        assert np.array_equal(i2[o2[pos]:o2[pos + 1]], i1[o1[s]:o1[s + 1]])
        assert np.array_equal(d2[o2[pos]:o2[pos + 1]], d1[o1[s]:o1[s + 1]])
    i3, d3, _ = _knn(clouds, 16)
    assert np.array_equal(i1, i3) and np.array_equal(d1, d3)


# ---- normals --------------------------------------------------------------------------------------
def _normals(clouds, K, orient, view=None, idx=None):
    from sonet_b200 import ops
    data, off = _upload(clouds, 6)
    if idx is None:
        idx, _ = ops.point_knn(data, off, K)
    vt = None if view is None else torch.as_tensor(np.asarray(view, np.float32)).to(DEV)
    n, c = ops.estimate_normals(data, off, idx, orient, view=vt, out=data[:, 3:6],
                                want_curvature=True)
    torch.cuda.synchronize()
    assert n.data_ptr() == data.data_ptr() + 12
    return data[:, 3:6].cpu().numpy(), c.cpu().numpy(), idx.cpu().numpy(), off.cpu().numpy()


def _shapes(rs):
    sph = rs.normal(size=(3000, 3))
    sph = (sph / np.linalg.norm(sph, axis=1, keepdims=True) * 2 + [1, -3, 0.5]).astype(np.float32)
    blob = rs.normal(size=(1500, 3)) * [3, 1, 0.2]
    wavy = rs.uniform(-1, 1, size=(2000, 3))
    wavy[:, 2] = 0.2 * np.sin(4 * wavy[:, 0]) + 1e-3 * rs.normal(size=2000)
    return [sph, blob.astype(np.float32), wavy.astype(np.float32), rs.normal(size=(5, 3)).astype(np.float32)]


@pytest.mark.parametrize("K", [3, 8, 16, 32])
def test_normals_against_eigh_on_the_kernels_neighbour_sets(K):
    from sonet_b200 import ops
    rs = np.random.RandomState(10 + K)
    clouds = _shapes(rs)
    n, curv, idx, off = _normals(clouds, K, ops.NORMALS_CANONICAL)
    pts = np.concatenate(clouds).astype(np.float64)
    checked = 0
    for s in range(len(clouds)):
        rows = np.arange(off[s], off[s + 1])
        w, v, cov, ok = pca_restated(pts[off[s]:off[s + 1]], idx[rows])
        g, gc = n[rows].astype(np.float64), curv[rows]
        assert (g[~ok] == 0).all() and np.isnan(gc[~ok]).all()
        g, w, v, cov, gc = g[ok], w[ok], v[ok], cov[ok], gc[ok]
        assert np.abs(np.linalg.norm(g, axis=1) - 1).max() <= 1e-6
        sep = (w[:, 1] - w[:, 0]) >= 1e-6 * w[:, 2]
        e0 = v[:, :, 0]
        sin = np.linalg.norm(np.cross(g, e0), axis=1)
        assert sin[sep].max(initial=0) <= 2e-6, sin[sep].max()
        quad = np.einsum("ti,tij,tj->t", g, cov, g) / np.einsum("ti,ti->t", g, g)
        assert (quad[~sep] <= w[~sep, 0] + 1e-9 * w[~sep, 2]).all()
        want_c = np.maximum(w[:, 0], 0) / np.maximum(w, 0).sum(1)
        assert np.abs(gc - want_c).max() <= 1e-7 + 1e-6 * want_c.max()
        assert np.array_equal(g.astype(np.float32), canonical(g.astype(np.float32)))
        checked += int(sep.sum())
    assert checked > 5000


def test_degenerate_neighbourhoods_give_zero_and_nan():
    from sonet_b200 import ops
    t = np.arange(20, dtype=np.float32)[:, None]
    collinear = t * np.array([[1, 2, 3]], np.float32)
    coincident = np.full((20, 3), 0.25, np.float32)
    nan_cloud = np.random.RandomState(5).uniform(-1, 1, size=(8, 3)).astype(np.float32)
    nan_cloud[3] = [0, np.nan, 0]
    inf_cloud = nan_cloud.copy()
    inf_cloud[3] = [0, np.inf, 0]
    good = np.random.RandomState(6).uniform(-1, 1, size=(50, 3)).astype(np.float32)
    clouds = [collinear, coincident, nan_cloud, inf_cloud, good]
    n, curv, idx, off = _normals(clouds, 8, ops.NORMALS_AWAY_FROM_CENTROID)
    bad = slice(0, off[4])
    assert (n[bad] == 0).all() and np.isnan(curv[bad]).all()
    assert (np.abs(np.linalg.norm(n[off[4]:], axis=1) - 1) <= 1e-6).all()
    # fewer than 3 valid neighbours: given sets with -1 and out-of-range indices
    from sonet_b200 import ops as o
    data, offs = _upload([good], 6)
    nb = np.tile(np.arange(8, dtype=np.int32), (50, 1))
    nb[:10, 2:] = -1
    nb[10:20, 2:] = 50
    nb[20:30, 3:] = -1                     # exactly 3 valid: a normal
    nn, cc = o.estimate_normals(data, offs, torch.from_numpy(nb).to(DEV), o.NORMALS_CANONICAL,
                                want_curvature=True)
    nn, cc = nn.cpu().numpy(), cc.cpu().numpy()
    assert (nn[:20] == 0).all() and np.isnan(cc[:20]).all()
    assert (np.abs(np.linalg.norm(nn[20:], axis=1) - 1) <= 1e-6).all() and np.isfinite(cc[20:]).all()


def test_orientation_codes_follow_their_rules():
    from sonet_b200 import ops
    rs = np.random.RandomState(7)
    clouds = _shapes(rs)[:3]
    view = rs.normal(size=(3, 3)) * 5
    view[1] = np.nan
    base, _, idx, off = _normals(clouds, 16, ops.NORMALS_CANONICAL)
    pts = np.concatenate(clouds)
    cen = np.stack([centroid_restated(c) for c in clouds])
    for code in (ops.NORMALS_AWAY_FROM_CENTROID, ops.NORMALS_TOWARD_VIEWPOINT):
        n, _, idx2, _ = _normals(clouds, 16, code, view=view if code == 2 else None)
        assert np.array_equal(idx, idx2)
        for s in range(3):
            r = slice(off[s], off[s + 1])
            want = orient_restated(base[r], pts[r], code, cen[s], view[s])
            assert np.array_equal(n[r], want), (code, s)
    assert np.array_equal(n[off[1]:off[2]], base[off[1]:off[2]])         # NaN viewpoint
    sph = slice(off[0], off[1])
    n, _, _, _ = _normals(clouds, 16, ops.NORMALS_AWAY_FROM_CENTROID)
    assert (np.einsum("ti,ti->t", n[sph], pts[sph] - [1, -3, 0.5]) > 0).all()


def test_a_dot_of_zero_keeps_the_canonical_sign():
    from sonet_b200 import ops
    rs = np.random.RandomState(8)
    plane = np.zeros((400, 3), np.float32)
    plane[:, :2] = rs.randint(-20, 21, size=(400, 2)) / 8.0
    plane[:, :2] += rs.uniform(-0.01, 0.01, size=(400, 2)).astype(np.float32)
    for code, view, want in ((ops.NORMALS_CANONICAL, None, 1), (ops.NORMALS_AWAY_FROM_CENTROID, None, 1),
                             (ops.NORMALS_TOWARD_VIEWPOINT, [[3, -2, 0]], 1),
                             (ops.NORMALS_TOWARD_VIEWPOINT, [[0, 0, -1]], -1)):
        n, _, _, _ = _normals([plane], 12, code, view=view)
        assert np.array_equal(n, np.tile(np.float32([0, 0, want]), (400, 1))), (code, view)


# ---- geometry -------------------------------------------------------------------------------------
def test_tilted_plane_gives_its_normal():
    from sonet_b200 import pointclouds
    rs = np.random.RandomState(9)
    nrm = np.array([1.0, -2.0, 0.5]) / np.linalg.norm([1.0, -2.0, 0.5])
    a = np.cross(nrm, [0, 0, 1.0])
    a /= np.linalg.norm(a)
    b = np.cross(nrm, a)
    uv = rs.uniform(-1, 1, size=(600, 2))
    pts = (0.3 + uv[:, :1] * a + uv[:, 1:] * b).astype(np.float32)
    data, off = _upload([pts])
    n = pointclouds.estimate_normals(data, off, k=16, orient="viewpoint",
                                     viewpoint=[nrm * 5 + 0.3]).cpu().numpy()
    assert np.abs(n - nrm).max() <= 1e-6


def test_sphere_gives_the_radial_direction_within_the_sampling_radius():
    from sonet_b200 import ops, pointclouds
    rs = np.random.RandomState(10)
    p = rs.normal(size=(4000, 3))
    p = (p / np.linalg.norm(p, axis=1, keepdims=True)).astype(np.float32)
    data, off = _upload([p])
    n = pointclouds.estimate_normals(data, off, k=16).cpu().numpy().astype(np.float64)
    _, dist = ops.point_knn(data, off, 16, want_dist=True)
    # the neighbours lie in a cap of chord radius r = sqrt(max dist) around the point; the fitted
    # plane is tilted from the radial direction by at most the cap's half angle, about r
    r = np.sqrt(dist.cpu().numpy().astype(np.float64).max(1))
    radial = p / np.linalg.norm(p, axis=1, keepdims=True)
    sin = np.linalg.norm(np.cross(n, radial), axis=1)
    assert (sin <= r).all() and (np.einsum("ti,ti->t", n, radial) > 0).all()


def _icosphere(level):
    t = (1 + 5 ** 0.5) / 2
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t],
         [0, 1, -t], [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4],
         [11, 10, 2], [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9],
         [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]]
    v = [np.array(p, float) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        cache, nf = {}, []

        def mid(i, j):
            k = (min(i, j), max(i, j))
            if k not in cache:
                p = v[i] + v[j]
                v.append(p / np.linalg.norm(p))
                cache[k] = len(v) - 1
            return cache[k]
        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return np.array(v), np.array(f)


def _cube():
    v = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], float) * 0.7
    f = [[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
         [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]]
    return v, np.array(f)


def _outward(v, f):
    """The faces of a convex mesh around the origin wound so that their normals point outward."""
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    inward = np.einsum("ti,ti->t", np.cross(b - a, c - a), a + b + c) < 0
    f = f.copy()
    f[inward] = f[inward][:, ::-1]
    return v, f


def test_convex_meshes_face_normals_recovered_with_centroid_orientation():
    from sonet_b200 import meshes, pointclouds
    ms = meshes.Meshes([_outward(*_cube()), _outward(*_icosphere(1))], device=DEV)
    N, k = 10000, 16
    pts = meshes.sample_surface(ms, N, seed=4)
    off = torch.tensor([0, N, 2 * N], dtype=torch.int64, device=DEV)
    xyz = pts[:, :3].contiguous()
    est = pointclouds.estimate_normals(xyz, off, k=k, orient="centroid").cpu().numpy()
    idx = pointclouds.knn(xyz, off, k).cpu().numpy()
    face_n = pts[:, 3:6].cpu().numpy()
    for s in range(2):
        r = np.arange(s * N, (s + 1) * N)
        nb = face_n[s * N + idx[r].astype(np.int64)]                 # [N, k, 3]
        one_face = (np.abs(nb - face_n[r][:, None, :]).max(axis=(1, 2)) <= 1e-6)
        assert one_face.sum() > N // 8, (s, one_face.sum())
        e, f = est[r][one_face], face_n[r][one_face]
        assert (np.einsum("ti,ti->t", e, f) > 0).all()
        assert np.abs(e - f).max() <= 1e-5, (s, np.abs(e - f).max())


# ---- determinism and composition ------------------------------------------------------------------
def test_two_runs_batch_position_and_graph_replay_give_the_same_bits():
    from sonet_b200 import ops
    rs = np.random.RandomState(11)
    clouds = _shapes(rs)[:3]
    data, off = _upload(clouds, 6)
    view = torch.from_numpy(rs.normal(size=(3, 3)).astype(np.float32)).to(DEV)

    def run():
        idx, _ = ops.point_knn(data, off, 16)
        a, ca = ops.estimate_normals(data, off, idx, ops.NORMALS_AWAY_FROM_CENTROID, want_curvature=True)
        b, _ = ops.estimate_normals(data, off, idx, ops.NORMALS_TOWARD_VIEWPOINT, view=view)
        return idx, a, ca, b

    eager = [t.clone() for t in run()]
    again = run()
    for x, y in zip(eager, again):
        assert torch.equal(x, y)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()                                     # warm the allocator outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = run()
    for t in outs:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(eager, outs):
        assert torch.equal(x, y)
    # a cloud's normals do not depend on its position or its neighbours in the batch
    n1, _, _, o1 = _normals(clouds, 16, ops.NORMALS_AWAY_FROM_CENTROID)
    n2, _, _, o2 = _normals([clouds[2], clouds[0]], 16, ops.NORMALS_AWAY_FROM_CENTROID)
    assert np.array_equal(n2[o2[0]:o2[1]], n1[o1[2]:o1[3]])
    assert np.array_equal(n2[o2[1]:o2[2]], n1[o1[0]:o1[1]])


# ---- end to end -----------------------------------------------------------------------------------
def _ragged_clouds(rs):
    out = []
    for P in (700, 1100, 900, 1300):
        p = rs.normal(size=(P, 3)) * rs.uniform(0.5, 1.5, size=3)
        out.append((p / np.linalg.norm(p, axis=1, keepdims=True).max()).astype(np.float32))
    return out


def test_build_dataset_feeds_classifier_and_segmenter_like_host_copies(tmp_path):
    from sonet_b200 import augmentation, classifier, networks, pointclouds, segmenter, synth
    rs = np.random.RandomState(12)
    clouds = _ragged_clouds(rs)
    labels = [3, 1, 4, 1]
    ds = pointclouds.build_dataset(clouds, labels, k=16, rows=8, n=512, seed=6)
    assert len(ds) == 4 and ds.node_num == 64 and list(ds.counts) == [len(c) for c in clouds]
    data, off = ds.data.cpu().numpy(), ds.offsets.cpu().numpy()
    points = [data[off[s]:off[s + 1]] for s in range(4)]
    for s, c in enumerate(clouds):
        assert np.array_equal(points[s][:, :3], c)
        assert (np.abs(np.linalg.norm(points[s][:, 3:], axis=1) - 1) <= 1e-6).all()
    nodes = [ds.som_nodes[s].t().cpu().numpy() for s in range(4)]
    assert all(np.isfinite(x).all() for x in nodes)
    host = augmentation.DeviceDataset(points, labels, nodes)
    # the (data, offsets) form builds the same dataset
    ds2 = pointclouds.build_dataset((torch.from_numpy(np.concatenate(clouds)).to(DEV), off), labels,
                                    k=16, rows=8, n=512, seed=6)
    assert torch.equal(ds2.data, ds.data) and torch.equal(ds2.som_nodes, ds.som_nodes)

    P = 256
    opt = synth.make_opt("classifier", batch_size=2, input_pc_num=P, device=DEV)
    cpu_opt = synth.make_opt("classifier", batch_size=2, input_pc_num=P)
    st_e = synth.synth_state_dict(networks.Encoder(cpu_opt), seed=1)
    st_c = synth.synth_state_dict(networks.Classifier(cpu_opt), seed=2)
    lopt = argparse.Namespace(dataset="modelnet", input_pc_num=P, node_num=64, som_k=opt.som_k)
    sopt = synth.make_opt("segmenter", batch_size=2, input_pc_num=P)
    st_s = build_states("segmenter", sopt, 5)
    sopt.device, sopt.gpu_id = torch.device(DEV), 0
    got = []
    for d in (ds, host):
        batch = d.batch([2, 0], lopt, train=False, seed=11)
        m = classifier.Model(opt)
        m.encoder.load_state_dict(st_e)
        m.classifier.load_state_dict(st_c)
        m.set_input(*batch)
        m.test_model()
        sm = segmenter.Model(sopt)
        sm.encoder.load_state_dict(st_s["encoder"])
        sm.segmenter.load_state_dict(st_s["head"])
        pc, sn, label, som, knn = batch
        sm.set_input(pc, sn, label, torch.zeros(2, P, dtype=torch.int64, device=DEV), som, knn)
        sm.test_model()
        pts, offs, _ = d.full_clouds([2, 0])
        got.append((batch, m.score.detach().cpu(), sm.score_points(pts, offs).cpu()))
    for a, b in zip(got[0][0], got[1][0]):
        assert torch.equal(a, b)
    assert torch.equal(got[0][1], got[1][1]) and torch.isfinite(got[0][1]).all()
    assert torch.equal(got[0][2], got[1][2]) and torch.isfinite(got[0][2]).all()
    assert got[0][2].shape[0] == len(clouds[2]) + len(clouds[0])

    names = ["a%d" % s for s in range(4)]
    paths = pointclouds.save_npz(str(tmp_path), names, ds)
    for s, path in enumerate(paths):
        assert os.path.basename(path) == "model_a%d.npz" % s
        z = np.load(path)
        assert sorted(z.files) == ["pc", "sn", "som_node"]
        assert np.array_equal(z["pc"], points[s][:, :3]) and np.array_equal(z["sn"], points[s][:, 3:])
        assert np.array_equal(z["som_node"], nodes[s])


def test_som_nodes_on_equal_clouds_match_meshes_som_nodes():
    from sonet_b200 import meshes, pointclouds
    rs = np.random.RandomState(13)
    B, P = 3, 1500
    pts = torch.from_numpy(rs.uniform(-1, 1, size=(B, P, 6)).astype(np.float32)).to(DEV)
    off = torch.arange(B + 1, dtype=torch.int64, device=DEV) * P
    want = meshes.som_nodes(pts, 8, 8, 1024, seed=5)
    got = pointclouds.som_nodes(pts.reshape(B * P, 6), off, 8, 8, 1024, seed=5)
    assert torch.equal(got.transpose(1, 2), want)
    want = meshes.som_nodes(pts, 4, 4, 512, rng=np.random.RandomState(2))
    got = pointclouds.som_nodes(pts.reshape(B * P, 6), off, 4, 4, 512, rng=np.random.RandomState(2))
    assert torch.equal(got.transpose(1, 2), want)
