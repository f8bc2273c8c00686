"""-m gpu: normal orientation along each component's minimum spanning tree
(sonet_point_normals_orient_f32, pointclouds.orient_normals, estimate_normals(orient="propagate")).

Signs and component ids are held bit for bit to the Kruskal restatement in orient_emu.py: ragged
batches at several K, an exactly flat grid where the tie rule decides the whole tree, random input
signs, zero and non-finite normals, clouds smaller than K, several components per cloud, a Möbius
band (deep tree paths) and a cloud of 100,000 points. Then geometry with known answers (a torus, two
spheres, a concave mesh, an open scan toward its viewpoint), invariance across runs, batch position
and CUDA graph replay, malformed offsets with canaries around every buffer, and build_dataset."""
import numpy as np
import pytest
import torch

import orient_emu
from test_gpu_ragged_envelope import Guarded, _off64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
AWAY, VIEW = 1, 2


def _upload(clouds, stride=6):
    counts = [len(c) for c in clouds]
    data = np.zeros((sum(counts), stride), np.float32)
    data[:, :3] = np.concatenate(clouds)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    return torch.from_numpy(data).to(DEV), torch.from_numpy(off).to(DEV)


def _estimate(data, off, K):
    """(idx, canonical normals written into data[:, 3:6])."""
    from sonet_b200 import ops
    idx, _ = ops.point_knn(data, off, K)
    ops.estimate_normals(data, off, idx, ops.NORMALS_CANONICAL, out=data[:, 3:6])
    return idx


def _orient(data, off, idx, code, view=None, max_points=None):
    """(normals [T, 3], component [T]) on the host after orienting data[:, 3:6] in place."""
    from sonet_b200 import ops
    v = None if view is None else torch.as_tensor(np.asarray(view, np.float32)).to(DEV)
    _, comp = ops.orient_normals(data, off, idx, data[:, 3:6], code, view=v, max_points=max_points,
                                 want_component=True)
    torch.cuda.synchronize()
    return data[:, 3:6].cpu().numpy(), comp.cpu().numpy()


def _check(data, off, idx, code, view=None, max_points=None):
    """Orient on the device and compare with the restatement bit for bit; -> (normals, comp)."""
    d, o, i = data.cpu().numpy(), off.cpu().numpy(), idx.cpu().numpy()
    want_n, want_c = orient_emu.orient(d, o, i, d[:, 3:6], code, view=view, max_points=max_points)
    got_n, got_c = _orient(data, off, idx, code, view, max_points)
    assert np.array_equal(got_c, want_c), "components: %d differ" % int((got_c != want_c).sum())
    bad = got_n.view(np.int32) != want_n.view(np.int32)
    assert not bad.any(), "signs: %d rows differ" % int(bad.any(1).sum())
    return got_n, got_c


def _flip_some(data, rs, frac=0.5):
    t = data[:, 3:6]
    s = torch.from_numpy(np.where(rs.uniform(size=len(t)) < frac, -1.0, 1.0).astype(np.float32))
    t.mul_(s.to(DEV)[:, None])


# ---- bit equality with the restatement ------------------------------------------------------------
@pytest.mark.parametrize("K", [3, 4, 16, 32])
@pytest.mark.parametrize("code", [AWAY, VIEW])
def test_random_ragged_batches(K, code):
    rs = np.random.RandomState(K + 100 * code)
    sizes = [1, 2, K - 1, K, 37, 300, 1000, 2500]
    clouds = [rs.normal(size=(P, 3)).astype(np.float32) * rs.uniform(0.5, 3) for P in sizes]
    data, off = _upload(clouds)
    idx = _estimate(data, off, K)
    _flip_some(data, rs)
    view = rs.uniform(-5, 5, size=(len(sizes), 3)).astype(np.float32)
    _check(data, off, idx, code, view)


def test_flat_grid_ties_decide_the_whole_tree():
    """Every normal is +-e_z, so every weight is exactly 0 and the (lo, hi) order alone builds the
    tree; the grid's points are also equally far from the centroid in rings."""
    rs = np.random.RandomState(1)
    g = np.stack(np.meshgrid(np.arange(60), np.arange(45), indexing="ij"), -1).reshape(-1, 2)
    pts = np.concatenate([g, np.zeros((len(g), 1))], 1).astype(np.float32)
    perm = rs.permutation(len(pts))
    data, off = _upload([pts[perm], pts])
    idx = _estimate(data, off, 8)
    _flip_some(data, rs)
    n, comp = _check(data, off, idx, AWAY)
    assert (np.abs(n[:, 2]) == 1).all()
    _check(data, off, idx, VIEW, [[0, 0, 1], [30, 20, -2]])


def test_zero_non_finite_normals_and_small_clouds():
    rs = np.random.RandomState(2)
    clouds = [rs.normal(size=(P, 3)).astype(np.float32) for P in (500, 2, 1, 3, 700)]
    data, off = _upload(clouds)
    idx = _estimate(data, off, 16)
    _flip_some(data, rs)
    h = data.cpu().numpy()
    h[rs.choice(len(h), 40, replace=False), 3:6] = 0
    h[rs.choice(len(h), 10, replace=False), 3 + rs.randint(3)] = np.nan
    h[rs.choice(len(h), 10, replace=False), 3 + rs.randint(3)] = np.inf
    h[rs.choice(len(h), 10, replace=False), rs.randint(3)] = np.nan     # non-finite points
    h[7, 3:6] = [3e38, -3e38, 1e-45]                                    # huge and subnormal
    data = torch.from_numpy(h).to(DEV)
    _, comp = _check(data, off, idx, AWAY)
    assert (comp[~np.isfinite(h).all(1)] == -1).all()
    _check(data, off, idx, VIEW, rs.normal(size=(5, 3)))


def test_several_components_per_cloud():
    rs = np.random.RandomState(3)
    blobs = [rs.normal(size=(300, 3)) * 0.1 + c for c in ([0, 0, 0], [5, 0, 0], [0, 7, 1], [3, 3, 3])]
    cloud = np.concatenate(blobs).astype(np.float32)[rs.permutation(1200)]
    data, off = _upload([cloud, cloud[:500]])
    idx = _estimate(data, off, 10)
    _flip_some(data, rs)
    _, comp = _check(data, off, idx, AWAY)
    assert len(np.unique(comp[:1200])) >= 4


def _mobius(n_u, n_v, width=0.05):
    u = np.linspace(0, 2 * np.pi, n_u, endpoint=False)
    v = np.linspace(-width, width, n_v)
    U, V = [a.reshape(-1) for a in np.meshgrid(u, v, indexing="ij")]
    r = 1 + V * np.cos(U / 2)
    return np.stack([r * np.cos(U), r * np.sin(U), V * np.sin(U / 2)], 1).astype(np.float32)


def test_mobius_band_deep_tree_paths():
    """Non-orientable, long and narrow: its tree paths run thousands of edges deep, so the pointer
    jumps have long chains to compress."""
    rs = np.random.RandomState(4)
    pts = _mobius(3000, 5, width=0.004)
    data, off = _upload([pts, pts[rs.permutation(len(pts))]])
    idx = _estimate(data, off, 6)
    _check(data, off, idx, AWAY)
    _flip_some(data, rs)
    _check(data, off, idx, VIEW, [[0, 0, 3], [2, 0, 0]])


def test_one_cloud_of_100k_points():
    rs = np.random.RandomState(5)
    a = rs.uniform(0, 2 * np.pi, size=(2, 100000))
    pts = np.stack([np.cos(a[0]) * np.sin(a[1] / 2), np.sin(a[0]) * np.sin(a[1] / 2),
                    np.cos(a[1] / 2)], 1).astype(np.float32)
    data, off = _upload([pts])
    idx = _estimate(data, off, 8)
    _flip_some(data, rs)
    _check(data, off, idx, AWAY)


@pytest.mark.parametrize("seed", range(3))
def test_flipping_input_signs_changes_nothing(seed):
    """With no dot exactly 0 the output does not depend on any input sign."""
    rs = np.random.RandomState(10 + seed)
    clouds = [rs.normal(size=(P, 3)).astype(np.float32) for P in (800, 50, 1500)]
    data, off = _upload(clouds)
    idx = _estimate(data, off, 12)
    n0, c0 = _orient(data.clone(), off, idx, AWAY)
    _flip_some(data, rs, frac=rs.uniform(0.1, 0.9))
    n1, c1 = _orient(data.clone(), off, idx, AWAY)
    assert np.array_equal(n0.view(np.int32), n1.view(np.int32)) and np.array_equal(c0, c1)


# ---- geometry -------------------------------------------------------------------------------------
def _torus(n, R=1.0, r=0.4, seed=6):
    """n points spread uniformly over the torus' area, and their analytic outward normals."""
    rs = np.random.RandomState(seed)
    u = rs.uniform(0, 2 * np.pi, 4 * n)
    v = rs.uniform(0, 2 * np.pi, 4 * n)
    keep = rs.uniform(0, R + r, 4 * n) < R + r * np.cos(v)      # area element (R + r cos v)
    u, v = u[keep][:n], v[keep][:n]
    nrm = np.stack([np.cos(v) * np.cos(u), np.cos(v) * np.sin(u), np.sin(v)], 1)
    pts = np.stack([(R + r * np.cos(v)) * np.cos(u), (R + r * np.cos(v)) * np.sin(u), r * np.sin(v)], 1)
    return pts.astype(np.float32), nrm


def test_torus_propagate_is_outward_where_centroid_is_not():
    from sonet_b200 import pointclouds
    pts, nrm = _torus(30000)
    data, off = _upload([pts])
    got = {}
    for orient in ("centroid", "propagate"):
        n = pointclouds.estimate_normals(data, off, k=16, orient=orient).cpu().numpy()
        got[orient] = float(((n * nrm).sum(1) <= 0).mean())
    print("torus, 30000 points, k=16: inward fraction centroid %.4f, propagate %.4f"
          % (got["centroid"], got["propagate"]))
    assert got["propagate"] == 0.0
    assert got["centroid"] > 0.1


def test_two_separated_spheres_are_two_outward_components():
    from sonet_b200 import pointclouds
    rs = np.random.RandomState(7)
    s = rs.normal(size=(2, 4000, 3))
    s /= np.linalg.norm(s, axis=2, keepdims=True)
    pts = np.concatenate([s[0] + [-3, 0, 0], s[1] * 0.5 + [3, 1, 0]]).astype(np.float32)
    out = np.concatenate([s[0], s[1]])
    perm = rs.permutation(len(pts))
    data, off = _upload([pts[perm]])
    n = pointclouds.estimate_normals(data, off, k=16, orient=None)
    n, comp = pointclouds.orient_normals(data, off, n, k=16, return_components=True)
    n, comp = n.cpu().numpy(), comp.cpu().numpy()
    assert len(np.unique(comp)) == 2
    assert ((n * out[perm]).sum(1) > 0).all()


def _l_prism():
    """An L-shaped prism (a cube with a notch): 12 vertices, 20 triangles, and a test for the
    solid's interior."""
    poly = np.array([[0, 0], [2, 0], [2, 1], [1, 1], [1, 2], [0, 2]], float)
    verts = np.concatenate([np.c_[poly, np.zeros(6)], np.c_[poly, np.ones(6)]])
    tris = [(0, 1, 2), (0, 2, 3), (0, 3, 4), (0, 4, 5)]                # bottom, a fan
    tris += [(6 + c, 6 + b, 6 + a) for a, b, c in tris]                  # top
    for i in range(6):
        j = (i + 1) % 6
        tris += [(i, j, 6 + j), (i, 6 + j, 6 + i)]

    def inside(p):
        x, y, z = p[..., 0], p[..., 1], p[..., 2]
        return (z > 0) & (z < 1) & (x > 0) & (y > 0) & (((x < 2) & (y < 1)) | ((x < 1) & (y < 2)))
    return verts, np.array(tris, np.int32), inside


def _segment_dist(p, a, b):
    ab = b - a
    t = np.clip(((p - a) @ ab) / (ab @ ab), 0, 1)
    return np.linalg.norm(p - (a + t[:, None] * ab), axis=1)


def test_concave_mesh_matches_its_face_normals_away_from_edges():
    """Points sampled on an L-shaped prism: away from its 18 edges (farther than 0.08, about three
    point spacings) every propagated normal has the sign of its outward face normal."""
    from sonet_b200 import meshes, pointclouds
    verts, faces, inside = _l_prism()
    N = 20000
    out, face, _ = meshes.sample_surface(meshes.Meshes([(verts, faces)], device=DEV), N, seed=1,
                                         want_faces=True)
    pts, face = out[:, :3].cpu().numpy().astype(np.float32), face.cpu().numpy()
    tri = verts[faces]
    fn = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    fn /= np.linalg.norm(fn, axis=1, keepdims=True)
    cen = tri.mean(1)
    fn[inside(cen + 1e-3 * fn)] *= -1                                    # outward
    data, off = _upload([pts])
    n = pointclouds.estimate_normals(data, off, k=16, orient="propagate").cpu().numpy()
    ref = fn[face]
    ring = [(i, (i + 1) % 6) for i in range(6)]
    segs = [(verts[i], verts[j]) for i, j in ring] + [(verts[6 + i], verts[6 + j]) for i, j in ring] \
        + [(verts[i], verts[6 + i]) for i in range(6)]
    edge = np.min([_segment_dist(pts.astype(float), a, b) for a, b in segs], axis=0)
    good = (n * ref).sum(1) > 0
    far = edge > 0.08
    print("L-prism, %d points: wrong signs away from edges %d of %d, near edges %d of %d"
          % (N, int((~good & far).sum()), int(far.sum()), int((~good & ~far).sum()), int((~far).sum())))
    assert good[far].all()


def test_open_scan_toward_its_viewpoint():
    from sonet_b200 import pointclouds
    rs = np.random.RandomState(8)
    xy = rs.uniform(-1, 1, size=(20000, 2))
    z = 0.2 * np.sin(3 * xy[:, 0]) * np.cos(2 * xy[:, 1])
    up = np.stack([-0.6 * np.cos(3 * xy[:, 0]) * np.cos(2 * xy[:, 1]),
                   0.4 * np.sin(3 * xy[:, 0]) * np.sin(2 * xy[:, 1]), np.ones(len(z))], 1)
    data, off = _upload([np.c_[xy, z].astype(np.float32)])
    n = pointclouds.estimate_normals(data, off, k=16, orient="propagate-viewpoint",
                                     viewpoint=[[0.3, -0.2, 4.0]]).cpu().numpy()
    assert ((n * up).sum(1) > 0).all()


# ---- invariance -----------------------------------------------------------------------------------
def test_runs_batch_position_and_graph_replay_agree():
    from sonet_b200 import ops
    rs = np.random.RandomState(9)
    clouds = [rs.normal(size=(P, 3)).astype(np.float32) for P in (900, 131, 2000, 77)]
    data, off = _upload(clouds)
    idx = _estimate(data, off, 16)
    _flip_some(data, rs)
    n1, c1 = _orient(data.clone(), off, idx, AWAY)
    n2, c2 = _orient(data.clone(), off, idx, AWAY)
    assert np.array_equal(n1.view(np.int32), n2.view(np.int32)) and np.array_equal(c1, c2)
    # each cloud alone, and the clouds in another order
    o = off.cpu().numpy()
    h = data.cpu().numpy()
    perm = [2, 0, 3, 1]
    data2, off2 = _upload([h[o[s]:o[s + 1], :3] for s in perm])
    data2[:, 3:6] = torch.from_numpy(np.concatenate([h[o[s]:o[s + 1], 3:6] for s in perm])).to(DEV)
    idx2 = torch.cat([idx[o[s]:o[s + 1]] for s in perm])
    n3, c3 = _orient(data2, off2, idx2, AWAY)
    o2 = off2.cpu().numpy()
    for pos, s in enumerate(perm):
        assert np.array_equal(n3[o2[pos]:o2[pos + 1]].view(np.int32), n1[o[s]:o[s + 1]].view(np.int32))
        assert np.array_equal(c3[o2[pos]:o2[pos + 1]], c1[o[s]:o[s + 1]])
    # CUDA graph replay on static buffers
    work = data.clone()
    comp = torch.empty(len(h), dtype=torch.int32, device=DEV)
    nbytes = int(ops._C.lib().sonet_point_normals_orient_scratch_bytes(len(h), len(clouds)))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)

    def call():
        ops._call("sonet_point_normals_orient_f32", ops._C.ptr(work), len(h), 6, ops._C.ptr(off),
                  len(clouds), 2000, ops._C.ptr(idx), 16, AWAY, None, ops._C.ptr(scratch), nbytes,
                  ops._C.ptr(work) + 12, 6, ops._C.ptr(comp), ops._stream(work))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    for _ in range(2):
        work.copy_(data)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(work[:, 3:6].cpu().numpy().view(np.int32), n1.view(np.int32))
        assert np.array_equal(comp.cpu().numpy(), c1)


# ---- malformed offsets at the C-ABI ---------------------------------------------------------------
BAD_OFFSETS = {
    "negative": [-7, 10, 25, 40, 60],
    "past_T": [0, 10, 25, 80, 97],
    "gap": [3, 10, 10, 40, 52],
    "decreasing": [0, 20, 12, 30, 25, 60],
    "unsorted_same_start": [0, 5, 0, 10, 60],
    "b_large": [0, 30, 60, 60, 60, 60, 60],
}


@pytest.mark.parametrize("case", list(BAD_OFFSETS))
def test_malformed_offsets_stay_in_range(case):
    """Offsets that are negative, past T, decreasing or leave rows in no cloud, and idx entries
    outside [0, P): every canary is intact and the output equals the restatement, which gives each
    row at most one cloud by ragged_find."""
    from sonet_b200 import _C
    offsets = BAD_OFFSETS[case]
    T, K, S = 60, 5, len(offsets) - 1
    rs = np.random.RandomState(len(case))
    pts = rs.normal(size=(T, 3)).astype(np.float32)
    nrm = rs.normal(size=(T, 3)).astype(np.float32)
    idx = rs.randint(-3, 45, size=(T, K)).astype(np.int32)
    los, his = orient_emu.ragged_ranges(offsets, T)
    maxp = int((his - los).max())
    want_n, want_c = orient_emu.orient(pts, offsets, idx, nrm, AWAY, max_points=maxp)
    g_pts = Guarded(3 * T, torch.from_numpy(pts))
    g_nrm = Guarded(3 * T, torch.from_numpy(nrm))
    g_idx = Guarded(K * T, torch.from_numpy(idx), torch.int32)
    g_off = _off64(offsets)
    g_comp = Guarded(T, dtype=torch.int32)
    nbytes = int(_C.lib().sonet_point_normals_orient_scratch_bytes(T, S))
    g_scr = Guarded(nbytes // 4, dtype=torch.int32)
    rc = _C.lib().sonet_point_normals_orient_f32(g_pts.ptr, T, 3, g_off.ptr, S, maxp, g_idx.ptr, K,
                                                 AWAY, None, g_scr.ptr, nbytes, g_nrm.ptr, 3,
                                                 g_comp.ptr, None)
    assert rc == 0, _C.last_error()
    torch.cuda.synchronize()
    for name, g in (("points", g_pts), ("normals", g_nrm), ("idx", g_idx), ("offsets", g_off),
                    ("component", g_comp), ("scratch", g_scr)):
        assert g.intact(), "%s: canary overwritten" % name
    assert np.array_equal(g_comp.body(), want_c)
    assert np.array_equal(g_nrm.body().reshape(T, 3).view(np.int32), want_n.view(np.int32))


# ---- end to end -----------------------------------------------------------------------------------
def test_build_dataset_propagate_equals_estimate_then_orient():
    from sonet_b200 import pointclouds
    clouds = [_torus(P, seed=s)[0] for s, P in enumerate((1500, 900, 2200))]
    ds = pointclouds.build_dataset(clouds, [0, 1, 2], k=16, orient="propagate", rows=4, n=256)
    data, off = _upload(clouds)
    n = pointclouds.estimate_normals(data, off, k=16, orient=None, out=data[:, 3:6])
    pointclouds.orient_normals(data, off, n, k=16)
    assert torch.equal(ds.data[:, 3:6].cpu().view(torch.int32), data[:, 3:6].cpu().view(torch.int32))
    again = pointclouds.estimate_normals(data, off, k=16, orient="propagate")
    assert torch.equal(again.cpu().view(torch.int32), data[:, 3:6].cpu().view(torch.int32))
