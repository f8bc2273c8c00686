"""-m gpu: area-weighted surface sampling of meshes (csrc/mesh_sample.cu, sonet_b200.meshes) and the
single-cloud SOM class.

With given draws the kernel is held bit for bit to the numpy float64 restatement below, which follows
the order the header documents (face geometry, the run / tile blocked CDF, upper bound, reflection,
(a + u*e1) + v*e2). The in-kernel draws are held to the distributions they must have (chi-square of
face counts against area weights, Kolmogorov-Smirnov of the barycentric marginals) and to their
determinism: the key is the mesh id, so chunking and neighbours do not change a mesh's bits."""
import numpy as np
import pytest
import torch

from helpers import assert_close, golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RUN, TILE = 8, 2048


# ---- the numpy restatement ------------------------------------------------------------------------
def face_geometry(v, f):
    """a, e1, e2, n [F,3], |n| and area [F] in float64, the kernel's operation order."""
    V = len(v)
    fc = np.clip(f.astype(np.int64), 0, max(V - 1, 0))
    a, b, c = v[fc[:, 0]], v[fc[:, 1]], v[fc[:, 2]]
    e1, e2 = b - a, c - a
    nx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    ny = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    nz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    with np.errstate(invalid="ignore", over="ignore"):
        ln = np.sqrt((nx * nx + ny * ny) + nz * nz)
    return a, e1, e2, np.stack([nx, ny, nz], 1), ln, 0.5 * ln


def blocked_cdf(w):
    """cdf[f] = toff + (roff + run[f]): sequential sums (np.add.accumulate is sequential) over runs
    of RUN faces, of the run totals within a tile of TILE faces, and of the tile totals."""
    F = len(w)
    K = -(-F // TILE)
    pad = np.zeros(K * TILE)
    pad[:F] = w
    run = np.cumsum(pad.reshape(K, TILE // RUN, RUN), axis=2)
    tot = run[:, :, -1]
    roff = np.concatenate([np.zeros((K, 1)), np.cumsum(tot, axis=1)[:, :-1]], axis=1)
    loc = roff[:, :, None] + run
    ttot = loc[:, -1, -1]
    toff = np.concatenate([[0.0], np.cumsum(ttot)[:-1]])
    return (toff[:, None, None] + loc).reshape(-1)[:F]


def restate(v, f, draws):
    """(out [N,6] f32, face [N], area) of one mesh sampled with draws [N,3] (r, u, v)."""
    N = len(draws)
    a, e1, e2, n, ln, area = face_geometry(v, f)
    with np.errstate(invalid="ignore"):
        w = np.where(np.isfinite(area) & (area > 0), area, 0.0)
    cdf = blocked_cdf(w) if len(f) else np.zeros(0)
    total = cdf[-1] if len(f) else 0.0
    bad = not np.isfinite(area).all()
    area_out = np.nan if bad else total
    pos = np.flatnonzero(w > 0)
    if bad or not (total > 0 and np.isfinite(total)) or len(pos) == 0:
        return np.full((N, 6), np.nan, np.float32), np.full(N, -1), area_out
    r, u, vv = draws[:, 0], draws[:, 1], draws[:, 2]
    fi = np.minimum(np.searchsorted(cdf, r * total, side="right"), pos[-1])
    sw = (u + vv) > 1.0
    u = np.where(sw, 1.0 - u, u)
    vv = np.where(sw, 1.0 - vv, vv)
    p = (a[fi] + u[:, None] * e1[fi]) + vv[:, None] * e2[fi]
    nn = n[fi] / ln[fi][:, None]
    return np.concatenate([p, nn], 1).astype(np.float32), fi, area_out


def check_given(mesh_list, N, seed=0, ids=None):
    """The entry itself (not sample_surface, which raises on a mesh without area) with draw_host's
    draws, every mesh against the restatement, NaN rows included."""
    from sonet_b200 import meshes, ops
    m = meshes.Meshes(mesh_list, mesh_ids=ids, device=DEV)
    d = meshes.draw_host(np.random.RandomState(seed), len(mesh_list), N)
    out, face, area = ops.mesh_sample(m.verts, m.v_off, m.faces, m.f_off, m.mesh_ids, N,
                                      draws=torch.from_numpy(d).to(DEV), want_faces=True,
                                      want_area=True)
    out, face, area = out.cpu().numpy(), face.cpu().numpy(), area.cpu().numpy()
    for b, (v, f) in enumerate(mesh_list):
        rows = slice(b * N, (b + 1) * N)
        want, wf, wa = restate(np.asarray(v, np.float64), np.asarray(f), d[rows])
        assert np.array_equal(out[rows].view(np.uint32), want.view(np.uint32)), "mesh %d points" % b
        assert np.array_equal(face[rows], wf), "mesh %d faces" % b
        assert area[b] == wa or (np.isnan(area[b]) and np.isnan(wa)), (b, area[b], wa)
    return out, face, area


# ---- meshes ---------------------------------------------------------------------------------------
def tetrahedron():
    return np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], float), \
        np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]])


def icosphere(level):
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


def random_mesh(rs, F, V=None):
    V = V or max(16, F // 2)
    return rs.uniform(-1, 1, size=(V, 3)), rs.randint(0, V, size=(F, 3))


def skinny(rs, F):
    v, f = [], []
    for i in range(F):
        x = rs.uniform(-1, 1, 3)
        v += [x, x + rs.uniform(-1, 1, 3), x + 1e-9 * rs.uniform(-1, 1, 3)]
        f.append([3 * i, 3 * i + 1, 3 * i + 2])
    return np.array(v), np.array(f)


def with_degenerate_faces(rs, F):
    v, f = random_mesh(rs, F)
    v = np.concatenate([v, [[0, 0, 0], [1, 1, 1], [2, 2, 2]]])    # three collinear points
    V = len(v)
    f[::5] = [V - 3, V - 2, V - 1]                  # collinear
    f[1::7, 1] = f[1::7, 0]                         # a repeated vertex
    f[2::11] = [V - 1, V - 1, V - 1]                # one point
    return v, f


# ---- given draws: bit-exact -----------------------------------------------------------------------
def test_small_meshes_bit_exact():
    rs = np.random.RandomState(1)
    tri = (np.array([[0.1, 0.2, 0.3], [1.7, -0.4, 0.2], [0.3, 2.1, -1.1]]), np.array([[0, 1, 2]]))
    check_given([tri, tetrahedron(), icosphere(1), icosphere(3), skinny(rs, 50),
                 with_degenerate_faces(rs, 3000)], 3000, seed=2)


@pytest.mark.parametrize("F", [7, 8, 9, 255, 256, 257, 2047, 2048, 2049, 4095, 4096, 4097, 10000])
def test_run_and_tile_edges_bit_exact(F):
    rs = np.random.RandomState(F)
    check_given([random_mesh(rs, F), with_degenerate_faces(rs, F + 3)], 4096, seed=F)


def test_several_blocks_mixed_sizes_in_one_launch():
    rs = np.random.RandomState(5)
    sizes = [1, 3000, 20000, 5, 2048, 70000, 9]
    check_given([random_mesh(rs, F) for F in sizes], 2000, seed=6, ids=[40, 2, 13, 7, 0, 99, 1])


def test_large_mesh_bit_exact():
    """2^22 faces: 2048 tiles of one mesh, next to a small one."""
    rs = np.random.RandomState(9)
    check_given([random_mesh(rs, 1 << 22, 1 << 20), tetrahedron()], 1 << 16, seed=10)


# ---- CDF edges ------------------------------------------------------------------------------------
def unit_faces(F, lead_zero=0, trail_zero=0):
    """F faces of area exactly 1 ((0,0,0),(2,0,0),(0,1,0) shifted), with zero-area faces around."""
    v, f = [], []
    for i in range(lead_zero + F + trail_zero):
        z = float(i)
        k = len(v)
        if lead_zero <= i < lead_zero + F:
            v += [[0, 0, z], [2, 0, z], [0, 1, z]]
        else:
            v += [[0, 0, z], [1, 0, z], [2, 0, z]]
        f.append([k, k + 1, k + 2])
    return np.array(v, float), np.array(f)


def _given(mesh, draws):
    from sonet_b200 import meshes
    m = meshes.Meshes([mesh], device=DEV)
    out, face, area = meshes.sample_surface(m, len(draws), draws=np.asarray(draws, float),
                                            want_faces=True, want_area=True)
    want = restate(mesh[0], mesh[1], np.asarray(draws, float))
    assert np.array_equal(face.cpu().numpy(), want[1])
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want[0].view(np.uint32))
    return face.cpu().numpy(), float(area[0])


def test_cdf_edges():
    top = 1.0 - 2.0 ** -53
    mesh = unit_faces(4, lead_zero=3, trail_zero=5)
    face, area = _given(mesh, [[0.0, 0.2, 0.3], [top, 0.2, 0.3], [0.25, 0.1, 0.1], [0.5, 0.1, 0.1],
                               [0.75, 0.1, 0.1], [0.5 - 2.0 ** -53, 0.1, 0.1], [0.9, 0.9, 0.9]])
    assert area == 4.0
    # r = 0: the first face of positive area; the top draw: the last one (trailing zeros never);
    # t exactly on a CDF value k: face k (the first with cdf > t); just below: face k - 1
    assert face.tolist() == [3, 6, 4, 5, 6, 4, 6]


# ---- in-kernel draws: statistics ------------------------------------------------------------------
def test_face_counts_follow_area_weights_chi_square():
    from scipy import stats
    from sonet_b200 import meshes
    rs = np.random.RandomState(11)
    F = 100
    areas = 10.0 ** rs.uniform(-6, 0, F)
    v, f = [], []
    for i, A in enumerate(areas):   # right triangles with legs s, 2s: area s^2
        s = np.sqrt(A)
        v += [[0, 0, i], [s, 0, i], [0, 2 * s, i]]
        f.append([3 * i, 3 * i + 1, 3 * i + 2])
    v, f = np.array(v), np.array(f)
    _, _, _, _, _, area = face_geometry(v, f)
    N = 1 << 20
    m = meshes.Meshes([(v, f)], device=DEV)
    _, face, _ = meshes.sample_surface(m, N, seed=3, want_faces=True)
    counts = np.bincount(face.cpu().numpy(), minlength=F)
    exp = N * area / area.sum()
    big = exp >= 5
    obs = np.append(counts[big], counts[~big].sum())
    e = np.append(exp[big], exp[~big].sum())
    assert stats.chisquare(obs, e).pvalue > 1e-4
    assert counts[area < 1e-5].sum() <= 10 * max(exp[area < 1e-5].sum(), 1)


def test_barycentric_marginals_ks_and_points_on_faces():
    from scipy import stats
    from sonet_b200 import meshes
    tri = (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], float), np.array([[0, 1, 2]]))
    N = 1 << 17
    out = meshes.sample_surface(meshes.Meshes([tri], device=DEV), N, seed=4).cpu().numpy()
    x, y = out[:, 0].astype(float), out[:, 1].astype(float)
    assert (out[:, 2] == 0).all() and (x >= 0).all() and (y >= 0).all() and (x + y <= 1 + 1e-7).all()
    for c in (x, y):
        assert stats.kstest(c, stats.beta(1, 2).cdf).pvalue > 1e-4
    assert np.array_equal(out[:, 3:], np.tile(np.float32([0, 0, 1]), (N, 1)))


def test_in_kernel_points_lie_on_their_faces_with_the_restated_normals():
    from sonet_b200 import meshes
    rs = np.random.RandomState(12)
    ms = [icosphere(2), random_mesh(rs, 5000), with_degenerate_faces(rs, 3000)]
    N = 20000
    out, face, _ = meshes.sample_surface(meshes.Meshes(ms, device=DEV), N, seed=5, want_faces=True)
    out, face = out.cpu().numpy(), face.cpu().numpy()
    for b, (v, f) in enumerate(ms):
        rows = slice(b * N, (b + 1) * N)
        a, e1, e2, n, ln, area = face_geometry(v, f)
        fi = face[rows]
        assert (area[fi] > 0).all()
        assert np.array_equal(out[rows, 3:], (n[fi] / ln[fi][:, None]).astype(np.float32))
        # barycentric coordinates of the f32 point, by least squares in the face's plane
        d = out[rows, :3].astype(np.float64) - a[fi]
        G = np.stack([e1[fi], e2[fi]], 2)                     # [N,3,2]
        GtG = np.einsum("nki,nkj->nij", G, G)
        rhs = np.einsum("nki,nk->ni", G, d)
        st = np.linalg.solve(GtG, rhs[..., None])[..., 0]
        resid = d - np.einsum("nki,ni->nk", G, st)
        scale = np.abs(a[fi]).max(1) + np.abs(e1[fi]).max(1) + np.abs(e2[fi]).max(1)
        assert (np.linalg.norm(resid, axis=1) <= 4e-7 * scale).all()
        # the f32 rounding moves a point by 2^-24 of its size; in barycentric units by that over
        # the triangle's smallest height
        tol = 1e-6 * scale * scale / np.maximum(ln[fi], 1e-300) * 4
        assert (st >= -tol[:, None]).all() and (st.sum(1) <= 1 + tol).all()


# ---- in-kernel draws: determinism -----------------------------------------------------------------
def test_same_seed_same_bits_chunks_and_neighbours():
    from sonet_b200 import meshes
    rs = np.random.RandomState(13)
    ms = [random_mesh(rs, F) for F in (300, 5000, 2049, 40000, 17)]
    ids = [11, 3, 27, 5, 8]
    N = 3000
    whole = meshes.sample_surface(meshes.Meshes(ms, ids, DEV), N, seed=77).cpu()
    again = meshes.sample_surface(meshes.Meshes(ms, ids, DEV), N, seed=77).cpu()
    assert torch.equal(whole.view(torch.int32), again.view(torch.int32))
    other = meshes.sample_surface(meshes.Meshes(ms, ids, DEV), N, seed=78).cpu()
    assert not torch.equal(whole, other)
    # a chunked build, in another order
    for chunk in ([3, 0], [4], [2, 1]):
        part = meshes.sample_surface(meshes.Meshes([ms[i] for i in chunk], [ids[i] for i in chunk],
                                                   DEV), N, seed=77).cpu()
        for k, i in enumerate(chunk):
            assert torch.equal(part[k * N:(k + 1) * N].view(torch.int32),
                               whole[i * N:(i + 1) * N].view(torch.int32)), (chunk, i)
    # change one mesh: the others keep their bits
    ms2 = list(ms)
    ms2[1] = random_mesh(rs, 7000)
    changed = meshes.sample_surface(meshes.Meshes(ms2, ids, DEV), N, seed=77).cpu()
    for i in (0, 2, 3, 4):
        assert torch.equal(changed[i * N:(i + 1) * N].view(torch.int32),
                           whole[i * N:(i + 1) * N].view(torch.int32)), i
    assert not torch.equal(changed[N:2 * N], whole[N:2 * N])


# ---- degenerate and invalid meshes ----------------------------------------------------------------
def test_degenerate_and_non_finite_meshes():
    from sonet_b200 import meshes, ops
    rs = np.random.RandomState(14)
    good1, good2 = random_mesh(rs, 900), icosphere(1)
    flat = (np.array([[0, 0, 0], [1, 1, 1], [2, 2, 2], [3, 3, 3]], float),
            np.array([[0, 1, 2], [1, 2, 3], [0, 0, 0]]))
    nanv = good2[0].copy()
    nanv[3, 1] = np.nan
    infm = (good2[0] * 1e300, good2[1])                   # cross products overflow to inf
    empty = (np.zeros((3, 3)), np.zeros((0, 3), np.int64))
    ms = [good1, flat, good2, (nanv, good2[1]), infm, empty]
    ids = [0, 1, 2, 3, 4, 5]
    N = 500
    m = meshes.Meshes(ms, ids, DEV)
    out, face, area = ops.mesh_sample(m.verts, m.v_off, m.faces, m.f_off, m.mesh_ids, N, seed=9,
                                      want_faces=True, want_area=True)
    out, face, area = out.cpu().numpy(), face.cpu().numpy(), area.cpu().numpy()
    assert area[1] == 0.0 and area[5] == 0.0
    assert np.isnan(area[3]) and np.isnan(area[4])
    assert np.isfinite(area[[0, 2]]).all() and (area[[0, 2]] > 0).all()
    for b in (1, 3, 4, 5):
        assert np.isnan(out[b * N:(b + 1) * N]).all() and (face[b * N:(b + 1) * N] == -1).all()
    # the valid neighbours have the bits they have alone
    alone = ops.mesh_sample(*(lambda q: (q.verts, q.v_off, q.faces, q.f_off, q.mesh_ids))(
        meshes.Meshes([good1, good2], [0, 2], DEV)), N, seed=9)[0].cpu().numpy()
    assert np.array_equal(out[:N].view(np.uint32), alone[:N].view(np.uint32))
    assert np.array_equal(out[2 * N:3 * N].view(np.uint32), alone[N:].view(np.uint32))
    with pytest.raises(ValueError, match="mesh 1 \\(id 1\\)"):
        meshes.sample_surface(m, N)
    # given draws: the restatement agrees on the NaN rows and area_out
    check_given([good1, flat, (nanv, good2[1]), good2], 300, seed=15)


def test_out_of_range_face_indices_are_clamped():
    from sonet_b200 import meshes
    v, f = icosphere(1)
    V = len(v)
    bad = f.copy()
    bad[::3, 0] = -5
    bad[1::3, 2] = V + 100
    clamped = np.clip(bad, 0, V - 1)
    N = 2000
    a = meshes.sample_surface(meshes.Meshes([(v, bad)], device=DEV), N, seed=1).cpu()
    b = meshes.sample_surface(meshes.Meshes([(v, clamped)], device=DEV), N, seed=1).cpu()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    check_given([(v, bad)], N, seed=16)


# ---- the SOM class --------------------------------------------------------------------------------
def test_som_class_matches_the_reference_and_batch_som():
    from sonet_b200 import som
    g = golden("som_single")
    rows = int(g["rows"])
    x = torch.from_numpy(g["x"]).to(DEV)
    s = som.SOM(rows, rows, 3, 0)
    assert s.node.shape == (3, rows * rows)
    assert np.array_equal(s.node_init_value.numpy(), g["node_init_value"])
    s.node_init()
    s.batch_update(x, 0)
    assert_close(s.node, g["node_after_1"], "batch_update(x, 0)", 1e-6)
    s.batch_update(x, 7)
    assert_close(s.node, g["node_after_2"], "batch_update(x, 7)", 1e-6)
    s.optimize(x)
    assert_close(s.node, g["node_optimized"], "optimize")
    mask, row_max = s.query(x)
    assert mask.shape == (x.shape[1], rows * rows) and row_max.shape == (rows * rows,)
    d = ((x.t()[:, :, None].double() - s.node[None].double()) ** 2).sum(1)
    assert torch.equal(mask.argmax(1), d.argmin(1))
    assert (mask.argmax(1).cpu().numpy() == g["query_argmax"]).mean() > 0.99
    bs = som.BatchSOM(rows, rows, 3, 0, 1)
    bs.optimize(x[None])
    assert torch.equal(bs.node[0], s.node)


def test_notebook_som_cell_runs_under_install():
    import sys
    from sonet_b200 import install
    saved = {k: sys.modules.get(k) for k in ("util", "util.som", "index_max", "models")}
    try:
        install.install(None)
        from util import som
        rs = np.random.RandomState(0)
        pc_np = rs.uniform(-1, 1, size=(10000, 3))
        pc_np_sampled = pc_np[np.random.choice(pc_np.shape[0], 4096, replace=False), :]
        pc = torch.from_numpy(pc_np_sampled.transpose().astype(np.float32)).cuda()  # 3xN tensor
        som_builder = som.SOM(8, 8, 3, 0)
        som_builder.optimize(pc)
        som_node_np = som_builder.node.cpu().numpy().transpose().astype(np.float32)  # node_numx3
        assert som_node_np.shape == (64, 3) and np.isfinite(som_node_np).all()
        som.SOM(8, 8, 3, True).optimize(pc)          # the notebook's gpu_ids=True
    finally:
        for k, mod in saved.items():
            if mod is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = mod


def test_som_nodes_batched_equals_per_cloud_som():
    from sonet_b200 import meshes, ops, som
    rs = np.random.RandomState(17)
    ms = [icosphere(2), random_mesh(rs, 3000), tetrahedron()]
    N, n = 5000, 1024
    pts = meshes.sample_surface(meshes.Meshes(ms, device=DEV), N, seed=2).view(len(ms), N, 6)
    rng = np.random.RandomState(5)
    nodes = meshes.som_nodes(pts, 8, 8, n, rng=rng)
    rng = np.random.RandomState(5)
    for b in range(len(ms)):
        sel = rng.choice(N, n, replace=False)
        s = som.SOM(8, 8, 3, 0)
        s.optimize(pts[b, torch.from_numpy(sel).to(DEV), :3].t().contiguous())
        assert torch.equal(nodes[b], s.node.t()), b
    k = meshes.som_nodes(pts, 8, 8, n, seed=3)
    assert k.shape == (3, 64, 3) and torch.isfinite(k).all()
    assert torch.equal(k, meshes.som_nodes(pts, 8, 8, n, seed=3))
    assert ops.SAMPLE_SUBSET == 0


# ---- end to end -----------------------------------------------------------------------------------
def test_build_dataset_feeds_the_classifier_like_host_copies():
    import argparse
    from sonet_b200 import augmentation, classifier, meshes, networks, synth
    rs = np.random.RandomState(18)
    ms = [icosphere(2), random_mesh(rs, 2000), tetrahedron(), icosphere(1)]
    labels = [3, 1, 4, 1]
    N, P = 1024, 256
    ds = meshes.build_dataset(meshes.Meshes(ms, device=DEV), labels, N=N, rows=8, n=512, seed=6)
    assert len(ds) == 4 and ds.node_num == 64
    host = augmentation.DeviceDataset([ds.data[b * N:(b + 1) * N].cpu().numpy() for b in range(4)],
                                      labels, [ds.som_nodes[b].t().cpu().numpy() for b in range(4)])
    opt = synth.make_opt("classifier", batch_size=2, input_pc_num=P, device=DEV)
    cpu_opt = synth.make_opt("classifier", batch_size=2, input_pc_num=P)
    st_e = synth.synth_state_dict(networks.Encoder(cpu_opt), seed=1)
    st_c = synth.synth_state_dict(networks.Classifier(cpu_opt), seed=2)
    lopt = argparse.Namespace(dataset="modelnet", input_pc_num=P, node_num=64, som_k=opt.som_k)
    scores = []
    for d in (ds, host):
        batch = d.batch([2, 0], lopt, train=False, seed=11)
        m = classifier.Model(opt)
        m.encoder.load_state_dict(st_e)
        m.classifier.load_state_dict(st_c)
        m.set_input(*batch)
        m.test_model()
        scores.append((batch, m.score.detach().cpu()))
    for a, b in zip(scores[0][0], scores[1][0]):
        assert torch.equal(a, b)
    assert torch.equal(scores[0][1], scores[1][1]) and torch.isfinite(scores[0][1]).all()
