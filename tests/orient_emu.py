"""A numpy restatement of sonet_point_normals_orient_f32 (include/sonet_b200.h), without the package:
the vertex and edge rules with the fp64 dot, Kruskal over the stated edge order with a union-find that
tracks sign parity, the anchor rules and the resulting signs and component ids. A different
algorithm than the kernel's Borůvka rounds, held to the same tree by the strict edge order."""
import numpy as np

from test_point_normals_host import centroid_restated

AWAY_FROM_CENTROID, TOWARD_VIEWPOINT = 1, 2


def ragged_ranges(offsets, T):
    """(lo [S], hi [S]) of every cloud: each offset clamped into [0, T], hi never below lo."""
    c = np.clip(np.asarray(offsets, np.int64), 0, T)
    return c[:-1], np.maximum(c[:-1], c[1:])


def ragged_find(offsets, T, g):
    """common.cuh's ragged_find for the rows g, step for step: the binary search over the clamped
    offsets for the last cloud b with offset <= g (on unsorted offsets, the one the search lands
    on). -> (b, inside) where inside is lo_b <= g < hi_b."""
    c = np.clip(np.asarray(offsets, np.int64), 0, T)
    g = np.asarray(g, np.int64)
    a = np.zeros(g.shape, np.int64)
    z = np.full(g.shape, len(c) - 2, np.int64)
    while (a < z).any():
        act = a < z
        mid = (a + z + 1) >> 1
        le = c[np.minimum(mid, len(c) - 2)] <= g
        a = np.where(act & le, mid, a)
        z = np.where(act & ~le, mid - 1, z)
    lo, hi = ragged_ranges(offsets, T)
    return a, (lo[a] <= g) & (g < hi[a])


def dot64(a, b):
    """(ax*bx + ay*by) + az*bz in fp64, op by op, of f32 rows a, b [.., 3]."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def weight(dot):
    """w = fp32(1 - |dot|), rounded once; -0 counts as +0 (they are one value in the order)."""
    with np.errstate(over="ignore"):                    # 1 - |dot| past the f32 range is -inf
        return (np.float32(1.0 - np.abs(dot)) + np.float32(0)).astype(np.float32)


def vertices(data, offsets, normals, max_points):
    """(cloud [T] i64 or -1, lo [T] first row of that cloud): rows with finite xyz and a finite,
    non-zero normal that lie in the cloud ragged_find gives them, at a local index < max_points."""
    data, normals = np.asarray(data, np.float32), np.asarray(normals, np.float32)
    T = len(data)
    los, his = ragged_ranges(offsets, T)
    b, inside = ragged_find(offsets, T, np.arange(T))
    lo = los[b] if T else np.zeros(0, np.int64)
    ok = inside & (np.arange(T) - lo < max_points)
    ok &= np.isfinite(data[:, :3]).all(1) & np.isfinite(normals[:, :3]).all(1)
    ok &= (normals[:, :3] != 0).any(1)
    return np.where(ok, b, -1), lo, his[b] if T else np.zeros(0, np.int64)


def edges(idx, cloud, lo, hi, normals):
    """The undirected edges (g_lo, g_hi, w, flip) as global rows, one per pair, from every vertex's
    idx entries in [0, P), not itself, naming a vertex of the same cloud."""
    idx = np.asarray(idx, np.int64)
    T, K = idx.shape
    u = np.repeat(np.arange(T), K)
    j = idx.reshape(-1)
    ul = u - lo[u]
    ok = (cloud[u] >= 0) & (j >= 0) & (j < (hi - lo)[u]) & (j != ul)
    v = np.where(ok, lo[u] + j, 0)
    ok &= cloud[v] == cloud[u]
    a, b = np.minimum(u[ok], v[ok]), np.maximum(u[ok], v[ok])
    pairs = np.unique(np.stack([a, b], 1), axis=0) if len(a) else np.zeros((0, 2), np.int64)
    n = np.asarray(normals, np.float32)
    d = dot64(n[pairs[:, 0], :3], n[pairs[:, 1], :3])
    return pairs[:, 0], pairs[:, 1], weight(d), d < 0


def kruskal(T, ga, gb, w, flip):
    """Kruskal in the order (w, min, max) (within a cloud the global rows order as the local ones)
    with a parity union-find. -> (root [T], parity [T] relative to the root, tree edge indices)."""
    parent = np.arange(T)
    par = np.zeros(T, np.int64)

    def find(x):
        p = 0
        path = []
        while parent[x] != x:
            path.append(x)
            p ^= par[x]
            x = parent[x]
        q = p
        for y in path:                      # compress, each node straight onto the root
            py = par[y]
            parent[y], par[y] = x, q
            q ^= py
        return x, p

    order = np.lexsort((gb, ga, w))
    tree = []
    for e in order:
        (ra, pa), (rb, pb) = find(ga[e]), find(gb[e])
        if ra == rb:
            continue
        parent[rb], par[rb] = ra, pa ^ pb ^ int(flip[e])
        tree.append(e)
    root = np.empty(T, np.int64)
    parity = np.empty(T, np.int64)
    for x in range(T):
        root[x], parity[x] = find(x)
    return root, parity, np.asarray(tree, np.int64)


def anchor_dist(data, offsets, cloud, code, view):
    """(squared fp64 distance, ref [T, 3]) of every row to its cloud's centroid or view point."""
    data = np.asarray(data, np.float32)
    T = len(data)
    p = data[:, :3].astype(np.float64)
    los, his = ragged_ranges(offsets, T)
    c = np.maximum(cloud, 0)
    if code == AWAY_FROM_CENTROID:
        cen = np.array([centroid_restated(data[l:h, :3]) if h > l else [np.nan] * 3
                        for l, h in zip(los, his)]).reshape(-1, 3)
        ref = p - cen[c]
    else:
        ref = np.asarray(view, np.float32).astype(np.float64).reshape(-1, 3)[c] - p
    with np.errstate(invalid="ignore", over="ignore"):
        d = (ref[:, 0] * ref[:, 0] + ref[:, 1] * ref[:, 1]) + ref[:, 2] * ref[:, 2]
    return d, ref


def orient(data, offsets, idx, normals, code, view=None, max_points=None, want_tree=False):
    """-> (normals [T, 3] f32 with the kernel's signs, component [T] i32), and with want_tree the
    tree's edges (ga, gb) as global rows."""
    data = np.asarray(data, np.float32)
    n_in = np.asarray(normals, np.float32)[:, :3].copy()
    T = len(data)
    if max_points is None:
        los, his = ragged_ranges(offsets, T)
        max_points = int((his - los).max()) if len(los) else 0
    cloud, lo, hi = vertices(data, offsets, n_in, max_points)
    ga, gb, w, flip = edges(idx, cloud, lo, hi, n_in)
    root, parity, tree = kruskal(T, ga, gb, w, flip)
    with np.errstate(invalid="ignore", over="ignore"):
        d, ref = anchor_dist(data, offsets, cloud, code, view)
        adot = dot64(n_in, ref)
    out = n_in.copy()
    comp = np.full(T, -1, np.int32)
    vert = np.flatnonzero(cloud >= 0)
    vert = vert[np.argsort(root[vert], kind="stable")]        # grouped by root, ascending within
    far = code == AWAY_FROM_CENTROID
    cuts = np.flatnonzero(np.diff(root[vert])) + 1
    for members in np.split(vert, cuts) if len(vert) else []:
        dm = d[members]
        nan = np.isnan(dm)
        if nan.all():
            a = members[0]
        else:
            best = dm[~nan].max() if far else dm[~nan].min()
            a = members[~nan & (dm == best)][0]      # members ascend: the lowest index on ties
        neg = (int(adot[a] < 0) ^ parity[a] ^ parity[members]).astype(bool)
        out[members[neg]] = -out[members[neg]]
        comp[members] = a - lo[a]
    res = (out, comp)
    return res + ((ga[tree], gb[tree]),) if want_tree else res
