"""Plain restatements of full-resolution part segmentation's kernels, and their checks where they
run without a GPU: the ragged SOM assignment (k nearest loader nodes, the decentred rows) and the
ragged IoU of the reference's compute_iou rule. test_gpu_seg_full_envelope.py holds the kernels to
them; here they meet the oracle's C top-k, torch.max's CPU argmax and the library's host twin
sonet_seg_iou_ragged_cpu_f32 at the same edges: empty and one-point shapes, tile edges, ties,
non-finite values, custom part tables and bad arguments."""
import ctypes

import numpy as np
import pytest
import torch

from sonet_b200 import _C, ops


# ---- the ragged SOM assignment --------------------------------------------------------------------
def dist_f32(xyz, node):
    """xyz [P,3] f32, node [3,M] f32 -> [P,M] f32 ((dx*dx + dy*dy) + dz*dz), dx = x - node, every
    op rounded to fp32 (numpy's float32 ufuncs never fuse a multiply-add)."""
    with np.errstate(all="ignore"):
        d = [np.subtract(xyz[:, c:c + 1], node[c][None, :], dtype=np.float32) for c in range(3)]
        return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]


def topk_ref(xyz, node, k):
    """[P,k] the k nearest nodes of each point: ascending distance, the lower index on ties, every
    +inf distance after the finite ones and NaN last (a stable sort; numpy sorts NaN last). k
    distinct nodes whatever the distances; a NaN point gets nodes 0..k-1."""
    return np.argsort(dist_f32(xyz, node), axis=1, kind="stable")[:, :k]


def assign_ref(points, offsets, node, cm, k, with_sn, row0, rows, rows_pad):
    """sonet_seg_points_assign_f32 restated: rows [row0, row0+rows) of points [T,6] -> (gidx
    [k*rows_pad] int32, x_aug [3(+3), k*rows_pad] f32, pt [9(+3), k*rows_pad] f32), copy-major
    (column s*rows_pad + r), padding columns zero with gidx 0. Row g belongs to the last cloud b
    with offsets[b] <= g (an empty cloud owns no row)."""
    B, _, M = node.shape
    KR = k * rows_pad
    gidx = np.zeros(KR, np.int32)
    xa = np.zeros((6 if with_sn else 3, KR), np.float32)
    pt = np.zeros((12 if with_sn else 9, KR), np.float32)
    if rows == 0:
        return gidx, xa, pt
    g = np.arange(row0, row0 + rows)
    b = np.searchsorted(offsets[:B], g, side="right") - 1
    ids = np.empty((rows, k), np.int64)
    for bb in np.unique(b):
        sel = b == bb
        ids[sel] = topk_ref(points[g[sel], :3], node[bb], k)
    xyz, nrm = points[g, :3].T, points[g, 3:].T
    for s in range(k):
        cols = s * rows_pad + np.arange(rows)
        gidx[cols] = b * M + ids[:, s]
        ctr = cm[b, :, ids[:, s]].T                                   # [3, rows]
        with np.errstate(all="ignore"):
            dec = np.subtract(xyz, ctr, dtype=np.float32)
        xa[:3, cols] = dec
        pt[0:3, cols], pt[3:6, cols], pt[6:9, cols] = dec, xyz, ctr
        if with_sn:
            xa[3:6, cols] = nrm
            pt[9:12, cols] = nrm
    return gidx, xa, pt


def same_bits(a, b):
    """Bit equality of two float arrays, NaN matching NaN whatever its payload."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool((na == nb).all() and (a.view(np.uint32)[~na] == b.view(np.uint32)[~nb]).all())


def lattice(M):
    """The first M nodes of a square grid of step 0.25 in z = 0: [3, M] f32, exactly representable."""
    side = int(np.ceil(np.sqrt(M)))
    a = (np.arange(side) - (side - 1) / 2.0) * 0.25
    gx, gy = np.meshgrid(a, a, indexing="ij")
    return np.stack([gx.ravel(), gy.ravel(), np.zeros(side * side)])[:, :M].astype(np.float32)


def overflow_case(M):
    """(points [P,6], node [3,M]) whose squared distances overflow for some nodes only (|x| ~
    1.5e19: the square of one such difference is finite, the sum of two is not; node 0 is the
    finite one of points 0 and 3, node M-1 of point 1), then NaN and +-inf points."""
    node = lattice(M)
    big = np.float32(1.5e19)
    pts = [[big, big, 0], [-big, 0, big], [0, big, -big], [big, big, 1e18],
           [np.nan, 0, 0], [0, np.nan, 0], [np.nan] * 3, [np.inf, 0, 0], [0, -np.inf, 0],
           [np.inf, -np.inf, 0], [1e30, 0, 0], [0.1, 0.2, 0.3]]
    node[:, 0] = (big, big, 0)                      # finite for points 0 and 3 only
    if M > 1:
        node[:, M - 1] = (-big, 0, big)             # finite for point 1 only
    p = np.asarray(pts, np.float32)
    return np.concatenate([p, np.ones_like(p)], axis=1), node


def test_topk_restatement_on_ties_and_non_finite(oracle_mod):
    """topk_ref against the oracle's C top-k (the insertion the kernels run, restated on the
    host): finite clouds with exact ties give the same slots; the overflow points get k distinct
    nodes with the finite ones first, then the +inf ones by index."""
    rs = np.random.RandomState(0)
    for M, k in ((1, 1), (3, 3), (64, 4), (121, 3), (256, 4)):
        node = lattice(M)
        if M > 2:
            node[:, 2] = node[:, 1]                  # a duplicated node
        on = node[:, rs.randint(0, M, 50)]
        mid = on + np.float32(0.125) * np.array([[1], [0], [0]], np.float32)
        x = np.concatenate([on, mid, rs.uniform(-2, 2, (3, 100)).astype(np.float32)], 1)
        want = topk_ref(x.T, node, k)
        got, _ = oracle_mod.som_topk(torch.from_numpy(x[None]), torch.from_numpy(node[None]), k)
        np.testing.assert_array_equal(got.view(k, -1).numpy().T, want)

    for M in (1, 2, 4, 64, 256):
        pts, node = overflow_case(M)
        k = min(4, M)
        want = topk_ref(pts[:, :3], node, k)
        assert all(len(set(r)) == k for r in want.tolist())      # distinct nodes
        got, _ = oracle_mod.som_topk(torch.from_numpy(np.ascontiguousarray(pts[:, :3].T[None])),
                                     torch.from_numpy(node[None]), k)
        np.testing.assert_array_equal(got.view(k, -1).numpy().T, want)
        assert want[0].tolist() == list(range(k))    # node 0 finite, then the +inf ones
        assert want[1].tolist() == ([M - 1] + [m for m in range(M - 1)])[:k]
        for n in (4, 5, 6):                          # NaN points: nodes 0..k-1
            assert want[n].tolist() == list(range(k))


# ---- the ragged IoU -------------------------------------------------------------------------------
def argmax_cpu(score):
    """[P,C] -> [P]: torch.max(score, dim=1)'s index on CPU tensors: the first maximum, and the
    first NaN of a row holding one (np.argmax's rule too)."""
    return np.argmax(score, axis=1) if score.shape[0] else np.zeros(0, np.int64)


def iou_ref(score, seg, label, offsets, table=ops.SHAPENET_PART_TABLE):
    """models/losses.py:119-189 (compute_iou) per shape over all its points -> (iou [B] f64 with
    the parts summed left to right as Python does, the same with np.mean, pred [T], correct [B])."""
    B = len(label)
    iou, iou_np = np.empty(B), np.empty(B)
    correct = np.zeros(B, np.int64)
    pred = np.zeros(score.shape[0], np.int64)
    for b in range(B):
        o0, o1 = offsets[b], offsets[b + 1]
        p = argmax_cpu(score[o0:o1])
        pred[o0:o1] = p
        gt = seg[o0:o1]
        correct[b] = int((p == gt).sum())
        ious = []
        for part in table[label[b]]:
            i, u = np.sum((p == part) & (gt == part)), np.sum((p == part) | (gt == part))
            ious.append(1.0 if u == 0 else i / float(u + 0.0001))
        s = 0.0
        for v in ious:
            s += v
        iou[b] = s / len(ious)
        iou_np[b] = np.mean(ious)
    return iou, iou_np, pred, correct


def iou_cases():
    """(name, score [T,C], seg [T], label [B], offsets [B+1], table or None) at the edges."""
    rs = np.random.RandomState(7)
    tab = ops.SHAPENET_PART_TABLE
    out = []

    def make(sizes, C=50, table=None, seed=0):
        r = np.random.RandomState(seed)
        table = tab if table is None else table
        off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        label = r.randint(0, len(table), len(sizes)).astype(np.int64)
        score = r.normal(size=(int(off[-1]), C)).astype(np.float32)
        seg = np.empty(int(off[-1]), np.int64)
        for b, lab in enumerate(label):
            parts = np.asarray(table[lab])
            n = sizes[b]
            seg[off[b]:off[b + 1]] = r.choice(parts, n)
            sc = score[off[b]:off[b + 1]]
            sc[np.arange(n), seg[off[b]:off[b + 1]]] += r.uniform(0, 2, n).astype(np.float32)
        return score, seg, label, off

    out.append(("empty_and_tiny", *make([0, 1, 0, 2, 1, 0], seed=1), None))
    out.append(("tile_edges", *make([255, 256, 257, 1, 513], seed=2), None))
    s, g, l, o = make([400, 300, 200, 256], seed=3)
    s[0:50] = np.nan                                            # whole rows NaN: class 0
    s[50:100, 7] = np.nan                                       # one NaN: its class
    s[100:150, :] = np.inf
    s[100:150, 3] = np.nan                                      # NaN beats +inf
    s[150:200] = -np.inf                                        # all -inf: class 0
    s[200:250, 10:13] = np.inf                                  # first +inf
    s[400:500] = 0.5                                            # all equal: class 0
    s[500:550] = -0.0
    s[500:550, 4] = 0.0                                         # -0 == +0: the first
    out.append(("non_finite_and_equal", s, g, l, o, None))
    s, g, l, o = make([300, 200, 100], seed=4)
    g[0:60] = 49 - g[0:60] % 3                                  # parts of other categories
    g[60:90] = -1 - (np.arange(30) % 5)                         # negative seg values
    g[300:400] = 10 ** 12                                       # far outside any table
    out.append(("seg_outside_category", s, g, l, o, None))
    C1 = make([3, 0, 50], C=1, table=((0,),), seed=5)
    out.append(("one_class", *C1, ((0,),)))
    dup = ((1, 3, 1), (0, 2), (4, 4, 4, 5))
    out.append(("part_listed_twice", *make([100, 37, 0, 250], C=6, table=dup, seed=6), dup))
    eight = (tuple(range(8)), tuple(range(3, 11)), (12,))
    out.append(("eight_parts", *make([500, 700, 1, 300], C=13, table=eight, seed=7), eight))
    big = (tuple(range(256)), tuple(rs.permutation(300)[:256]), (299,))
    out.append(("256_parts", *make([3000, 2000, 5], C=300, table=big, seed=8), big))
    return out


CASES = iou_cases()


def host_iou(score, seg, label, offsets, table, C=None, thread_num=4):
    """sonet_seg_iou_ragged_cpu_f32 on host arrays with a raw CSR table -> (rc, iou, pred,
    correct)."""
    C = score.shape[1] if C is None else C
    poff = np.concatenate([[0], np.cumsum([len(p) for p in table])]).astype(np.int32)
    ids = np.asarray([p for parts in table for p in parts], np.int32)
    B = len(label)
    iou, pred, corr = np.full(B, -7.0), np.full(score.shape[0], -7, np.int64), np.full(B, -7, np.int32)
    score, seg = np.ascontiguousarray(score), np.ascontiguousarray(seg)
    rc = _C.lib().sonet_seg_iou_ragged_cpu_f32(
        score.ctypes.data, seg.ctypes.data, label.ctypes.data, offsets.ctypes.data, B, C,
        int(offsets[-1]) if len(offsets) else 0, poff.ctypes.data, ids.ctypes.data, len(table),
        iou.ctypes.data, pred.ctypes.data, corr.ctypes.data, thread_num)
    return rc, iou, pred, corr


def check_iou(iou, pred, correct, ref, table_parts_max):
    want, want_np, want_pred, want_corr = ref
    np.testing.assert_array_equal(pred, want_pred)
    np.testing.assert_array_equal(correct, want_corr)
    np.testing.assert_array_equal(iou, want)        # left to right, as the header states
    if table_parts_max < 8:
        np.testing.assert_array_equal(iou, want_np)
    else:   # numpy's pairwise mean: within 1 ulp at 8 parts (the header's bound), P ulps beyond
        ulps = 1 if table_parts_max == 8 else table_parts_max
        assert (np.abs(iou - want_np) <= ulps * np.spacing(np.abs(want_np))).all()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_host_twin_against_restatement(lib_built, case):
    name, score, seg, label, off, table = case
    table = ops.SHAPENET_PART_TABLE if table is None else table
    for b in range(len(label)):                      # the restatement's argmax is torch.max's
        sc = score[off[b]:off[b + 1]]
        if len(sc):
            np.testing.assert_array_equal(argmax_cpu(sc), torch.max(torch.from_numpy(sc), 1)[1])
    ref = iou_ref(score, seg, label, off, table)
    for threads in (1, 3):
        rc, iou, pred, corr = host_iou(score, seg, label, off, table, thread_num=threads)
        assert rc == 0, _C.last_error()
        check_iou(iou, pred, corr, ref, max(len(p) for p in table))
    assert (ref[0][np.diff(off) == 0] == 1.0).all()  # an empty shape: every part's union is empty


def test_host_twin_300k_points(lib_built):
    rs = np.random.RandomState(11)
    sizes = [300_001, 0, 7]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    score = rs.normal(size=(int(off[-1]), 50)).astype(np.float32)
    label = np.array([4, 0, 15], np.int64)
    seg = rs.randint(0, 50, int(off[-1])).astype(np.int64)
    ref = iou_ref(score, seg, label, off)
    rc, iou, pred, corr = host_iou(score, seg, label, off, ops.SHAPENET_PART_TABLE, thread_num=8)
    assert rc == 0, _C.last_error()
    check_iou(iou, pred, corr, ref, 6)


def test_host_twin_rejects_what_the_device_marks_nan(lib_built):
    """257 parts, a label outside the table and bad offsets: the host entry refuses them (the
    device entry writes NaN for that shape instead; test_gpu_seg_full_envelope)."""
    bad = _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    rs = np.random.RandomState(2)
    off = np.array([0, 5, 9], np.int64)
    score = rs.normal(size=(9, 300)).astype(np.float32)
    seg = rs.randint(0, 300, 9).astype(np.int64)
    label = np.array([0, 1], np.int64)
    assert host_iou(score, seg, label, off, (tuple(range(257)), (1,)))[0] == bad
    assert "257 parts" in _C.last_error()
    assert host_iou(score, seg, label, off, ((), (1,)))[0] == bad
    assert host_iou(score, seg, np.array([0, 2], np.int64), off, ((0,), (1,)))[0] == bad
    assert "outside the part table" in _C.last_error()
    assert host_iou(score, seg, np.array([0, -1], np.int64), off, ((0,), (1,)))[0] == bad
    assert host_iou(score, seg, label, np.array([0, 10, 9], np.int64), ((0,), (1,)))[0] == bad
    assert "decrease" in _C.last_error()
    assert host_iou(score, seg, label, off, ((0,), (300,)))[0] == bad
    assert "part id 300" in _C.last_error()
    assert host_iou(score, seg, label, off, ((0,), (1,)))[0] == 0


def test_assign_restatement_layout():
    """assign_ref's own layout on a hand-checked case: two clouds, one empty between, padding."""
    pts = np.array([[0, 0, 0, 1, 2, 3], [1, 1, 1, 4, 5, 6], [5, 5, 5, 7, 8, 9]], np.float32)
    off = np.array([0, 2, 2, 3], np.int64)
    node = np.zeros((3, 3, 2), np.float32)
    node[:, 0, 1] = 1
    node[2, :, 0] = (5, 5, 5)
    cm = node + np.float32(0.5)
    gidx, xa, pt = assign_ref(pts, off, node, cm, 2, 1, 1, 2, 3)
    assert gidx.tolist() == [1, 4, 0, 0, 5, 0]        # slot 0: row 1 (cloud 0), row 2 (cloud 2), pad
    np.testing.assert_array_equal(xa[:3, 0], [-0.5, 0.5, 0.5])
    np.testing.assert_array_equal(pt[3:6, 1], [5, 5, 5])
    np.testing.assert_array_equal(pt[9:12, 4], [7, 8, 9])
    assert not xa[:, 2].any() and not pt[:, 5].any()
    assert same_bits(np.float32([np.nan, 1]), np.float32([-np.nan, 1]))
    assert not same_bits(np.float32([0.0]), np.float32([-0.0]))
