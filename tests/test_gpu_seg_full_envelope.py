"""-m gpu: full-resolution part segmentation at its edges, against plain restatements
(test_seg_full_envelope_host.py):

  A. sonet_seg_points_assign_f32 at every node count M = 1..256 and k = 1..4, empty, one-point and
     tile-edge clouds, chunks starting on and beside cloud boundaries, padding, exact ties,
     duplicated loader nodes and non-finite points: its nodes against the oracle's top-k and
     ops.som_assign, its rows against numpy, bit for bit;
  B. score_points over the sampled points against the sampled forward's score_segmenter
     (torch.equal) at every node count, k, activation, normals and SONET_TC mode, at the
     benchmarked shape and at batches small enough that a layer leaves wgmma; each case asserts
     the kernel of every head layer from the C-ABI calls (ops.PROFILE); one float64 case at M = 256;
  C. the ragged IoU kernel against the host twin and the numpy restatement, the fixed-N kernel,
     custom part tables and bad arguments passed straight to the C-ABI."""
import contextlib

import numpy as np
import pytest
import torch

import test_gpu_seg_full as full        # the end-to-end test's clouds and fp64 restatement
import test_seg_full_envelope_host as host
from helpers import build_states
from sonet_b200 import _C, ops, segmenter, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# ---- A. the ragged SOM assignment ------------------------------------------------------------------
def _clouds(M, rs):
    """Clouds of 1, 255, 0, 256, 257, 5000 and 0 points (empty in the middle and at the end) with
    M loader nodes each, drawn like the loader's (from the cloud's points, with repeats when
    P < M), plus points exactly on nodes and halfway between lattice nodes (exact ties)."""
    sizes = [1, 255, 0, 256, 257, 5000, 0]
    pts, nodes = [], []
    for b, P in enumerate(sizes):
        xyz = rs.uniform(-1, 1, (P, 3)).astype(np.float32)
        if b in (3, 5):                     # lattice nodes, points on them and between neighbours
            node = host.lattice(M)
            q = P // 3
            xyz[:q] = node.T[rs.randint(0, M, q)]
            xyz[q:2 * q] = node.T[rs.randint(0, M, q)] + np.float32([0.125, 0, 0])
        elif P:
            node = xyz[rs.choice(P, M, replace=P < M)].T.copy()  # duplicated when P < M
            xyz[:P // 4] = node.T[rs.randint(0, M, P // 4)]
        else:
            node = rs.uniform(-1, 1, (3, M)).astype(np.float32)
        nrm = rs.normal(size=(P, 3)).astype(np.float32)
        pts.append(np.concatenate([xyz, nrm], 1))
        nodes.append(node)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return np.concatenate(pts), off, np.stack(nodes).astype(np.float32)


def _chunks(off):
    """(row0, rows, rows_pad): on every cloud boundary and one beside it, padding 0 / 1 / 255,
    an empty chunk, the whole set in one."""
    T = int(off[-1])
    out = [(0, 0, 256), (0, T, T)]
    for i, o in enumerate(sorted(set(off[1:-1].tolist()))):
        for d in (-1, 0, 1):
            r0 = min(max(o + d, 0), T - 1)
            rows = min(300, T - r0)
            out.append((r0, rows, rows + (0, 1, 255)[(i + d) % 3]))
    return out


def _assign(pts_d, off_d, node_d, cm_d, k, with_sn, r0, rows, rp):
    # the caching allocator hands the outputs blocks that hold NaN / -1 bytes, so that a padding
    # column the kernel did not write shows
    cols = k * rp
    junk = [torch.full((n,), float("nan"), device=DEV) for n in (cols, (6 if with_sn else 3) * cols,
                                                             (12 if with_sn else 9) * cols)]
    del junk
    g, xa, pt = ops.seg_points_assign(pts_d, off_d, node_d, cm_d, k, with_sn, r0, rows, rp)
    return g.cpu().numpy()[0], xa.cpu().numpy()[0], pt.cpu().numpy()[0]


def _check_assign(got, want, what):
    g, xa, pt = got
    wg, wxa, wpt = want
    np.testing.assert_array_equal(g, wg, err_msg=what)
    assert host.same_bits(xa, wxa), what
    assert host.same_bits(pt, wpt), what


@pytest.mark.parametrize("with_sn", [0, 1])
@pytest.mark.parametrize("M", [1, 2, 3, 63, 64, 65, 121, 255, 256])
def test_assign_against_restatement(oracle_mod, M, with_sn):
    rs = np.random.RandomState(M * 2 + with_sn)
    pts, off, node = _clouds(M, rs)
    cm = rs.uniform(-1, 1, node.shape).astype(np.float32)
    pts_d, off_d = torch.from_numpy(pts).to(DEV), torch.from_numpy(off).to(DEV)
    node_d, cm_d = torch.from_numpy(node).to(DEV), torch.from_numpy(cm).to(DEV)
    for k in range(1, min(4, M) + 1):
        for r0, rows, rp in _chunks(off):
            want = host.assign_ref(pts, off, node, cm, k, with_sn, r0, rows, rp)
            _check_assign(_assign(pts_d, off_d, node_d, cm_d, k, with_sn, r0, rows, rp), want,
                          "M=%d k=%d chunk=%s" % (M, k, (r0, rows, rp)))
        # the nodes of every cloud: the oracle's top-k and ops.som_assign, slot order included
        g = _assign(pts_d, off_d, node_d, cm_d, k, with_sn, 0, int(off[-1]), int(off[-1]))[0]
        g = g.reshape(k, -1)
        for b in range(len(off) - 1):
            o0, o1 = int(off[b]), int(off[b + 1])
            if o0 == o1:
                continue
            x = torch.from_numpy(np.ascontiguousarray(pts[o0:o1, :3].T[None]))
            nb = torch.from_numpy(node[b:b + 1])
            want, _ = oracle_mod.som_topk(x, nb, k)
            got = torch.from_numpy(g[:, o0:o1].reshape(1, -1).astype(np.int32))
            assert torch.equal(got, b * M + want), (M, k, b)
            sa = ops.som_assign(x.to(DEV), nb.to(DEV), k, want_stats=False)["min_idx_i32"]
            assert torch.equal(got, b * M + sa.cpu()), (M, k, b)


@pytest.mark.parametrize("M", [1, 2, 3, 64, 121, 256])
def test_assign_non_finite_points(oracle_mod, M):
    """NaN points take nodes 0..k-1; +-inf points the +inf nodes by index; points whose distance
    overflows for all nodes but one or two get those first, then the others by index: k distinct
    nodes, in the same order from seg_points_assign, som_assign and the oracle."""
    p1, node = host.overflow_case(M)
    rs = np.random.RandomState(M)
    pts = np.concatenate([rs.uniform(-1, 1, (40, 6)).astype(np.float32), p1,
                          rs.uniform(-1, 1, (30, 6)).astype(np.float32)])
    off = np.array([0, 5, len(pts)], np.int64)            # two clouds, the same nodes
    nodes = np.stack([node, node])
    cm = rs.uniform(-1, 1, nodes.shape).astype(np.float32)
    d = [torch.from_numpy(a).to(DEV) for a in (pts, off, nodes, cm)]
    for k in range(1, min(4, M) + 1):
        want = host.assign_ref(pts, off, nodes, cm, k, 1, 0, len(pts), len(pts) + 3)
        got = _assign(*d, k, 1, 0, len(pts), len(pts) + 3)
        _check_assign(got, want, "M=%d k=%d" % (M, k))
        ids = np.ascontiguousarray(got[0].reshape(k, -1)[:, 40:40 + len(p1)]) - M   # cloud 1
        assert all(len(set(c)) == k for c in ids.T.tolist()), ids
        assert ids[:, 0].tolist() == list(range(k))                  # node 0, then +inf ones
        for n in (4, 5, 6):                                          # NaN points
            assert ids[:, n].tolist() == list(range(k))
        x = torch.from_numpy(np.ascontiguousarray(p1[:, :3].T[None]))
        sa = ops.som_assign(x.to(DEV), torch.from_numpy(node[None]).to(DEV), k)
        assert torch.equal(sa["min_idx_i32"].cpu().view(k, -1), torch.from_numpy(ids).int())
        assert int(sa["count"].sum()) == k * len(p1)
        want_o, _ = oracle_mod.som_topk(x, torch.from_numpy(node[None]), k)
        assert torch.equal(want_o.view(k, -1), torch.from_numpy(ids).int())


# ---- B. score_points against the sampled forward ---------------------------------------------------
TC_ENTRY = {"1": "sonet_pointwise_tc_forward", "fp16": "sonet_pointwise_tc_forward_f16"}
POINTWISE = ("sonet_pointwise_layer_f32", "sonet_pointwise_tc_forward",
             "sonet_pointwise_tc_forward_f16")


@contextlib.contextmanager
def _profiled():
    calls = []
    ops.PROFILE = calls
    try:
        yield calls
    finally:
        ops.PROFILE = None


def _head_routes(calls):
    """The entries of the head's layers 2-5: the last four point-wise layer calls (args[9] is
    Cout in both entries' signatures), after checking that they are those layers."""
    pw = [(c[0], c[3][9]) for c in calls if c[0] in POINTWISE]
    assert [co for _, co in pw[-4:]] == [512, 256, 128, 50], pw[-4:]
    return [n for n, _ in pw[-4:]]


def _model(monkeypatch, tc, M, k, act, sn, B, N, seed):
    monkeypatch.setenv("SONET_TC", tc)
    opt = synth.make_opt("segmenter", batch_size=B, input_pc_num=N, k=k, activation=act,
                         surface_normal=sn, node_num=M)
    st = build_states("segmenter", opt, seed)
    opt.device, opt.gpu_id = torch.device(DEV), 0
    m = segmenter.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.segmenter.load_state_dict(st["head"])
    return m, st


def _sampled_case(monkeypatch, tc, fused, M, k, act, sn, B, N, sizes, seed):
    """score_points over the sampled points == score_segmenter, and every head layer on the
    kernel the sampled forward used: wgmma for >= 256 columns (layers 2-3: B*k*N, layers 4-5:
    B*N) unless SONET_TC=0, the exact-fp32 kernel below."""
    m, _ = _model(monkeypatch, tc, M, k, act, sn, B, N, seed)
    m.encoder.fuse_pool = fused
    clouds = full._ragged(sizes, seed=seed)
    m.set_input(*full._batch_from(clouds, N, M, seed=seed))
    with _profiled() as calls:
        m.test_model()
        if fused:
            m.encoder._fpo_demand = False
            m.test_model()
    sampled = _head_routes(calls)
    pts, off = full._sampled_as_ragged(m)
    with _profiled() as calls:
        got = m.score_points(pts, off)
    routes = _head_routes(calls)
    want_routes = [TC_ENTRY[tc] if tc != "0" and rows >= 256 else "sonet_pointwise_layer_f32"
                   for rows in (B * k * N, B * k * N, B * N, B * N)]
    want = m.score_segmenter.permute(0, 2, 1).reshape(-1, m.opt.classes)
    assert sampled == want_routes, sampled
    assert routes == want_routes and torch.equal(got, want), \
        (routes, torch.equal(got, want), float((got - want).abs().max()))


# (B, N, k, M, cloud sizes): the benchmarked shape, then batches where B*N or B*k*N < 256
SHAPES = [
    (32, 1024, 3, 64, [2000 + 31 * i for i in range(32)]),
    (1, 128, 3, 64, [500]),           # layers 2-3 on wgmma, 4-5 on fp32
    (1, 64, 3, 64, [90]),             # every head layer on fp32
    (2, 100, 1, 64, [60, 300]),       # k = 1, 100 of the sampled points < 128: fp32 throughout
    (2, 100, 2, 121, [70, 40]),       # clouds with fewer points than N
    (3, 64, 2, 256, [50, 64, 200]),   # 384 columns at layers 2-3, 192 at 4-5
]


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tc", ["1", "0", "fp16"])
@pytest.mark.parametrize("shape", SHAPES, ids=["B%d_N%d_k%d_M%d" % s[:4] for s in SHAPES])
def test_sampled_points_small_and_benchmarked_shapes(monkeypatch, shape, tc, fused):
    B, N, k, M, sizes = shape
    i = SHAPES.index(shape)
    _sampled_case(monkeypatch, tc, fused, M, k, ("relu", "elu")[i % 2], i % 3 != 1, B, N, sizes,
                  seed=40 + i)


@pytest.mark.parametrize("sn", [True, False])
@pytest.mark.parametrize("act", ["relu", "elu"])
@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("M", [64, 121, 256])
def test_sampled_points_node_counts_and_options(monkeypatch, M, k, act, sn):
    # B*N = 120 < 256: layers 4-5 leave wgmma; B*k*N crosses 256 from k = 3
    _sampled_case(monkeypatch, "1", M % 2 == 1, M, k, act, sn, 1, 120, [150], seed=M + k)


def test_full_clouds_fp64_at_256_nodes(monkeypatch):
    """The float64 restatement of the reference's per-point path at M = 256 without normals,
    ragged clouds smaller and larger than N."""
    sizes = [1, 90, 700]
    m, st = _model(monkeypatch, "1", 256, 3, "relu", False, len(sizes), 256, 17)
    clouds = full._ragged(sizes, seed=17)
    m.set_input(*full._batch_from(clouds, 256, 256, seed=18))
    m.test_model()
    pts = torch.from_numpy(np.concatenate(clouds)).to(DEV)
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device=DEV)
    got = m.score_points(pts, off).double().cpu()
    enc = m.encoder
    dd = lambda t: t.detach().double().cpu()  # noqa: E731
    node, cm = m.input_node.cpu().numpy(), dd(enc.som_node)
    for b, c in enumerate(clouds):
        ref = full._oracle_cloud(st["encoder"], st["head"], m.opt, c, node[b], cm[b],
                                 dd(enc.first_pn_out_masked_max[b]), dd(enc.knn_feature_1[b]),
                                 dd(enc.final_pn_out[b]), dd(m.feature[b]), int(m.input_label[b]))
        g = got[int(off[b]):int(off[b + 1])]
        err = float(((g - ref).abs() / ref.abs().clamp(min=1)).max())
        assert err <= 1e-4, "cloud %d (%d points): rel err %.3e" % (b, len(c), err)


# ---- C. the ragged IoU -------------------------------------------------------------------------------
def _device_iou(score, seg, label, off, table):
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    iou, pred, corr = ops.seg_iou_ragged(d(score), d(seg), d(label), d(off), table, want_pred=True,
                                         want_correct=True)
    return iou.cpu().numpy(), pred.cpu().numpy(), corr.cpu().numpy()


@pytest.mark.parametrize("case", host.CASES, ids=[c[0] for c in host.CASES])
def test_iou_kernel_against_host_twin_and_restatement(lib_built, case):
    _, score, seg, label, off, table = case
    tab = ops.SHAPENET_PART_TABLE if table is None else table
    iou, pred, corr = _device_iou(score, seg, label, off, table)
    host.check_iou(iou, pred, corr, host.iou_ref(score, seg, label, off, tab),
                   max(len(p) for p in tab))
    rc, h_iou, h_pred, h_corr = host.host_iou(score, seg, label, off, tab)
    assert rc == 0, _C.last_error()
    assert h_iou.tobytes() == iou.tobytes()
    np.testing.assert_array_equal(h_pred, pred)
    np.testing.assert_array_equal(h_corr, corr)


def test_iou_kernel_300k_point_shape(lib_built):
    rs = np.random.RandomState(3)
    sizes = [5, 300_001, 0, 2]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    score = rs.normal(size=(int(off[-1]), 50)).astype(np.float32)
    label = np.array([1, 4, 0, 15], np.int64)
    seg = rs.randint(-1, 51, int(off[-1])).astype(np.int64)
    iou, pred, corr = _device_iou(score, seg, label, off, None)
    host.check_iou(iou, pred, corr, host.iou_ref(score, seg, label, off), 6)


@pytest.mark.parametrize("C, N", [(50, 1), (50, 256), (50, 257), (1, 100), (50, 1024)])
def test_ragged_equals_fixed_n(lib_built, C, N):
    """Every shape with N points: the same bits as the fixed-N kernel (ops.seg_iou)."""
    rs = np.random.RandomState(C + N)
    B = 5
    score = rs.normal(size=(B, N, C)).astype(np.float32)
    score[0, : N // 2] = np.nan
    table = None if C == 50 else ((0,),)
    label = rs.randint(0, 16 if C == 50 else 1, B).astype(np.int64)
    seg = rs.randint(0, C, (B, N)).astype(np.int64)
    off = np.arange(0, B * N + 1, N, dtype=np.int64)
    iou, pred, corr = _device_iou(score.reshape(-1, C), seg.reshape(-1), label, off, table)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    fi, fp, fc = ops.seg_iou(d(score.transpose(0, 2, 1)), d(seg), d(label), table, want_pred=True,
                             want_correct=True)
    assert fi.cpu().numpy().tobytes() == iou.tobytes()
    np.testing.assert_array_equal(fp.cpu().numpy().reshape(-1), pred)
    np.testing.assert_array_equal(fc.cpu().numpy(), corr)


def _raw_device_iou(score, seg, label, off, poff, ids, K, C=None):
    """sonet_seg_iou_ragged_f32 with raw offsets and part table, as a caller that skips
    ops.seg_iou_ragged's checks passes them: outputs pre-filled with sentinels."""
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    score_d, seg_d, lab_d, off_d = d(score), d(seg), d(label), d(off)
    poff_d, ids_d = d(np.asarray(poff, np.int32)), d(np.asarray(ids, np.int32))
    B, T = len(label), score.shape[0]
    iou = torch.full((B,), -7.0, dtype=torch.float64, device=DEV)
    pred = torch.full((T,), -7, dtype=torch.int64, device=DEV)
    corr = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    rc = _C.lib().sonet_seg_iou_ragged_f32(
        _C.ptr(score_d), _C.ptr(seg_d), _C.ptr(lab_d), _C.ptr(off_d), B,
        score.shape[1] if C is None else C, T, _C.ptr(poff_d), _C.ptr(ids_d), K, _C.ptr(iou),
        _C.ptr(pred), _C.ptr(corr), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _C.last_error()
    torch.cuda.synchronize()
    return iou.cpu().numpy(), pred.cpu().numpy(), corr.cpu().numpy()


def test_iou_kernel_marks_bad_shapes_nan(lib_built):
    """A label outside the table, a category of 257 parts (or none) and offsets out of order or
    out of range: that shape's IoU is NaN; the other shapes keep their values, and pred and
    correct are written for every shape whose rows are in range."""
    rs = np.random.RandomState(9)
    sizes = [40, 30, 50, 20, 60]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    T = int(off[-1])
    C = 300
    score = rs.normal(size=(T, C)).astype(np.float32)
    seg = rs.randint(0, C, T).astype(np.int64)
    table = ((0, 1, 2), tuple(range(257)), (), (5, 6))
    poff = np.concatenate([[0], np.cumsum([len(p) for p in table])])
    ids = [p for parts in table for p in parts]
    label = np.array([0, 1, 2, 3, 4], np.int64)        # ok, 257 parts, none, ok, outside
    iou, pred, corr = _raw_device_iou(score, seg, label, off, poff, ids, len(table))
    ref_tab = (table[0], (0,), (0,), table[3], (0,))
    want, _, want_pred, want_corr = host.iou_ref(score, seg, label, off, ref_tab)
    assert np.isnan(iou[[1, 2, 4]]).all()
    np.testing.assert_array_equal(iou[[0, 3]], want[[0, 3]])
    np.testing.assert_array_equal(pred, want_pred)
    np.testing.assert_array_equal(corr, want_corr)
    lab2 = np.array([0, -1, 3, 0, 3], np.int64)
    iou, _, corr = _raw_device_iou(score, seg, lab2, off, poff, ids, len(table))
    assert np.isnan(iou[1]) and not np.isnan(iou[[0, 2, 3, 4]]).any()
    np.testing.assert_array_equal(corr, want_corr)

    # bad offsets: shape 1 decreasing, shape 3 past T, shape 4 starting past T
    label = np.array([0, 3, 0, 3, 0], np.int64)
    good, _, g_pred, g_corr = host.iou_ref(score, seg, label, off, table)
    bad = off.copy()
    bad[2] = 30                                         # shape 1: [40, 30)
    bad[4] = T + 5                                      # shape 3: [120, T+5); shape 4: [T+5, T)
    iou, pred, corr = _raw_device_iou(score, seg, label, bad, poff, ids, len(table))
    assert np.isnan(iou[[1, 3, 4]]).all()
    np.testing.assert_array_equal(iou[0], good[0])
    # shape 2 reads rows bad[2] .. bad[3] = [30, 120)
    sub = host.iou_ref(score[30:120], seg[30:120], label[2:3], np.array([0, 90]), table)
    assert iou[2] == sub[0][0]
    assert corr[2] == sub[3][0] and corr[0] == g_corr[0]
    assert corr[1] == 0 and corr[3] == 0 and corr[4] == 0     # written, no rows counted
    np.testing.assert_array_equal(pred[:120], np.concatenate([g_pred[:30], sub[2]]))
