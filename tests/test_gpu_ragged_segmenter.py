"""Whole shapes of any size through the part segmenter on the GPU (segmenter.Model.segment_clouds,
losses.seg_loss_ragged): test_model()'s bits at equal sizes, each shape against its own dense forward
at mixed sizes, permutation and chunk invariance, the reference goldens as ragged sets, untouched
model and graph state, the dataset path end to end, and the ragged loss kernel against the dense
one and an fp64 restatement."""
import numpy as np
import pytest
import torch

from helpers import assert_close, assert_golden, build_states, golden, golden_case
from sonet_b200 import augmentation, losses, ops, segmenter, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C50 = 50


def _model(monkeypatch, tc="1", B=2, N=256, seed=3, fuse_pool=True, **over):
    monkeypatch.setenv("SONET_TC", tc)
    opt = synth.make_opt("segmenter", batch_size=B, input_pc_num=N, **over)
    st = build_states("segmenter", opt, seed)
    opt.device, opt.gpu_id = torch.device(DEV), 0
    m = segmenter.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.segmenter.load_state_dict(st["head"])
    m.encoder.fuse_pool = fuse_pool      # True: the first test_model() takes the group route
    m.encoder.eval()
    m.segmenter.eval()
    return m


def _as_ragged(pc, sn):
    B, _, N = pc.shape
    pts = torch.cat((pc, sn), dim=1).permute(0, 2, 1).reshape(-1, 6).contiguous().to(DEV)
    return pts, torch.arange(0, B * N + 1, N, dtype=torch.int64, device=DEV)


def _targets(rs, shape, ignore=0.05, C=C50):
    t = rs.randint(0, C, size=shape).astype(np.int64)
    t[rs.uniform(size=shape) < ignore] = -100
    return torch.from_numpy(t)


def _clouds(sizes, M, som_k, seed):
    """Ragged clouds U(-1,1)^3 with unit normals, nodes drawn from each cloud (+ jitter)."""
    rs = np.random.RandomState(seed)
    pts, nodes = [], []
    for P in sizes:
        xyz = rs.uniform(-1, 1, size=(P, 3)).astype(np.float32)
        n = rs.normal(size=(P, 3))
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        pts.append(np.concatenate([xyz, n.astype(np.float32)], axis=1))
        sel = rs.choice(P, M, replace=P < M)
        nodes.append(xyz[sel].T + rs.normal(0, 1e-2, size=(3, M)).astype(np.float32))
    node = torch.from_numpy(np.ascontiguousarray(np.stack(nodes), dtype=np.float32)).to(DEV)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)).to(DEV)
    label = torch.from_numpy(rs.randint(0, 16, size=len(sizes)).astype(np.int64)).to(DEV)
    seg = _targets(rs, (int(sum(sizes)),)).to(DEV)
    return torch.from_numpy(np.concatenate(pts)).to(DEV), off, node, \
        augmentation.som_knn(node, som_k, M), label, seg


def _dense(m, inp, seg):
    m.set_input(inp["pc"], inp["sn"], inp["label"], seg, inp["node"], inp["node_knn_I"])
    m.test_model()


def _point_major(score):
    return score.permute(0, 2, 1).reshape(-1, score.shape[1])


# ---- 1. equal sizes: test_model()'s bits --------------------------------------------------------
EQUAL = [  # tc, activation, k, M, surface_normal, N
    ("1", "relu", 3, 64, True, 256),
    ("1", "relu", 1, 9, True, 255),
    ("1", "elu", 2, 121, True, 257),
    ("1", "relu", 3, 256, False, 1024),
    ("1", "elu", 1, 64, False, 1024),
    ("1", "relu", 2, 9, False, 256),
    ("fp16", "relu", 3, 64, True, 256),
    ("fp16", "elu", 2, 256, False, 255),
    ("fp16", "relu", 1, 121, True, 257),
    ("fp16", "elu", 3, 9, True, 1024),
]


@pytest.mark.parametrize("tc,act,k,M,sn,N", EQUAL)
def test_equal_sizes_give_test_model_bits(monkeypatch, tc, act, k, M, sn, N):
    B = 2
    m = _model(monkeypatch, tc, B=B, N=N, k=k, node_num=M, activation=act, surface_normal=sn)
    assert ops.som_group_fits(N, M, k, torch.device(DEV))       # the dense group route
    inp = synth.synth_inputs(B, N, M, 9, seed=k + M + N)
    seg = _targets(np.random.RandomState(N), (B, N))
    _dense(m, inp, seg)
    pts, off = _as_ragged(inp["pc"], inp["sn"])
    r = m.segment_clouds(pts, off, inp["label"].to(DEV), inp["node"].to(DEV),
                         inp["node_knn_I"].to(DEV), seg=seg.reshape(-1).to(DEV))
    assert torch.equal(r["feature"], m.feature)
    assert torch.equal(r["score"], _point_major(m.score_segmenter))
    assert torch.equal(r["loss"], m.loss_segmenter)
    for b in range(B):                       # each shape's own mean, against fp64
        sc = m.score_segmenter[b].t().double()
        t = seg[b].to(DEV)
        keep = t != -100
        want = -torch.log_softmax(sc, dim=1)[keep].gather(1, t[keep].view(-1, 1)).mean()
        assert abs(float(r["loss_array"][b]) - float(want)) <= 1e-6 * abs(float(want))


# ---- 2. equal sizes against the default segmenter ------------------------------------------------
@pytest.mark.parametrize("tc", ["1", "0"])
def test_equal_sizes_against_the_default_segmenter(monkeypatch, tc):
    """fuse_pool False: test_model() sums the cluster means in som_stats_kernel's order. The
    assignment and the counts stay bit-equal; scores and loss are within the 1e-4 bar."""
    B, N, M, k = 3, 512, 64, 3
    m = _model(monkeypatch, tc, B=B, N=N, k=k, node_num=M, fuse_pool=False)
    inp = synth.synth_inputs(B, N, M, 9, seed=7)
    seg = _targets(np.random.RandomState(7), (B, N))
    _dense(m, inp, seg)
    enc = m.encoder
    pts, off = _as_ragged(inp["pc"], inp["sn"])
    node = inp["node"].to(DEV)
    idx, count, _ = ops.som_assign_ragged(pts, off, node, k)
    assert torch.equal(idx, enc.min_idx.reshape(-1))
    assert torch.equal(count, enc._assign["count"])
    r = m.segment_clouds(pts, off, inp["label"].to(DEV), node, inp["node_knn_I"].to(DEV),
                         seg=seg.reshape(-1).to(DEV))
    assert_close(r["feature"], m.feature, "feature")
    assert_close(r["score"], _point_major(m.score_segmenter), "score")
    assert_close(r["loss"], m.loss_segmenter, "loss")


# ---- 3. mixed sizes: each shape against its own dense forward ------------------------------------
def test_mixed_sizes_match_each_shape_alone(monkeypatch):
    k, M = 3, 64
    sizes = [1, k - 1, 63, 256, 2718, 10000]
    pts, off, node, knn, label, seg = _clouds(sizes, M, 9, seed=11)
    m = _model(monkeypatch, B=1, N=256, k=k, node_num=M)
    r = m.segment_clouds(pts, off, label, node, knn, seg=seg)
    o = off.tolist()
    for b, P in enumerate(sizes):
        c = pts[o[b]:o[b + 1]]
        m1 = _model(monkeypatch, B=1, N=P, k=k, node_num=M)
        inp = dict(pc=c[:, :3].t().contiguous()[None].cpu(),
                   sn=c[:, 3:].t().contiguous()[None].cpu(), label=label[b:b + 1].cpu(),
                   node=node[b:b + 1].cpu(), node_knn_I=knn[b:b + 1].cpu())
        _dense(m1, inp, seg[o[b]:o[b + 1]].view(1, -1).cpu())
        assert_close(r["feature"][b], m1.feature[0], "feature %d" % b)
        assert_close(r["score"][o[b]:o[b + 1]], m1.score_segmenter[0].t(), "score %d" % b)
        assert_close(r["loss_array"][b], m1.loss_segmenter, "loss %d" % b)
        del m1


# ---- 4. invariance -------------------------------------------------------------------------------
def test_permutation_and_chunks_change_no_bit(monkeypatch):
    k, M = 2, 64
    sizes = [300, 1200, 77, 5000, 640]
    pts, off, node, knn, label, seg = _clouds(sizes, M, 9, seed=2)
    m = _model(monkeypatch, B=1, N=256, k=k, node_num=M)
    ref = m.segment_clouds(pts, off, label, node, knn, seg=seg)
    for chunk in (50, 1000, 10 ** 6):      # below the smallest shape, mid-shape, everything
        c = m.segment_clouds(pts, off, label, node, knn, seg=seg, chunk_points=chunk)
        for key, v in ref.items():
            assert torch.equal(c[key], v), (chunk, key)
    perm = [3, 0, 4, 2, 1]
    o = off.tolist()
    rows = lambda t: torch.cat([t[o[b]:o[b + 1]] for b in perm])  # noqa: E731
    p_off = torch.tensor(np.concatenate([[0], np.cumsum([sizes[b] for b in perm])]),
                         dtype=torch.int64, device=DEV)
    p = m.segment_clouds(rows(pts), p_off, label[perm], node[perm], knn[perm], seg=rows(seg))
    assert torch.equal(p["score"], rows(ref["score"]))
    assert torch.equal(p["feature"], ref["feature"][perm])
    assert torch.equal(p["loss_array"], ref["loss_array"][perm])
    assert abs(float(p["loss"]) - float(ref["loss"])) <= 1e-6 * abs(float(ref["loss"]))


# ---- 5. the reference goldens as ragged sets ------------------------------------------------------
@pytest.mark.parametrize("name", ["segmenter_b2_n128", "segmenter_b2_n200_m100_k2",
                                  "elu_segmenter_b2_n128"])
def test_golden_clouds_as_ragged_set(name):
    g = golden(name)
    opt, inp, seed = golden_case(g, "segmenter")
    st = build_states("segmenter", opt, seed)
    opt.device, opt.gpu_id = torch.device(DEV), 0
    m = segmenter.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.segmenter.load_state_dict(st["head"])
    m.encoder.eval()
    m.segmenter.eval()
    B, N = int(g["B"]), int(g["N"])
    seg = _targets(np.random.RandomState(seed), (B * N,))
    pts, off = _as_ragged(inp["pc"], inp["sn"])
    r = m.segment_clouds(pts, off, inp["label"].to(DEV), inp["node"].to(DEV),
                         inp["node_knn_I"].to(DEV), seg=seg.to(DEV))
    dense = r["score"].view(B, N, -1).permute(0, 2, 1)
    # test_gpu_elu.py's HEAD_TOL: the ELU fixture's dense score_segmenter measures 1.01e-4 on the
    # wgmma routes, and so do these scores (H100 80GB HBM3)
    assert_golden(g, "score_segmenter", dense, tol=2e-4 if name.startswith("elu") else 1e-4)
    # the loss of the reference's own scores (complete in the fixture), in fp64
    assert int(g["score_segmenter__stride"]) == 1
    ref = torch.from_numpy(g["score_segmenter"]).double().view(B, -1, N)
    want = torch.nn.functional.cross_entropy(ref, seg.view(B, N), ignore_index=-100)
    assert_close(r["loss"].cpu(), want.float(), "loss")


# ---- 6. model and graph state untouched -----------------------------------------------------------
@pytest.mark.parametrize("tc", ["1", "0"])
def test_model_and_graph_state_untouched(monkeypatch, tc):
    B, N, M = 3, 512, 64
    m = _model(monkeypatch, tc, B=B, N=N, fuse_pool=False)
    m.enable_cuda_graph(True)
    inp = synth.synth_inputs(B, N, M, 9, seed=21)
    seg = _targets(np.random.RandomState(21), (B, N))
    _dense(m, inp, seg)
    pts_s, off_s = _as_ragged(inp["pc"], inp["sn"])
    want_points = m.score_points(pts_s, off_s)
    enc = m.encoder
    inputs = ("input_pc", "input_sn", "input_label", "input_seg", "input_node", "input_node_knn_I")
    names = ("feature", "score_segmenter", "loss_segmenter", "loss")
    enc_names = ("som_node", "feature", "first_pn_out_masked_max", "knn_center_1", "knn_feature_1",
                 "final_pn_out", "min_idx")

    def snap():
        return ({n: getattr(m, n) for n in inputs + names}, {n: getattr(enc, n) for n in enc_names})
    ref = snap()
    vals = [{n: t.clone() for n, t in d.items()} for d in ref]
    pts, off, node, knn, label, sg = _clouds([900, 3000, 12, 40], M, 9, seed=5)
    r = m.segment_clouds(pts, off, label, node, seg=sg)          # node_knn_I computed
    assert r["score"].shape == (pts.shape[0], m.opt.classes)
    assert m._evaluated
    after = snap()
    for d0, d1, v in zip(ref, after, vals):
        for n in d0:
            assert d1[n] is d0[n], "attribute %s rebound" % n
            assert torch.equal(d1[n], v[n]), "attribute %s changed" % n
    assert torch.equal(m.score_points(pts_s, off_s), want_points)
    m.test_model()                                                # graph replay
    for d1, v in zip(snap(), vals):
        for n in d1:
            assert torch.equal(d1[n], v[n]), "replay: %s" % n


# ---- 7. end to end from the device dataset --------------------------------------------------------
def test_dataset_to_iou(monkeypatch):
    m = _model(monkeypatch, B=2, N=256, fuse_pool=False)
    rs = np.random.RandomState(1)
    sizes = (400, 2900, 1300)
    clouds = [rs.uniform(-1, 1, size=(P, 6)).astype(np.float32) for P in sizes]
    labels = [1, 4, 15]
    segs = [rs.choice(ops.SHAPENET_PART_TABLE[l], size=P) for l, P in zip(labels, sizes)]
    nodes = [c[rs.choice(len(c), 64, replace=False), :3] for c in clouds]
    ds = augmentation.DeviceDataset(clouds, labels, nodes, seg=segs, device=DEV)
    pts, off, label, node, knn = ds.full_batch([2, 0, 1], m.opt)
    _, _, seg = ds.full_clouds([2, 0, 1])
    r = m.segment_clouds(pts, off, label, node, knn, seg=seg)
    assert r["score"].shape == (sum(sizes), m.opt.classes) and torch.isfinite(r["score"]).all()
    assert r["feature"].shape == (3, m.opt.feature_num) and torch.isfinite(r["feature"]).all()
    assert torch.isfinite(r["loss"]) and torch.isfinite(r["loss_array"]).all()
    assert r["loss_array"].shape == (3,)
    iou = losses.compute_iou_full(r["score"], seg, label, off)
    assert iou.shape == (3,) and np.isfinite(iou).all() and ((iou >= 0) & (iou <= 1)).all()
    n = m.segment_clouds(pts, off, label, node, knn)
    assert n["loss"] is None and n["loss_array"] is None
    assert torch.equal(n["score"], r["score"])


# ---- 8. the ragged segmentation loss -------------------------------------------------------------
def _fp64_loss(score, target, sizes):
    """(batch mean, per-shape means) of -log_softmax(score)[target] in fp64, -100 not counted."""
    s = score.astype(np.float64)
    mx = s.max(axis=1, keepdims=True)
    lsm = s - mx - np.log(np.exp(s - mx).sum(axis=1, keepdims=True))
    keep = target != -100
    nll = np.zeros(len(target))
    nll[keep] = -lsm[np.flatnonzero(keep), target[keep]]
    off = np.concatenate([[0], np.cumsum(sizes)])
    per = np.array([nll[off[b]:off[b + 1]][keep[off[b]:off[b + 1]]].mean()
                    if keep[off[b]:off[b + 1]].any() else np.nan for b in range(len(sizes))])
    return nll[keep].sum() / keep.sum(), per


def _ragged_case(sizes, C, seed, scale=4.0):
    rs = np.random.RandomState(seed)
    T = int(sum(sizes))
    score = (rs.standard_normal((T, C)) * scale).astype(np.float32)
    return score, _targets(rs, (T,), C=C).numpy()


def _run(score, target, sizes):
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device=DEV)
    return ops.seg_loss_ragged(torch.from_numpy(score).to(DEV), torch.from_numpy(target).to(DEV),
                               off)


@pytest.mark.parametrize("B,P,C", [(1, 1, 50), (3, 255, 50), (3, 256, 50), (3, 257, 50),
                                   (32, 1024, 50), (5, 700, 1), (2, 300, 7)])
def test_seg_loss_equal_sizes_give_dense_bits(B, P, C):
    score, target = _ragged_case([P] * B, C, seed=B * P + C)
    loss, arr = _run(score, target, [P] * B)
    dense = torch.from_numpy(score).view(B, P, C).permute(0, 2, 1).contiguous().to(DEV)
    assert torch.equal(loss, ops.seg_loss(dense, torch.from_numpy(target).view(B, P).to(DEV)))
    _, per = _fp64_loss(score, target, [P] * B)
    np.testing.assert_allclose(arr.cpu().numpy(), per, rtol=1e-6)


def test_seg_loss_mixed_sizes_against_fp64():
    sizes = [1, 255, 256, 257, 3000, 1 << 20, 77]
    score, target = _ragged_case(sizes, C50, seed=3)
    loss, arr = _run(score, target, sizes)
    want, per = _fp64_loss(score, target, sizes)
    assert abs(float(loss) - want) <= 1e-6 * abs(want)
    np.testing.assert_allclose(arr.cpu().numpy(), per, rtol=1e-6)
    # the shapes' own means weigh every shape once
    assert abs(float(arr.double().mean()) - per.mean()) <= 1e-6 * abs(per.mean())


def test_seg_loss_edge_cases():
    sizes = [300, 257, 1, 1000]
    score, target = _ragged_case(sizes, C50, seed=5)
    off = np.concatenate([[0], np.cumsum(sizes)])
    base_loss, base = _run(score, target, sizes)
    _, per = _fp64_loss(score, target, sizes)

    # an all-ignored shape: NaN there only; the batch is the mean over the other shapes' points
    t = target.copy()
    t[off[1]:off[2]] = -100
    loss, arr = _run(score, t, sizes)
    want, _ = _fp64_loss(score, t, sizes)
    a = arr.cpu().numpy()
    assert np.isnan(a[1]) and np.isfinite(a[[0, 2, 3]]).all()
    assert np.array_equal(a[[0, 2, 3]], base.cpu().numpy()[[0, 2, 3]])
    assert abs(float(loss) - want) <= 1e-6 * abs(want)

    # an out-of-range target (other than -100): NaN in its shape and the batch only
    for bad in (C50, -1, 1 << 40):
        t = target.copy()
        t[off[3] + 5] = bad
        loss, arr = _run(score, t, sizes)
        a = arr.cpu().numpy()
        assert torch.isnan(loss) and np.isnan(a[3]), bad
        assert np.array_equal(a[:3], base.cpu().numpy()[:3]), bad

    # a NaN score: the dense rule per point (its loss is NaN), so its shape and the batch are NaN
    s = score.copy()
    s[off[0] + 7, 3] = np.nan
    t = target.copy()
    t[off[0] + 7] = 3
    loss, arr = _run(s, t, sizes)
    a = arr.cpu().numpy()
    assert torch.isnan(loss) and np.isnan(a[0]) and np.array_equal(a[1:], base.cpu().numpy()[1:])
    d = torch.from_numpy(s[off[0]:off[1]].T.copy())[None].to(DEV)
    assert torch.isnan(ops.seg_loss(d, torch.from_numpy(t[off[0]:off[1]])[None].to(DEV)))

    # ignored targets count nowhere: the batch and every shape against fp64
    np.testing.assert_allclose(base.cpu().numpy(), per, rtol=1e-6)
    assert (target == -100).any()

    # the losses wrapper returns the same and refuses a gradient
    sc = torch.from_numpy(score).to(DEV)
    offs = torch.from_numpy(off).to(DEV)
    l2, a2 = losses.seg_loss_ragged(sc, torch.from_numpy(target).to(DEV), offs)
    assert torch.equal(l2, base_loss) and torch.equal(a2, base)
    with pytest.raises(RuntimeError, match="evaluation only"):
        losses.seg_loss_ragged(sc.requires_grad_(True), torch.from_numpy(target).to(DEV), offs)


def test_seg_loss_empty_shapes():
    """Empty shapes (equal offsets) have no counted point: NaN in loss_array, nothing in loss."""
    sizes = [0, 40, 0, 300, 0]
    score, target = _ragged_case(sizes, C50, seed=8)
    loss, arr = _run(score, target, sizes)
    want, per = _fp64_loss(score, target, sizes)
    a = arr.cpu().numpy()
    assert np.isnan(a[[0, 2, 4]]).all()
    np.testing.assert_allclose(a[[1, 3]], per[[1, 3]], rtol=1e-6)
    assert abs(float(loss) - want) <= 1e-6 * abs(want)
