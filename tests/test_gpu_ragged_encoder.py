"""Whole clouds of any size on the GPU (networks.Encoder.forward_ragged, classifier.Model.score_clouds):
the dense forward's bits at equal sizes, each cloud against its own dense forward at mixed sizes,
permutation and chunk invariance, the fused ragged pool against the ragged index_max at its edges,
the reference golden, the numpy restatement of the statistics, and untouched model state."""
import numpy as np
import pytest
import torch

import ragged_emu
from helpers import assert_close, assert_golden, build_states, golden, golden_case
from sonet_b200 import augmentation, classifier, ops, segmenter, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cls(monkeypatch, tc="1", B=2, N=256, seed=3, **over):
    monkeypatch.setenv("SONET_TC", tc)
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, **over)
    st = build_states("classifier", opt, seed)
    opt.device, opt.gpu_id = torch.device(DEV), 0
    m = classifier.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.classifier.load_state_dict(st["head"])
    m.encoder.eval()
    m.classifier.eval()
    return m


def _as_ragged(pc, sn):
    B, _, N = pc.shape
    pts = torch.cat((pc, sn), dim=1).permute(0, 2, 1).reshape(-1, 6).contiguous().to(DEV)
    return pts, torch.arange(0, B * N + 1, N, dtype=torch.int64, device=DEV)


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
    return torch.from_numpy(np.concatenate(pts)).to(DEV), off, node, \
        augmentation.som_knn(node, som_k, M)


# ---- 1. equal sizes give the dense forward's bits -----------------------------------------------
EQUAL = [  # tc, activation, k, M, som_k, som_k_type, surface_normal, N
    ("1", "relu", 3, 64, 9, "avg", True, 256),
    ("1", "relu", 1, 9, 9, "avg", True, 255),
    ("1", "elu", 2, 121, 9, "center", True, 257),
    ("1", "relu", 4, 256, 9, "avg", True, 5000),
    ("1", "relu", 3, 64, 0, "avg", True, 256),
    ("1", "elu", 2, 256, 0, "avg", False, 255),
    ("1", "relu", 3, 64, 9, "center", False, 5000),
    ("fp16", "relu", 3, 64, 9, "avg", True, 256),
    ("fp16", "elu", 4, 121, 9, "center", False, 257),
    ("fp16", "relu", 1, 256, 0, "avg", True, 5000),
]


@pytest.mark.parametrize("tc,act,k,M,som_k,som_k_type,sn,N", EQUAL)
def test_equal_sizes_give_dense_bits(monkeypatch, tc, act, k, M, som_k, som_k_type, sn, N):
    B = 2
    m = _cls(monkeypatch, tc, B=B, N=N, k=k, node_num=M, som_k=som_k, som_k_type=som_k_type,
             activation=act, surface_normal=sn)
    assert ops.som_group_fits(N, M, k, torch.device(DEV))       # the dense group route
    inp = synth.synth_inputs(B, N, M, max(som_k, 1), seed=k + M)
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    m.test_model()
    enc = m.encoder
    pts, off = _as_ragged(inp["pc"], inp["sn"])
    node, knn = inp["node"].to(DEV), inp["node_knn_I"].to(DEV)
    feat, nodes = enc.forward_ragged(pts, off, node, knn, return_nodes=True)
    score = m.score_clouds(pts, off, node, knn)
    assert torch.equal(nodes["som_node"], enc.som_node)
    assert torch.equal(nodes["first_pn_out_masked_max"], enc.first_pn_out_masked_max)
    assert torch.equal(nodes["final_pn_out"], enc.final_pn_out)
    assert torch.equal(feat, enc.feature)
    assert torch.equal(score, m.score)
    idx, count, row_max = ops.som_assign_ragged(pts, off, node, k)
    assert torch.equal(idx, enc.min_idx.reshape(-1))
    assert torch.equal(count, enc._assign["count"])


@pytest.mark.parametrize("act,k,M,som_k,sn,N", [("relu", 3, 64, 9, True, 256),
                                                ("elu", 1, 121, 0, False, 257)])
def test_fp32_route_within_bar(monkeypatch, act, k, M, som_k, sn, N):
    """SONET_TC=0: the dense forward sums cluster means in som_stats_kernel's order; assignment and
    counts stay bit-equal, the rest within the 1e-4 bar; the ragged index_max serves the pool."""
    B = 2
    m = _cls(monkeypatch, "0", B=B, N=N, k=k, node_num=M, som_k=som_k, activation=act,
             surface_normal=sn)
    inp = synth.synth_inputs(B, N, M, max(som_k, 1), seed=5)
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    m.test_model()
    enc = m.encoder
    pts, off = _as_ragged(inp["pc"], inp["sn"])
    node, knn = inp["node"].to(DEV), inp["node_knn_I"].to(DEV)
    idx, count, row_max = ops.som_assign_ragged(pts, off, node, k)
    assert torch.equal(idx, enc.min_idx.reshape(-1))
    assert torch.equal(count, enc._assign["count"])
    assert torch.equal(row_max, enc._assign["row_max"])
    feat, nodes = enc.forward_ragged(pts, off, node, knn, return_nodes=True)
    assert_close(nodes["som_node"], enc.som_node, "cluster_mean")
    assert_close(feat, enc.feature, "feature")
    assert_close(m.score_clouds(pts, off, node, knn), m.score, "score")


# ---- 2. mixed sizes: each cloud against its own dense B=1 forward ---------------------------------
@pytest.mark.parametrize("tc", ["1", "fp16"])
def test_mixed_sizes_match_each_cloud_alone(monkeypatch, tc):
    k, M, som_k = 3, 64, 9
    sizes = [1, k - 1, 63, 256, 2718, 10000]
    m = _cls(monkeypatch, tc, B=1, N=256, k=k, node_num=M, som_k=som_k)
    enc = m.encoder
    pts, off, node, knn = _clouds(sizes, M, som_k, seed=11)
    feat, nodes = enc.forward_ragged(pts, off, node, knn, return_nodes=True)
    score = m.score_clouds(pts, off, node, knn)
    idx, count, _ = ops.som_assign_ragged(pts, off, node, k)
    o = off.tolist()
    for b, P in enumerate(sizes):
        c = pts[o[b]:o[b + 1]]
        x = c[:, :3].t().contiguous().unsqueeze(0)
        s = c[:, 3:].t().contiguous().unsqueeze(0)
        with torch.no_grad():
            f1 = enc(x, s, node[b:b + 1], knn[b:b + 1])
            s1 = m.classifier(f1)
        assert torch.equal(idx[k * o[b]:k * o[b + 1]], enc.min_idx.reshape(-1)), b
        assert torch.equal(count[b], enc._assign["count"][0]), b
        if ops.som_group_fits(P, M, k, torch.device(DEV)):
            assert torch.equal(nodes["som_node"][b], enc.som_node[0]), b
        else:
            assert_close(nodes["som_node"][b], enc.som_node[0], "cluster_mean %d" % b)
        assert torch.equal(nodes["first_pn_out_masked_max"][b], enc.first_pn_out_masked_max[0]), b
        # the node-level routes differ with B*M; one fp16 product per MAC carries ~2^-10 per term
        tol = 4e-3 if tc == "fp16" else 1e-4
        assert_close(feat[b], f1[0], "feature %d" % b, tol)
        assert_close(score[b], s1[0], "score %d" % b, tol)


def test_statistics_match_the_numpy_restatement(monkeypatch):
    k, M = 3, 64
    sizes = [1, 2, 63, 700, 20000]
    pts, off, node, _ = _clouds(sizes, M, 9, seed=4)
    idx, count, row_max = ops.som_assign_ragged(pts, off, node, k)
    xs, ns, p0, cm = ops.som_group_decenter_ragged(pts, off, idx, M, k, True)
    h_pts, h_off, h_node = pts.cpu().numpy(), off.cpu().numpy(), node.cpu().numpy()
    e_idx, e_count = ragged_emu.assign(h_pts, h_off, h_node, k)
    order, e_ns, e_p0, e_cm = ragged_emu.group(h_pts, h_off, e_idx, M, k)
    assert np.array_equal(idx.cpu().numpy(), e_idx)
    assert np.array_equal(count.cpu().numpy(), e_count)
    assert np.array_equal(row_max.cpu().numpy(), (e_count > 0).astype(np.int32))
    assert np.array_equal(ns.cpu().numpy(), e_ns)
    assert np.array_equal(p0.cpu().numpy(), e_p0)
    assert np.array_equal(cm.cpu().numpy().view(np.int32), e_cm.view(np.int32))
    # x_sorted: the decentred copies in that order
    T = h_pts.shape[0]
    cloud = np.repeat(np.arange(len(sizes)), k * np.array(sizes))
    pt_of = np.concatenate([h_off[b] + np.tile(np.arange(P), k) for b, P in enumerate(sizes)])
    src = pt_of[order]
    want = h_pts[src, :3].T - e_cm[cloud[order], :, e_ns % M].T
    assert np.array_equal(xs[:3].cpu().numpy(), want.astype(np.float32))
    assert np.array_equal(xs[3:].cpu().numpy(), h_pts[src, 3:].T)
    assert xs.shape == (6, k * T)


# ---- 3. invariance ---------------------------------------------------------------------------------
@pytest.mark.parametrize("tc", ["1", "0"])
def test_permutation_and_chunks_change_no_bit(monkeypatch, tc):
    k, M, som_k = 2, 64, 9
    sizes = [300, 1, 5000, 77, 1200]
    m = _cls(monkeypatch, tc, B=1, N=256, k=k, node_num=M, som_k=som_k)
    enc = m.encoder
    pts, off, node, knn = _clouds(sizes, M, som_k, seed=2)
    ref, rn = enc.forward_ragged(pts, off, node, knn, return_nodes=True)
    for chunk in (1, 1500, 10 ** 6):
        f, n = enc.forward_ragged(pts, off, node, knn, chunk_points=chunk, return_nodes=True)
        assert torch.equal(f, ref), chunk
        for key in ("som_node", "first_pn_out_masked_max", "final_pn_out"):
            assert torch.equal(n[key], rn[key]), (chunk, key)
    perm = [3, 0, 4, 2, 1]
    o = off.tolist()
    p_pts = torch.cat([pts[o[b]:o[b + 1]] for b in perm])
    p_off = torch.tensor(np.concatenate([[0], np.cumsum([sizes[b] for b in perm])]),
                         dtype=torch.int64, device=DEV)
    f = enc.forward_ragged(p_pts, p_off, node[perm], knn[perm])
    assert torch.equal(f, ref[perm])


# ---- 4. pool edges: fused ragged pool against the ragged index_max ---------------------------------
@pytest.mark.parametrize("tc", ["1", "fp16"])
@pytest.mark.parametrize("edge", ["one_node", "sentinel", "nonfinite"])
def test_fused_pool_matches_ragged_index_max(monkeypatch, tc, edge):
    k, M = 3, 64
    m = _cls(monkeypatch, tc, B=1, N=256, k=1 if edge == "one_node" else k, node_num=M)
    k = m.opt.k
    fpn = m.encoder.first_pointnet
    sizes = [500, 37, 2000]
    pts, off, node, _ = _clouds(sizes, M, 9, seed=9)
    if edge == "one_node":       # cloud 0 sits on one node: the other nodes take copy 0's feature
        pts[:500, :3] = node[0, :, 5]
    if edge == "nonfinite":
        pts[3, 0] = float("nan")
        pts[600, 1] = float("inf")
        pts[601, 2] = -float("inf")
    blob, fpar = fpn._tc_params()
    if edge == "sentinel":       # a layer-3 shift that pushes half the channels below -1000
        fpar = fpar.clone()
        s3 = 64 * 6 + 64 + 128 + 256
        fpar[s3:s3 + 384:2] = -1.0e5
    idx, _, _ = ops.som_assign_ragged(pts, off, node, k)
    xs, ns, p0s, cm = ops.som_group_decenter_ragged(pts, off, idx, M, k, True)
    keys, p0 = ops.pointresnet_tc_pool_ragged(xs, blob, fpar, ns, p0s, M, f16=tc == "fp16")
    fused = ops.pool_finalize(keys, p0)
    x_aug = ops.som_decenter_ragged(pts, off, idx, cm, k, True)
    fpo = ops.pointresnet_tc(x_aug, blob, fpar, f16=tc == "fp16")
    out_idx, val = ops.index_max_ragged(fpo[0], idx, off, M, k)
    assert torch.equal(fused.view(torch.int32), val.view(torch.int32))
    o = off.tolist()
    for b in range(len(sizes)):   # index_max's own definition, per cloud, on the dense layout
        blk = fpo[:, :, k * o[b]:k * o[b + 1]].contiguous()
        want_i, want_v = ops.index_max(blk, idx[k * o[b]:k * o[b + 1]].view(1, -1).contiguous(), M,
                                       with_values=True)
        assert torch.equal(out_idx[b], want_i[0]), b
        assert torch.equal(val[b].view(torch.int32), want_v[0].view(torch.int32)), b
    if edge == "one_node":
        cnt = torch.bincount(idx[:k * 500].long(), minlength=M)
        empty = (cnt == 0).nonzero().view(-1)
        assert len(empty) == M - 1
        assert torch.equal(fused[0][:, empty], fpo[0, :, 0:1].expand(-1, len(empty)))
    if edge == "sentinel":
        assert torch.equal(fused[:, 0::2, :], p0[:, 0::2, None].expand(-1, -1, M))


# ---- 5. the reference golden as a ragged set ------------------------------------------------------
def test_golden_clouds_as_ragged_set():
    g = golden("classifier_b2_n256")
    opt, inp, seed = golden_case(g, "classifier")
    st = build_states("classifier", opt, seed)
    opt.device, opt.gpu_id = torch.device(DEV), 0
    m = classifier.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.classifier.load_state_dict(st["head"])
    m.encoder.eval()
    m.classifier.eval()
    pts, off = _as_ragged(inp["pc"], inp["sn"])
    node, knn = inp["node"].to(DEV), inp["node_knn_I"].to(DEV)
    assert_golden(g, "feature", m.encoder.forward_ragged(pts, off, node, knn))
    assert_golden(g, "score", m.score_clouds(pts, off, node, knn))


# ---- 6. model state untouched ---------------------------------------------------------------------
def test_classifier_graph_state_untouched(monkeypatch):
    m = _cls(monkeypatch, "1", B=3, N=512)
    m.enable_cuda_graph(True)
    inp = synth.synth_inputs(3, 512, 64, 9, seed=21)
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    m.test_model()
    s1, f1 = m.score.clone(), m.encoder.feature.clone()
    sn1 = m.encoder.som_node.clone()
    pts, off, node, knn = _clouds([900, 3000, 12], 64, 9, seed=5)
    m.score_clouds(pts, off, node)                       # node_knn_I computed
    assert torch.equal(m.score, s1) and torch.equal(m.encoder.som_node, sn1)
    m.test_model()
    assert torch.equal(m.score, s1)
    assert torch.equal(m.encoder.feature, f1)
    assert torch.equal(m.encoder.som_node, sn1)


def test_segmenter_state_untouched(monkeypatch):
    monkeypatch.setenv("SONET_TC", "1")
    B, N, M = 2, 256, 64
    opt = synth.make_opt("segmenter", batch_size=B, input_pc_num=N)
    st = build_states("segmenter", opt, 8)
    opt.device, opt.gpu_id = torch.device(DEV), 0
    m = segmenter.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.segmenter.load_state_dict(st["head"])
    pts, off, node, knn = _clouds([700, 1500], M, 9, seed=6)
    rs = np.random.RandomState(0)
    o = off.tolist()
    sel = [o[b] + rs.choice(o[b + 1] - o[b], N, replace=False) for b in range(B)]
    pc = torch.stack([pts[s, :3].t() for s in sel]).cpu()
    sn = torch.stack([pts[s, 3:].t() for s in sel]).cpu()
    label = torch.tensor([1, 2])
    seg = torch.zeros(B, N, dtype=torch.int64)
    m.set_input(pc, sn, label, seg, node.cpu(), knn.cpu())
    m.test_model()
    want = m.score_points(pts, off)
    m.encoder.forward_ragged(pts, off, node, knn)
    assert torch.equal(m.score_points(pts, off), want)


def test_full_batch_feeds_score_clouds(monkeypatch):
    m = _cls(monkeypatch, "1", B=2, N=256)
    rs = np.random.RandomState(1)
    clouds = [rs.uniform(-1, 1, size=(P, 6)).astype(np.float32) for P in (400, 900, 1300)]
    nodes = [c[rs.choice(len(c), 64, replace=False), :3] for c in clouds]
    ds = augmentation.DeviceDataset(clouds, [1, 2, 3], nodes, device=DEV)
    pts, off, label, som, knn = ds.full_batch([2, 0], m.opt)
    assert off.tolist() == [0, 1300, 1700] and label.tolist() == [3, 1]
    assert torch.equal(som, ds.som_nodes[[2, 0]])
    assert torch.equal(knn, augmentation.som_knn(som, 9, 64))
    s = m.score_clouds(pts, off, som, knn)
    assert s.shape == (2, 40) and torch.isfinite(s).all()
