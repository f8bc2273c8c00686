"""-m gpu: kernel-level parity of the CUDA path (through the C-ABI) against the oracle.
Integer/index outputs bit-exact; fp32 within TOL = 1e-4 * max(|ref|, 1) (helpers.TOL)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import assert_close, golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rand_case(rs, B, C, N, K, ties=True, empty=True):
    data = torch.from_numpy(rs.normal(size=(B, C, N)).astype(np.float32))
    if ties and N > 16:
        data[:, :, ::5] = data[:, :, 1::5][:, :, :data[:, :, ::5].shape[2]]
    index = torch.from_numpy(rs.randint(0, K, size=(B, N)).astype(np.int32))
    if empty and K > 3:
        index[index == 2] = 0
    return data, index


# ---- index_max --------------------------------------------------------------------------------
# golden vectors, eight shapes and one full-size property test; test_gpu_pool_envelope.py reaches every
# branch of the launcher, the -1000 sentinel and non-finite values on purpose
def test_index_max_golden_reference_binary():
    from sonet_b200 import index_max
    g = golden("index_max")
    for tag, K in (("kat", 5), ("a", int(g["a_K"])), ("b", int(g["b_K"]))):
        d = torch.from_numpy(g[tag + "_data"]).to(DEV)
        i = torch.from_numpy(g[tag + "_index"]).to(DEV)
        for fn in (index_max.forward_cuda, index_max.forward_cuda_shared_mem):
            out = fn(d, i, K)
            assert out.dtype == torch.int32 and out.is_cuda
            assert np.array_equal(out.cpu().numpy(), g[tag + "_out"]), tag


@pytest.mark.parametrize("B,C,N,K", [
    (2, 384, 3072, 64),      # cfg-1 shape per cloud (vector path, several chunks)
    (3, 37, 1000, 64),       # N % 4 == 0, C not a multiple of the warp count
    (2, 16, 1023, 64),       # N % 4 != 0 -> scalar path
    (1, 5, 7, 3),            # tiny
    (2, 8, 2048 * 3 + 4, 64),  # chunk boundary + 1 vector
    (2, 4, 512, 256),        # K at the limit (fewer warps per CTA)
    (1, 3, 70000, 40),       # N > 65536 -> 32-bit index table
    (1, 20, 128, 1),         # single node
])
def test_index_max_vs_oracle(oracle_mod, B, C, N, K):
    from sonet_b200 import ops
    rs = np.random.RandomState(B * 1000 + C + N + K)
    data, index = _rand_case(rs, B, C, N, K)
    data[0, 0, :] = -1500.0                               # never beats the -1000 sentinel -> idx 0
    want = oracle_mod.index_max(data, index, K)
    idx, val = ops.index_max(data.to(DEV), index.to(DEV), K, with_values=True)
    assert torch.equal(idx.cpu(), want)
    # fused masked gather (models/networks.py:185): value at the arg-max; point 0 if never updated
    row_has = torch.zeros(B, K, dtype=torch.int64).scatter_(1, index.long(), 1)
    ref_val = torch.gather(data, 2, want.long() * row_has.unsqueeze(1))
    assert torch.equal(val.cpu(), ref_val)


def test_index_max_misaligned_views_and_repeatability(oracle_mod):
    from sonet_b200 import ops
    rs = np.random.RandomState(5)
    data, index = _rand_case(rs, 2, 9, 1028, 64)
    base = torch.zeros(2 * 9 * 1028 + 1, dtype=torch.float32, device=DEV)
    view = base[1:].view(2, 9, 1028)                      # 4-byte aligned only
    view.copy_(data)
    out = ops.index_max(view, index.to(DEV), 64)
    assert torch.equal(out.cpu(), oracle_mod.index_max(data, index, 64))
    again = ops.index_max(view, index.to(DEV), 64)
    assert torch.equal(out, again)


def test_index_max_full_size_properties():
    """cfg-2 size (B=64,C=384,kN=15000): checked through size-independent properties —
    (1) gather(data, idx) equals a torch segmented amax, (2) idx is the FIRST arg-max,
    (3) idempotent under channel permutation."""
    from sonet_b200 import ops
    B, C, N, K = 64, 384, 15000, 64
    g = torch.Generator(device=DEV).manual_seed(0)
    data = torch.randn(B, C, N, device=DEV, generator=g)
    data = (data * 8).round() / 8                          # many exact ties
    index = torch.randint(0, K, (B, N), device=DEV, generator=g, dtype=torch.int32)
    idx, val = ops.index_max(data, index, K, with_values=True)
    seg = torch.full((B, C, K), -1000.0, device=DEV)
    seg.scatter_reduce_(2, index.long().unsqueeze(1).expand(B, C, N), data, reduce="amax",
                        include_self=True)
    assert torch.equal(val, seg)
    # first arg-max: no earlier point of the same node has the same value
    sel = slice(0, 4)
    d, ix, vv = data[sel, :8], index[sel].long(), val[sel, :8]
    node_of = ix.unsqueeze(1).expand(-1, 8, -1)
    is_max = d == torch.gather(vv, 2, node_of)
    pos = torch.arange(N, device=DEV).view(1, 1, N).expand_as(d)
    first = torch.full((4, 8, K), N, device=DEV, dtype=torch.int64)
    first.scatter_reduce_(2, node_of, torch.where(is_max, pos, N), reduce="amin", include_self=True)
    assert torch.equal(first, idx[sel, :8].long())
    perm = torch.randperm(C, device=DEV)
    idx_p = ops.index_max(data[:, perm].contiguous(), index, K)
    assert torch.equal(idx_p, idx[:, perm])


# ---- SOM assignment ---------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N,M,k,mode", [(3, 1024, 64, 3, "sampled"), (2, 777, 64, 3, "uniform"),
                                          (2, 100, 16, 2, "uniform"), (1, 5000, 64, 3, "sampled"),
                                          (2, 64, 64, 1, "uniform"), (1, 3, 4, 3, "uniform")])
def test_som_assign_vs_oracle(oracle_mod, B, N, M, k, mode):
    from sonet_b200 import ops, synth
    inp = synth.synth_inputs(B, N, M, som_k=min(9, M), seed=N + M, node_mode=mode)
    x, node = inp["pc"], inp["node"]
    want_idx, _ = oracle_mod.som_topk(x, node, k)
    a = ops.som_assign(x.to(DEV), node.to(DEV), k, want_i64=True)
    # our kernel and the C restatement define the same slot order -> exact equality, which
    # implies the per-point set equality the parity definition asks for
    assert torch.equal(a["min_idx_i32"].cpu(), want_idx)
    assert torch.equal(a["min_idx_i64"].cpu(), want_idx.long())
    assert a["min_idx_i64"].dtype == torch.int64
    mask, row_max, _ = oracle_mod.query_topk(x, node, k)
    assert torch.equal(oracle_mod.canon_sets(a["min_idx_i32"].cpu(), k),
                       oracle_mod.canon_sets(torch.max(mask, 2)[1], k))
    assert torch.equal(a["row_max"].cpu(), row_max)
    assert torch.equal(a["count"].cpu().long(), mask.sum(dim=1))
    x_stack = torch.cat((x,) * k, dim=2)
    cm = torch.sum(x_stack.unsqueeze(3) * mask.unsqueeze(1).float(), dim=2) / \
        (mask.sum(dim=1).unsqueeze(1).float() + 1e-5)
    assert_close(a["cluster_mean"], cm, "cluster_mean")
    # dense mask (API of query_topk): bit-exact given the indices
    m2 = ops.som_mask(a["min_idx_i32"], M)
    assert m2.dtype == torch.int32
    assert torch.equal(m2.cpu(), F.one_hot(want_idx.long(), M).int())
    # centres / decentring
    x_aug, centers = ops.som_decenter(x.to(DEV), inp["sn"].to(DEV), a["cluster_mean"],
                                      a["min_idx_i32"], k, want_centers=True)
    cmean = a["cluster_mean"].cpu()
    ctr = torch.gather(cmean, 2, want_idx.long().unsqueeze(1).expand(-1, 3, -1))
    assert torch.equal(centers.cpu(), ctr)
    assert torch.equal(x_aug[:, :3].cpu(), x_stack - ctr)
    assert torch.equal(x_aug[:, 3:].cpu(), torch.cat((inp["sn"],) * k, dim=2))


def test_batchsom_query_topk_api(oracle_mod):
    from sonet_b200 import som, synth
    inp = synth.synth_inputs(2, 200, 64, seed=9, node_mode="uniform")
    bs = som.BatchSOM(8, 8, 3, 0, 2)
    bs.node = inp["node"].to(DEV)
    mask, row_max, min_idx = bs.query_topk(inp["pc"].to(DEV), 3)
    assert mask.shape == (2, 600, 64) and mask.dtype == torch.int32
    assert min_idx.dtype == torch.int64 and row_max.dtype == torch.int32
    rmask, rrow, _ = oracle_mod.query_topk(inp["pc"], inp["node"], 3)
    N = 200
    # set parity: the multiset of rows {slot s of point n} matches per point
    ours = mask.cpu().view(2, 3, N, 64).sum(1)
    ref = rmask.view(2, 3, N, 64).sum(1)
    assert torch.equal(ours, ref)
    assert torch.equal(row_max.cpu(), rrow)


# ---- point-wise layer, linear, rowmax, gathers ------------------------------------------------------
@pytest.mark.parametrize("B,C0,C1,P,Cout,relu", [
    (2, 6, 0, 3072, 64, True), (2, 64, 0, 3072, 128, True), (1, 64, 256, 1500, 384, False),
    (2, 387, 0, 576, 512, True), (2, 3, 512, 64, 768, True), (1, 128, 0, 1023, 50, False),
    (1, 5, 0, 7, 3, True), (1, 3356, 0, 256, 1024, True)])
def test_pointwise_layer_vs_torch(B, C0, C1, P, Cout, relu):
    from sonet_b200 import ops
    rs = np.random.RandomState(C0 + P)
    x0 = torch.from_numpy(rs.normal(size=(B, C0, P)).astype(np.float32))
    x1 = torch.from_numpy(rs.normal(size=(B, C1, P)).astype(np.float32)) if C1 else None
    W = torch.from_numpy((rs.normal(size=(Cout, C0 + C1)) * np.sqrt(2.0 / (C0 + C1))).astype(np.float32))
    scale = torch.from_numpy(rs.uniform(0.5, 1.5, size=Cout).astype(np.float32))
    shift = torch.from_numpy(rs.normal(size=Cout).astype(np.float32))
    xin = x0 if x1 is None else torch.cat((x0, x1), 1)
    want = F.conv1d(xin.double(), W.double().unsqueeze(2)) * scale.double()[None, :, None] \
        + shift.double()[None, :, None]
    want = (F.relu(want) if relu else want).float()
    got = ops.pointwise_layer(x0.to(DEV), W.t().contiguous().to(DEV), scale.to(DEV), shift.to(DEV),
                              relu, x1=None if x1 is None else x1.to(DEV))
    assert_close(got, want, "pointwise layer", 2e-5)


def test_pointwise_layer_gathered_addend():
    from sonet_b200 import ops
    rs = np.random.RandomState(0)
    B, C0, P, Cout, G = 2, 24, 1536, 128, 64
    x0 = torch.from_numpy(rs.normal(size=(B, C0, P)).astype(np.float32))
    W = torch.from_numpy(rs.normal(size=(Cout, C0)).astype(np.float32))
    add = torch.from_numpy(rs.normal(size=(B, Cout, G)).astype(np.float32))
    gidx = torch.from_numpy(rs.randint(0, G, size=(B, P)).astype(np.int32))
    want = F.relu(F.conv1d(x0, W.unsqueeze(2)) +
                  torch.gather(add, 2, gidx.long().unsqueeze(1).expand(B, Cout, P)))
    got = ops.pointwise_layer(x0.to(DEV), W.t().contiguous().to(DEV), None, None, True,
                              addend=add.to(DEV), gidx=gidx.to(DEV))
    assert_close(got, want, "pointwise + gathered addend", 2e-5)


def test_linear_rowmax_kcopy():
    from sonet_b200 import ops
    rs = np.random.RandomState(1)
    x = torch.from_numpy(rs.normal(size=(5, 1024)).astype(np.float32))
    W = torch.from_numpy((rs.normal(size=(40, 1024)) / 32).astype(np.float32))
    shift = torch.from_numpy(rs.normal(size=40).astype(np.float32))
    want = F.relu(F.linear(x, W) + shift)
    assert_close(ops.linear(x.to(DEV), W.to(DEV), None, shift.to(DEV), True), want, "linear", 2e-5)
    # rows are independent: a sub-batch gives the same bits
    xb = torch.from_numpy(rs.normal(size=(67, 1024)).astype(np.float32)).to(DEV)
    full = ops.linear(xb, W.to(DEV), None, shift.to(DEV), False)
    assert torch.equal(ops.linear(xb[:3].contiguous(), W.to(DEV), None, shift.to(DEV), False), full[:3])
    assert_close(full.cpu(), F.linear(xb.cpu(), W) + shift, "linear B=67", 2e-5)
    assert torch.equal(ops.linear(xb[66:].contiguous(), W.to(DEV), None, shift.to(DEV), False), full[66:])
    # the tiled kernel with ragged Cout and B and a folded scale, the blocked kernel with one
    # channel per block (Cin 12288) and the warp-per-output kernel (Cin % 4 != 0);
    # test_gpu_fp32_envelope.py reaches every branch of the launcher on purpose
    for B_, cin, cout in ((64, 1024, 512), (64, 512, 256), (33, 1040, 1024), (7, 256, 41), (1, 64, 3),
                          (5, 1030, 17), (4, 12288, 8)):
        x = torch.from_numpy(rs.normal(size=(B_, cin)).astype(np.float32))
        W2 = torch.from_numpy((rs.normal(size=(cout, cin)) / np.sqrt(cin)).astype(np.float32))
        sc = torch.from_numpy(rs.uniform(0.5, 2.0, size=cout).astype(np.float32))
        sh = torch.from_numpy(rs.normal(size=cout).astype(np.float32))
        want = F.relu(F.linear(x.double(), W2.double()) * sc.double() + sh.double())
        got = ops.linear(x.to(DEV), W2.to(DEV), sc.to(DEV), sh.to(DEV), True)
        assert_close(got, want, "linear %s" % ((B_, cin, cout),), 2e-5)
    for shape in ((3, 7, 64), (5, 3, 128), (2, 1033, 64), (2, 3, 40), (3, 5, 16)):
        t = torch.from_numpy(rs.normal(size=shape).astype(np.float32))
        assert torch.equal(ops.rowmax(t.to(DEV)).cpu(), t.max(dim=2)[0]), shape
    t = torch.from_numpy(rs.normal(size=(2, 6, 5, 9)).astype(np.float32))
    assert torch.equal(ops.rowmax(t.to(DEV)).cpu(), t.max(dim=3)[0])
    t = torch.from_numpy(rs.normal(size=(2, 4, 300)).astype(np.float32))
    sp = torch.split(t, 100, dim=2)
    assert torch.equal(ops.kcopy_mean(t.to(DEV), 3).cpu(), (1.0 / 3.0) * (sp[0] + sp[1] + sp[2]))
    sp = torch.split(t, 150, dim=2)
    assert torch.equal(ops.kcopy_mean(t.to(DEV), 2).cpu(), 0.5 * (sp[0] + sp[1]))
    # scalar path (N % 4 != 0) and an offset (not 16-byte aligned) view
    t = torch.from_numpy(rs.normal(size=(3, 5, 3 * 101)).astype(np.float32))
    sp = torch.split(t, 101, dim=2)
    assert torch.equal(ops.kcopy_mean(t.to(DEV), 3).cpu(), (1.0 / 3.0) * (sp[0] + sp[1] + sp[2]))


def test_seg_loss_vs_torch():
    """CrossEntropyLossSeg (models/losses.py:30-43): log_softmax over classes + NLL, mean / sum,
    NLLLoss's default ignore_index, ragged N; against PyTorch in fp64."""
    import torch.nn.functional as F
    from sonet_b200 import losses, ops
    rs = np.random.RandomState(21)
    for B, C, N in ((32, 50, 1024), (3, 50, 1000), (2, 7, 33), (1, 1, 1)):
        score = torch.from_numpy((rs.normal(size=(B, C, N)) * 4).astype(np.float32))
        tgt = torch.from_numpy(rs.randint(0, C, size=(B, N)).astype(np.int64))
        for avg in (True, False):
            got = ops.seg_loss(score.to(DEV), tgt.to(DEV), size_average=avg)
            want = F.cross_entropy(score.double(), tgt, reduction='mean' if avg else 'sum')
            assert abs(float(got) - float(want)) <= 2e-6 * max(1.0, abs(float(want))), (B, C, N, avg)
        # bit-reproducible
        assert torch.equal(ops.seg_loss(score.to(DEV), tgt.to(DEV)), ops.seg_loss(score.to(DEV), tgt.to(DEV)))
        if N > 4:
            tgt2 = tgt.clone()
            tgt2[:, ::3] = -100
            got = ops.seg_loss(score.to(DEV), tgt2.to(DEV))
            want = F.cross_entropy(score.double(), tgt2)
            assert abs(float(got) - float(want)) <= 2e-6 * max(1.0, abs(float(want)))
    # out-of-range target: loud (NaN), never a silent wrong number
    bad = torch.full((1, 8), 9, dtype=torch.int64)
    assert torch.isnan(ops.seg_loss(torch.zeros(1, 5, 8, device=DEV), bad.to(DEV)))
    # the module takes the kernel path in eval and PyTorch's when a gradient is wanted
    crit = losses.CrossEntropyLossSeg()
    sc = score.to(DEV)
    n0 = ops.LAUNCHES
    with torch.no_grad():
        a = crit(sc, tgt.to(DEV))
    assert ops.LAUNCHES == n0 + 1
    sc.requires_grad_(True)
    b = crit(sc, tgt.to(DEV))
    assert ops.LAUNCHES == n0 + 1 and b.requires_grad
    assert abs(float(a) - float(b.detach())) <= 1e-5 * max(1.0, abs(float(b.detach())))


def test_knn_gather_assemble_node_knn(oracle_mod):
    from sonet_b200 import operations, ops, synth
    inp = synth.synth_inputs(2, 300, 64, som_k=9, seed=4)
    node = inp["node"]
    knn = inp["node_knn_I"]
    feat = torch.from_numpy(np.random.RandomState(2).normal(size=(2, 20, 64)).astype(np.float32))
    want = oracle_mod.knn_gather(feat, knn)
    assert torch.equal(operations.knn_gather_by_indexing(feat.to(DEV), knn.to(DEV)).cpu(), want)
    assert torch.equal(operations.knn_gather_wrapper(node.to(DEV), knn.to(DEV)).cpu(),
                       oracle_mod.knn_gather(node, knn))
    # first K of a wider precomputed table (layers.py:332)
    g5 = ops.knn_gather(feat.to(DEV), knn.to(DEV), K=5)
    assert torch.equal(g5.cpu(), want[..., :5])
    for ct in ("avg", "center"):
        center, x_aug = ops.knn_assemble(node.to(DEV), feat.to(DEV), knn.to(DEV), 9, ct)
        nb = oracle_mod.knn_gather(node, knn)
        c = nb.mean(dim=3, keepdim=True) if ct == "avg" else node.unsqueeze(3)
        ref = torch.cat((nb - c, want), dim=1).view(2, 23, 64 * 9)
        assert_close(center, c.squeeze(3), "knn center " + ct, 1e-6)
        assert_close(x_aug, ref, "knn x_aug " + ct, 1e-6)
    # on-device exact node kNN == the loader's sorted kNN (no exact ties in sampled nodes)
    assert torch.equal(ops.node_knn(node.to(DEV), 9).cpu(), knn)
    assert torch.equal(ops.node_knn(node.to(DEV), 9).cpu(), oracle_mod.node_knn(node, 9))
    gi = torch.from_numpy(np.random.RandomState(3).randint(0, 64, size=(2, 500)).astype(np.int32))
    want = torch.gather(feat, 2, gi.long().unsqueeze(1).expand(2, 20, 500))
    assert torch.equal(ops.gather_points(feat.to(DEV), gi.to(DEV)).cpu(), want)


# ---- Chamfer -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,Mp,N", [(2, 96, 200), (3, 256, 1000), (1, 1280, 5000), (2, 1, 3)])
def test_chamfer_vs_oracle(oracle_mod, B, Mp, N):
    from sonet_b200 import ops
    rs = np.random.RandomState(Mp + N)
    pred = torch.from_numpy(rs.uniform(-1, 1, size=(B, 3, Mp)).astype(np.float32))
    gt = torch.from_numpy(rs.uniform(-1, 1, size=(B, 3, N)).astype(np.float32))
    want = oracle_mod.chamfer(pred, gt)
    r = ops.chamfer(pred.to(DEV), gt.to(DEV), want_idx=True)
    assert torch.equal(r["idx_fwd"].cpu().long(), want["idx_fwd"])      # exact NN indices
    assert torch.equal(r["idx_bwd"].cpu().long(), want["idx_bwd"])
    assert_close(r["loss"][2], want["loss"], "chamfer loss")
    assert_close(r["loss"][0], want["forward_loss"], "forward")
    assert_close(r["loss"][1], want["backward_loss"], "backward")
    assert_close(r["fwd_arr"] + r["bwd_arr"], want["loss_array"], "loss_array")


def test_chamfer_ties_lowest_index_and_value_only_path(oracle_mod):
    """Exact duplicates in both clouds: every query has several equidistant neighbours; the
    arg-min pass must return the LOWEST index (the oracle's strict '<' ascending scan), and the
    eval-mode value-only path must give bit-identical element losses."""
    from sonet_b200 import ops
    rs = np.random.RandomState(77)
    a = rs.uniform(-1, 1, size=(2, 3, 300)).astype(np.float32)
    g = rs.uniform(-1, 1, size=(2, 3, 700)).astype(np.float32)
    pred = torch.from_numpy(np.concatenate([a, a[:, :, ::-1], a[:, :, :57]], axis=2).copy())   # 657
    gt = torch.from_numpy(np.concatenate([g, g, g[:, :, 100:400]], axis=2).copy())              # 1700
    want = oracle_mod.chamfer(pred, gt)
    r = ops.chamfer(pred.to(DEV), gt.to(DEV), want_idx=True)
    assert torch.equal(r["idx_fwd"].cpu().long(), want["idx_fwd"])
    assert torch.equal(r["idx_bwd"].cpu().long(), want["idx_bwd"])
    assert int(r["idx_fwd"].max()) < 700 and int(r["idx_bwd"].max()) < 300      # never the copies
    v = ops.chamfer(pred.to(DEV), gt.to(DEV), want_idx=False)
    for k in ("elem_fwd", "elem_bwd", "fwd_arr", "bwd_arr", "loss"):
        assert torch.equal(v[k], r[k]), k
    assert_close(v["loss"][2], want["loss"], "chamfer loss with ties")


def test_chamfer_golden_and_properties():
    from sonet_b200 import losses, ops, synth
    g = golden("autoencoder_b2_n256")
    crit = losses.ChamferLoss(synth.make_opt("autoencoder"))
    with torch.no_grad():
        loss = crit(torch.from_numpy(g["ch_pred"]).to(DEV), torch.from_numpy(g["ch_gt"]).to(DEV))
    assert_close(loss, g["ch_loss"], "golden chamfer loss")
    assert_close(crit.loss_array, g["ch_loss_array"], "golden loss_array")
    assert_close(crit.forward_loss, g["ch_forward_loss"], "golden forward")
    assert_close(crit.backward_loss, g["ch_backward_loss"], "golden backward")
    # identical clouds -> every NN distance 0 -> loss = 2*sqrt(1e-8); permutation invariance
    x = torch.rand(2, 3, 777, device=DEV)
    r = ops.chamfer(x, x.clone(), want_idx=True)
    assert torch.equal(r["idx_fwd"], torch.arange(777, device=DEV, dtype=torch.int32).expand(2, 777))
    assert_close(r["loss"][2], 2e-4, "self chamfer", 1e-6)
    p = torch.randperm(777, device=DEV)
    r2 = ops.chamfer(x[:, :, p].contiguous(), x, want_idx=False)
    assert_close(r2["loss"][2], 2e-4, "permuted self chamfer", 1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,M,k,use_sn,mode", [(3, 1000, 64, 3, True, "sampled"),
                                                  (2, 777, 64, 3, False, "uniform"),
                                                  (2, 5000, 64, 3, True, "sampled"),
                                                  (2, 130, 16, 2, True, "sampled")])
def test_som_group_decenter_matches_two_kernel_path(B, N, M, k, use_sn, mode):
    """sonet_som_group_decenter (statistics + stable sort + decentre, one launch) against
    sonet_som_assign's statistics + a torch stable sort: counts equal, means within fp32 sum
    reordering, rows in ascending stacked order inside every node, decentring bit-exact given
    the kernel's own means, pos0 = sorted position of stacked copy 0; repeatable bit for bit."""
    from sonet_b200 import ops, synth
    inp = synth.synth_inputs(B, N, M, seed=N, node_mode=mode)
    x, sn, node = inp["pc"].to(DEV), inp["sn"].to(DEV), inp["node"].to(DEV)
    if mode == "uniform":
        node[:, :, 2:5] += 40.0                      # empty nodes
    a = ops.som_assign(x, node, k)
    idx = a["min_idx_i32"]
    xs, ns, p0, count, cmean = ops.som_group_decenter(x, sn if use_sn else None, idx, M, k)
    xs2, ns2, p02, count2, cmean2 = ops.som_group_decenter(x, sn if use_sn else None, idx, M, k)
    for u, v in ((xs, xs2), (ns, ns2), (p0, p02), (count, count2), (cmean, cmean2)):
        assert torch.equal(u, v)
    assert torch.equal(count, a["count"])
    assert_close(cmean, a["cluster_mean"], "cluster_mean", tol=1e-5)
    order = torch.argsort(idx.long(), dim=1, stable=True)             # [B,kN]
    assert torch.equal(ns.long(), torch.gather(idx.long(), 1, order))
    n_of = order % N
    x_g = torch.gather(x, 2, n_of.unsqueeze(1).expand(-1, 3, -1))
    ctr = torch.gather(cmean, 2, ns.long().unsqueeze(1).expand(-1, 3, -1))
    assert torch.equal(xs[:, 0:3], x_g - ctr)
    if use_sn:
        assert torch.equal(xs[:, 3:6], torch.gather(sn, 2, n_of.unsqueeze(1).expand(-1, 3, -1)))
    assert torch.equal(p0.long(), (order == 0).long().argmax(dim=1))


@pytest.mark.gpu
@pytest.mark.parametrize("center_type", ["avg", "center"])
def test_knn_assemble_pool_equals_finalize_then_assemble(center_type):
    """sonet_knn_assemble_pool_f32 == sonet_pool_finalize + sonet_knn_assemble_f32, bit for bit,
    incl. untouched keys (empty node -> copy-0 feature), values <= -1000, and the key reset."""
    from sonet_b200 import ops
    B, C, M, K = 3, 37, 64, 9
    g = torch.Generator().manual_seed(7)
    vals = torch.randn(B, C, M, generator=g) * 3
    vals[0, :, 5] = -2000.0                                           # fails the > -1000 test
    bits = vals.view(torch.int32)
    keys = (bits ^ ((bits >> 31) & 0x7fffffff)).to(DEV)
    keys[1, :, 7] = -2 ** 31                                          # never written: empty node
    p0 = torch.randn(B, C, generator=g).to(DEV)
    coord = torch.randn(B, 3, M, generator=g).to(DEV)
    idx = torch.randint(0, M, (B, M, K + 2), generator=g).to(DEV)
    k1, k2 = keys.clone(), keys.clone()
    want_mm = ops.pool_finalize(k1, p0)
    want_center, want_x = ops.knn_assemble(coord, want_mm, idx, K, center_type)
    center, x_aug, mm = ops.knn_assemble_pool(coord, k2, p0, idx, K, center_type)
    assert torch.equal(mm, want_mm) and torch.equal(center, want_center)
    assert torch.equal(x_aug, want_x)
    assert bool((k2 == -2 ** 31).all()) and bool((k1 == -2 ** 31).all())
    assert torch.equal(want_mm[0, :, 5], p0[0]) and torch.equal(want_mm[1, :, 7], p0[1])
