"""Training the classifier on whole clouds (classifier.Model.optimize_clouds) on the GPU: the ragged
BatchNorm records, fold, apply and backward against BNActTrain on the same data laid out [B,C,P]
and against an fp64 restatement at mixed sizes; the ragged pool backward against the dense one and
a numpy scatter; the ragged augmentation against ops.augment; the full step against dense
optimize() at equal sizes and against an fp64 CPU restatement at mixed sizes; determinism,
interleaving with a graphed optimize(), score_clouds after training and a short training run."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn

from helpers import build_states
from sonet_b200 import augmentation, classifier, ops, synth, train_ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REC_FWD = 3
STEP_GRAD_TOL = 1e-4      # test_gpu_train_parity.py's bar, in units of each tensor's largest gradient


def _cols(sizes):
    return torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)).to(DEV)


def _ragged_of(x):
    """[B,C,P] -> [1,C,B*P], cloud b's columns b*P .. (b+1)*P."""
    B, C, P = x.shape
    return x.permute(1, 0, 2).reshape(1, C, B * P).contiguous()


def _dense_of(y, B):
    C = y.shape[1]
    return y.reshape(C, B, -1).permute(1, 0, 2).contiguous()


def _bn_data(B, C, P, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, P, generator=g) * 2 + 0.5
    x[:, 0] += 3e3                          # a channel behind a large bias
    x[:, 1] = x[:, 1] * 1e-3 - 7.0
    dy = torch.randn(B, C, P, generator=g)
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g) * 0.1
    return [t.to(DEV) for t in (x, dy, gamma, beta)]


# ---- 1. BatchNorm records, fold, apply and backward ------------------------------------------------
@pytest.mark.parametrize("P", [1, 2, 31, 32, 1023, 1024, 1025, 15000])
@pytest.mark.parametrize("act", ["relu", "elu", None])
def test_bn_equal_sizes_give_dense_bits(P, act):
    B, C = 3, 5
    x, dy, gamma, beta = _bn_data(B, C, P, P)
    cols = _cols([P] * B)
    code = ops.act_code(act)
    # the dense entries: forward through BNActTrain, backward by autograd
    xd = x.clone().requires_grad_(True)
    gd, bd = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    y, mean, var = train_ops.BNActTrain.apply(xd, gd, bd, 1e-5, act)
    y.backward(dy)
    xr = _ragged_of(x).requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    yr, mr, vr = train_ops.BNActTrain.apply(xr, gr, br, 1e-5, act, cols)
    yr.backward(_ragged_of(dy))
    assert torch.equal(mr, mean) and torch.equal(vr, var)
    assert torch.equal(_dense_of(yr.detach(), B), y.detach())
    assert torch.equal(_dense_of(xr.grad, B), xd.grad)
    assert torch.equal(gr.grad, gd.grad) and torch.equal(br.grad, bd.grad)
    # the records themselves
    rec = torch.empty((B, C, REC_FWD), dtype=torch.float64, device=DEV)
    ops._call("sonet_bn_cloud_partials_f32", x.data_ptr(), None, None, None, None, None, B, C, P, code,
              0, rec.data_ptr(), ops._stream(x))
    assert torch.equal(ops.bn_cloud_partials_ragged(_ragged_of(x), cols), rec)


def _bn_fp64(x, dy, gamma, beta, sizes, act, eps=1e-5):
    """BatchNorm + act over all L columns of x [C,L] and its backward, in fp64."""
    x, dy, gamma, beta = (t.double().cpu() for t in (x, dy, gamma, beta))
    x = x.clone().requires_grad_(True)
    g, b = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    mean = x.mean(1, keepdim=True)
    var = ((x - mean) ** 2).mean(1, keepdim=True)
    z = g[:, None] * (x - mean) / torch.sqrt(var + eps) + b[:, None]
    y = torch.relu(z) if act == "relu" else (torch.nn.functional.elu(z) if act == "elu" else z)
    y.backward(dy)
    return y.detach(), mean[:, 0].detach(), var[:, 0].detach(), x.grad, g.grad, b.grad


@pytest.mark.parametrize("act", ["relu", "elu", None])
@pytest.mark.parametrize("sizes", [[1025, 3], [1, 40, 1025, 2, 3000, 7], [5000, 1]])
def test_bn_mixed_sizes_fp64(act, sizes):
    C = 6
    L = sum(sizes)
    x, dy, gamma, beta = _bn_data(1, C, L, L)
    cols = _cols(sizes)
    xr = x.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    yr, mr, vr = train_ops.BNActTrain.apply(xr, gr, br, 1e-5, act, cols)
    yr.backward(dy)
    y, m, v, dx, dg, db = _bn_fp64(x[0], dy[0], gamma, beta, sizes, act)
    scale = lambda t: t.abs().max().clamp(min=1e-30)  # noqa: E731
    assert float(((mr.double().cpu() - m).abs() / m.abs().clamp(min=1)).max()) <= 1e-6
    assert float(((vr.double().cpu() - v).abs() / v).max()) <= 1e-5
    # y and dx in fp32 carry the rounding of x - mean times invstd: 1e-4 of the largest on a
    # channel of std 2e-3 around -7
    assert float((yr[0].detach().double().cpu() - y).abs().max() / scale(y)) <= 1e-4
    assert float((xr.grad[0].double().cpu() - dx).abs().max() / scale(dx)) <= 1e-3
    assert float((gr.grad.double().cpu() - dg).abs().max() / scale(dg)) <= 1e-4
    assert float((br.grad.double().cpu() - db).abs().max() / scale(db)) <= 1e-4


def test_bn_ragged_running_var_uses_L():
    """norm_act_train with cols updates running_var with var * L/(L-1)."""
    from sonet_b200.layers import MyBatchNorm1d
    sizes = [7, 300, 2]
    L = sum(sizes)
    x, _, _, _ = _bn_data(1, 4, L, 5)
    bn = MyBatchNorm1d(4, momentum=0.1).to(DEV).train()
    _, _, var = train_ops.BNActTrain.apply(x, bn.weight, bn.bias, bn.eps, "relu", _cols(sizes))
    rv0 = bn.running_var.clone()
    train_ops.norm_act_train(x, bn, "relu", cols=_cols(sizes))
    torch.testing.assert_close(bn.running_var, rv0 * 0.9 + 0.1 * var * (L / (L - 1)), rtol=1e-6, atol=0)


# ---- 2. the pool backward -------------------------------------------------------------------------
def _pool_case(B, C, M, N, seed):
    g = torch.Generator().manual_seed(seed)
    go = torch.randn(B, C, M, generator=g)
    idx = torch.randint(0, N, (B, C, M), generator=g, dtype=torch.int32)
    idx[:, :, : M // 4] = 0                  # empty nodes gather copy 0
    idx[:, :, M // 4: M // 2] = idx[:, :, M // 2: M // 2 + M // 4]   # ties: one column twice
    idx[0, 0, 0] = -5                        # clamped
    idx[-1, -1, -1] = N + 9
    return go.to(DEV), idx.to(DEV)


@pytest.mark.parametrize("B,C,M,N", [(3, 384, 64, 300), (1, 7, 1, 1), (5, 130, 256, 2049)])
def test_pool_backward_equal_sizes_give_dense_bits(B, C, M, N):
    go, idx = _pool_case(B, C, M, N, N)
    dense = torch.empty((B, C, N), dtype=torch.float32, device=DEV)
    ops._call("sonet_index_max_backward_f32", go.data_ptr(), idx.data_ptr(), B, C, N, M,
              dense.data_ptr(), ops._stream(go))
    rag = ops.index_max_ragged_backward(go, idx, _cols([N] * B), B * N)
    assert torch.equal(_dense_of(rag.unsqueeze(0), B), dense)


def test_pool_backward_mixed_sizes_numpy():
    sizes = [300, 1, 47, 1025]
    B, C, M = len(sizes), 33, 64
    go, idx = _pool_case(B, C, M, 1, 3)
    g = torch.Generator().manual_seed(4)
    idx = torch.stack([torch.randint(-2, P + 2, (C, M), generator=g, dtype=torch.int32)
                       for P in sizes]).to(DEV)
    got = ops.index_max_ragged_backward(go, idx, _cols(sizes), sum(sizes)).cpu().numpy()
    ref = np.zeros((C, sum(sizes)), dtype=np.float32)
    off = np.concatenate([[0], np.cumsum(sizes)])
    gon, ixn = go.cpu().numpy(), idx.cpu().numpy()
    for b, P in enumerate(sizes):
        for c in range(C):
            for m in range(M):
                ref[c, off[b] + min(max(ixn[b, c, m], 0), P - 1)] += gon[b, c, m]
    assert np.array_equal(got, ref)


# ---- 3. augmentation ------------------------------------------------------------------------------
@pytest.mark.parametrize("rot1", [False, True])
@pytest.mark.parametrize("rot2", [False, True])
@pytest.mark.parametrize("shift", [False, True])
def test_augment_equal_sizes_give_dense_bits(rot1, rot2, shift):
    B, N, M = 3, 700, 64
    g = torch.Generator().manual_seed(11)
    pc, sn, som = torch.randn(B, 3, N, generator=g), torch.randn(B, 3, N, generator=g), \
        torch.randn(B, 3, M, generator=g)
    pc, sn, som = pc.to(DEV), sn.to(DEV), som.to(DEV)
    p = augmentation.draw_params(np.random.RandomState(5), B, N, M, rot_horizontal=rot1,
                                 rot_perturbation=rot2, translation_perturbation=shift)
    po, so, mo = augmentation.augment_batch(pc, sn, som, p, seed=77)
    pts = torch.cat((pc, sn), 1).permute(0, 2, 1).reshape(-1, 6).contiguous()
    d = augmentation._dev
    pr, mr = ops.augment_ragged(pts, _cols([N] * B), som, rot1=d(p["rot1"], DEV), rot2=d(p["rot2"], DEV),
                                scale=d(p["scale"], DEV), shift=d(p["shift"], DEV),
                                jitter_pc=augmentation.JITTER_PC, jitter_sn=augmentation.JITTER_PC,
                                jitter_som=augmentation.JITTER_SOM, seed=77)
    want = torch.cat((po, so), 1).permute(0, 2, 1).reshape(-1, 6)
    assert torch.equal(pr, want)
    assert torch.equal(mr, mo)


def test_augment_mixed_sizes_per_cloud():
    """Cloud b of a mixed batch gets the bits of cloud b of a dense batch at N = P_b."""
    sizes, M = [5, 1000, 1], 9
    g = torch.Generator().manual_seed(2)
    pts = torch.randn(sum(sizes), 6, generator=g).to(DEV)
    som = torch.randn(len(sizes), 3, M, generator=g).to(DEV)
    p = augmentation.draw_params(np.random.RandomState(1), len(sizes), 0, M, rot_horizontal=True,
                                 rot_perturbation=True, translation_perturbation=True)
    d = lambda a: augmentation._dev(a, DEV)  # noqa: E731
    pr, mr = ops.augment_ragged(pts, _cols(sizes), som, rot1=d(p["rot1"]), rot2=d(p["rot2"]),
                                scale=d(p["scale"]), shift=d(p["shift"]),
                                jitter_pc=augmentation.JITTER_PC, jitter_sn=augmentation.JITTER_PC,
                                jitter_som=augmentation.JITTER_SOM, seed=3)
    off = np.concatenate([[0], np.cumsum(sizes)])
    for b, P in enumerate(sizes):
        # cloud b as row b of a dense batch of B clouds of P points (the other clouds: copies)
        cl = pts[off[b]:off[b + 1]].T.contiguous()
        pc = cl[:3].unsqueeze(0).expand(len(sizes), 3, P).contiguous()
        sn = cl[3:].unsqueeze(0).expand(len(sizes), 3, P).contiguous()
        po, so, mo = augmentation.augment_batch(pc, sn, som, p, seed=3)
        assert torch.equal(pr[off[b]:off[b + 1]], torch.cat((po[b], so[b]), 0).T)
        assert torch.equal(mr[b], mo[b])


def test_full_batch_train_false_unchanged():
    pts, off, node, _ = _clouds([40, 7, 90], 16, 3, seed=1)
    ds = _dataset(pts, off, node)
    opt = synth.make_opt("classifier", node_num=16, som_k=3)
    got = ds.full_batch([2, 0], opt)
    points, offsets, _ = ds.full_clouds([2, 0])
    assert torch.equal(got[0], points) and torch.equal(got[1], offsets)
    assert torch.equal(got[3], ds.som_nodes[[2, 0]])
    assert torch.equal(got[4], augmentation.som_knn(got[3], 3, 16))


def test_full_batch_train_draws_like_batch():
    """full_batch(train=True) takes the per-cloud scalars from rng in batch(train=True,
    host_noise=False)'s order with the same dataset flags: from identically seeded rngs both give
    the same augmented nodes and kNN bit for bit and leave the rngs in the same state; every point
    of a cloud gets the same rotations, scale and shift (and only the shift skips the normals)."""
    pts, off, node, _ = _clouds([700, 512, 2000], 64, 9, seed=3)
    ds = _dataset(pts, off, node)
    idx = [2, 0, 1]
    for dataset in ("modelnet", "shrec"):
        opt = synth.make_opt("classifier", input_pc_num=512, dataset=dataset, rot_horizontal=True,
                             rot_perturbation=True, translation_perturbation=True)
        r0, r1 = np.random.RandomState(4), np.random.RandomState(4)
        _, _, _, som_b, knn_b = ds.batch(idx, opt, True, rng=r0, seed=9)
        p_f, o_f, _, som_f, knn_f = ds.full_batch(idx, opt, train=True, rng=r1, seed=9)
        assert torch.equal(som_f, som_b) and torch.equal(knn_f, knn_b)
        assert r0.randint(1 << 30) == r1.randint(1 << 30)
        # the same draws, applied by hand without jitter, give each cloud's rows up to the jitter clip
        r2 = np.random.RandomState(4)
        p = augmentation.draw_params(r2, len(idx), 0, 64, **augmentation._aug_flags(opt))
        src, o2, _ = ds.full_clouds(idx)
        d = lambda a: augmentation._dev(a, DEV)  # noqa: E731
        nj, _ = ops.augment_ragged(src.contiguous(), o2, None, rot1=d(p["rot1"]), rot2=d(p["rot2"]),
                                   scale=d(p["scale"]), shift=d(p["shift"]), seed=9)
        clip = augmentation.JITTER_PC[1] * 1.2 + 1e-5     # the clip, times the largest scale
        assert float((p_f - nj).abs().max()) <= clip


# ---- 4. the full step -----------------------------------------------------------------------------
def _clouds(sizes, M, som_k, seed, grid=None):
    """Clouds U(-1,1)^3 with unit normals and nodes drawn from them. grid: coordinates rounded to
    multiples of 1/grid, so that every cluster sum is exact in fp32 whatever its order."""
    rs = np.random.RandomState(seed)
    pts, nodes = [], []
    for P in sizes:
        xyz = rs.uniform(-1, 1, size=(P, 3)).astype(np.float32)
        if grid:
            xyz = np.round(xyz * grid).astype(np.float32) / grid
        n = rs.normal(size=(P, 3))
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        pts.append(np.concatenate([xyz, n.astype(np.float32)], axis=1))
        sel = rs.choice(P, M, replace=P < M)
        nodes.append(xyz[sel].T + rs.normal(0, 1e-2, size=(3, M)).astype(np.float32))
    node = torch.from_numpy(np.ascontiguousarray(np.stack(nodes), dtype=np.float32)).to(DEV)
    return torch.from_numpy(np.concatenate(pts)).to(DEV), _cols(sizes), node, \
        augmentation.som_knn(node, som_k, M)


def _dataset(pts, off, node, labels=None):
    o = off.cpu().numpy()
    B = len(o) - 1
    return augmentation.DeviceDataset.from_device(
        pts, off, torch.zeros(B, dtype=torch.int64, device=DEV) if labels is None else labels, node)


def _model(monkeypatch, tc, B, N, seed=5, **over):
    if tc == "fp16":
        monkeypatch.setenv("SONET_TRAIN_TC", "fp16")
    else:
        monkeypatch.delenv("SONET_TRAIN_TC", raising=False)
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, dropout=0.0, **over)
    st = build_states("classifier", opt, seed)
    opt.device, opt.gpu_id = torch.device(DEV), 0
    m = classifier.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.classifier.load_state_dict(st["head"])
    return m, st


def _state(m):
    mods = (m.encoder, m.classifier)
    state = {"%d.%s" % (i, k): v.detach().clone() for i, mm in enumerate(mods)
             for k, v in mm.state_dict().items()}
    grads = {"%d.%s" % (i, k): p.grad.detach().clone() for i, mm in enumerate(mods)
             for k, p in mm.named_parameters() if p.grad is not None}
    return state, grads


def _err(a, ref):
    return float((a.double() - ref.double()).abs().max() / ref.double().abs().max().clamp(min=1e-30))


def _check_grads(got, ref, other=None):
    """Each gradient within STEP_GRAD_TOL of its tensor's scale of ref's, or within 8x the
    difference of another arithmetic `other` of the same step (test_gpu_train_parity.py's fp64
    rule: 8x the error of a strict-fp32 run)."""
    assert set(got) == set(ref)
    for k, g in ref.items():
        if _zero_grad_bias(ref, k):
            continue
        bar = STEP_GRAD_TOL if other is None else max(STEP_GRAD_TOL, 8 * _err(other[k], g))
        assert _err(got[k], g) <= bar, "%s: gradient %.3e of its scale (bar %.3e)" % (
            k, _err(got[k], g), bar)


def _zero_grad_bias(grads, k):
    """A bias in front of a batch-statistics BN: its gradient is analytically zero, and what either
    arithmetic returns is rounding noise (test_gpu_train_parity.py's rule)."""
    w = k[:-4] + "weight"
    return (k.endswith(".bias") and w in grads
            and float(grads[k].abs().max()) < 1e-3 * float(grads[w].abs().max()))


def _check_step(on, g_on, off, g_off, before, lr, g_other=None, other=None):
    """test_optimize_step_state_dict_kernels_on_vs_off's bars, each gradient and running-statistic
    tolerance widened to 8x the other arithmetic's difference (g_other, other) where that is larger
    (_check_grads)."""
    for k, ref in off.items():
        got = on[k]
        if k.endswith("num_batches_tracked"):
            assert torch.equal(got, ref), k
        elif k.endswith(("running_mean", "running_var")):
            bar = 1e-4 if other is None else max(1e-4, 8 * _err(other[k], ref))
            assert _err(got, ref) <= bar, "%s: %.3e (bar %.3e)" % (k, _err(got, ref), bar)
        elif k not in g_off:
            assert torch.equal(got, ref), k
        else:
            g = g_off[k].double()
            tol = STEP_GRAD_TOL if g_other is None else max(STEP_GRAD_TOL, 8 * _err(g_other[k], g))
            eps_g = tol * g.abs().max()
            d = lambda t: t / (t.abs() + 1e-8)  # noqa: E731
            slack = lr * torch.maximum((d(g + eps_g) - d(g)).abs(), (d(g - eps_g) - d(g)).abs())
            if _zero_grad_bias(g_off, k):
                slack = 2 * lr * torch.ones_like(g)
            p0 = before[k].to(DEV).double()
            diff = (got.double() - ref.double()).abs()
            assert bool((diff <= 1e-6 * p0.abs().max() + 2 * lr).all()), k
            firm = g.abs() >= 1e-2 * g.abs().max()
            bad = firm & (diff > 1e-6 * p0.abs().max() + slack)
            assert int(bad.sum()) <= max(4, 1e-4 * g.numel()), k


FULL = [  # tc, activation, k, som_k, surface_normal
    ("default", "relu", 3, 9, True),
    ("default", "elu", 2, 9, False),
    ("default", "relu", 1, 0, True),
    ("default", "elu", 3, 0, True),
    ("fp16", "relu", 3, 9, True),
    ("fp16", "elu", 1, 9, False),
]


@pytest.mark.parametrize("tc,act,k,som_k,sn", FULL)
def test_full_step_equal_sizes_against_dense_optimize(monkeypatch, tc, act, k, som_k, sn):
    B, N, M = 4, 512, 64
    over = dict(k=k, node_num=M, som_k=som_k, activation=act, surface_normal=sn)
    # on a 1/256 grid every cluster sum is exact, so the dense path's cluster means (summed in
    # som_stats_kernel's order) are the group order's bits and both steps see the same inputs
    pts, off, node, knn = _clouds([N] * B, M, max(som_k, 1), seed=k + som_k, grid=256)
    label = torch.tensor([0, 3, 7, 3], dtype=torch.int64, device=DEV)
    dense, st = _model(monkeypatch, tc, B, N, **over)
    pc = pts.view(B, N, 6).permute(0, 2, 1)
    dense.set_input(pc[:, :3].contiguous(), pc[:, 3:].contiguous(), label, node, knn)
    torch.manual_seed(0)
    dense.optimize(epoch=2)
    loss_d, score_d = dense.loss.detach().clone(), dense.score.detach().clone()
    off_state, g_off = _state(dense)
    rag, _ = _model(monkeypatch, tc, B, N, **over)
    torch.manual_seed(0)
    out = rag.optimize_clouds(pts, off, label, node, knn, epoch=2)
    on_state, g_on = _state(rag)
    print("[ragged-train] %s %s k=%d som_k=%d sn=%s: score %.2e, worst gradient %.2e (%s)" % (
        (tc, act, k, som_k, sn, _err(out["score"], score_d))
        + max((_err(g_on[kk], g), kk) for kk, g in g_off.items() if not _zero_grad_bias(g_off, kk))))
    assert _err(out["score"], score_d) <= 1e-4
    assert abs(float(out["loss"]) - float(loss_d)) <= 1e-4 * max(1.0, abs(float(loss_d)))
    _check_grads(g_on, g_off)
    before = {"%d.%s" % (i, kk): v for i, sd in enumerate((st["encoder"], st["head"]))
              for kk, v in sd.items()}
    _check_step(on_state, g_on, off_state, g_off, before, rag.opt.lr)


def _knn_module(knn, coord, x, knn_I, K, center_type, epoch):
    """KNNModule's PyTorch composition (layers.py) up to the max over the K neighbours:
    -> (center [B,3,M], h [B,C,M,K])."""
    from sonet_b200 import operations
    idx = knn_I[:, :, 0:K]
    nb = operations.knn_gather_wrapper(coord, idx)
    ctr = nb.mean(dim=3, keepdim=True) if center_type == "avg" else coord.unsqueeze(3)
    h = torch.cat(((nb - ctr).detach(), operations.knn_gather_by_indexing(x, idx)), dim=1)
    for layer in knn.layers:
        h = layer(h, epoch)
    return ctr.squeeze(3).detach(), h


def _node_stage(enc, som_node, masked_max, knn, epoch, pin=None):
    """forward()'s node-level stage -> (final [B,F,M], arg-max of the max over K or None). With
    pin = (arg-max over K, arg-max over nodes) the two max pools take those elements."""
    opt = enc.opt
    kmax = None
    if opt.som_k >= 2:
        center, h = _knn_module(enc.knnlayer, som_node, masked_max, knn, opt.som_k, opt.som_k_type,
                                epoch)
        kmax = h.argmax(dim=3) if pin is None else pin[0]
        feat = h.gather(3, kmax.unsqueeze(3)).squeeze(3)
        final = enc.final_pointnet.forward_pair(center, feat, epoch)
    else:
        final = enc.final_pointnet(som_node, epoch, x1=masked_max)
    return final, kmax


def _argmax_pins(m, x_aug, idx, cm, off, knn, epoch):
    """The arg-max of each max pool in an fp32 run of the step's forward on the GPU (a deep copy on
    the train kernels): the per-node max (index_max_ragged's cloud-local columns), the max over the
    K neighbours and the max over nodes."""
    enc = copy.deepcopy(m.encoder).train()
    k, M = m.opt.k, cm.shape[2]
    with torch.enable_grad():
        fpo = enc.first_pointnet(x_aug, epoch, cols=off * k)
        col, mm = ops.index_max_ragged(fpo.detach()[0], idx, off, M, k)
        final, kmax = _node_stage(enc, cm, mm, knn, epoch)
    return col.long(), kmax, final.argmax(dim=2)


def _fp64_step(m, pts, off, node, knn, label, epoch, dtype=torch.float64, dev="cpu", pins=None):
    """The train step's loss and gradients in torch `dtype` on the CPU: deep copies of the modules
    (their PyTorch branch), the kernels' assignment and cluster means, BatchNorm over [1,C,k*T] and
    the per-cloud per-node max by gather. Every max pool takes the element an fp32 GPU run of the
    forward picked (_argmax_pins): at these node counts a near-tie that fp32 and fp64 resolve
    differently routes a whole pooled gradient elsewhere, the same in optimize() (measured with
    ReLU, som_k = 9, 16 nodes: 2.5e-2 of the KNN module's weight gradient, dense and ragged alike)."""
    enc, opt = m.encoder, m.opt
    k, M = opt.k, node.shape[2]
    sn = opt.surface_normal == True  # noqa: E712
    with torch.no_grad():
        idx, _, _ = ops.som_assign_ragged(pts, off, node, k)
        _, _, _, cm = ops.som_group_decenter_ragged(pts, off, idx, M, k, sn)
        x_aug = ops.som_decenter_ragged(pts, off, idx, cm, k, sn)
    pins = pins or _argmax_pins(m, x_aug, idx, cm, off, knn, epoch)
    col, kmax, fmax = pins
    e64 = copy.deepcopy(enc).to(dev, dtype).train()
    h64 = copy.deepcopy(m.classifier).to(dev, dtype).train()
    fpo = e64.first_pointnet(x_aug.to(dev, dtype), epoch)[0]          # [C, k*T]
    o = off.to(dev) * k
    C = fpo.shape[0]
    gcol = (o[:-1].view(-1, 1, 1) + col.to(dev)).permute(1, 0, 2).reshape(C, -1)   # [C, B*M]
    masked_max = fpo.gather(1, gcol).view(C, -1, M).permute(1, 0, 2)               # [B, C, M]
    final, _ = _node_stage(e64, cm.to(dev, dtype), masked_max, knn.to(dev), epoch,
                           pin=(None if kmax is None else kmax.to(dev), None))
    feature = final.gather(2, fmax.to(dev).unsqueeze(2)).squeeze(2)
    score = h64(feature, epoch)
    loss = nn.CrossEntropyLoss()(score, label.to(dev))
    loss.backward()
    grads = {"0." + kk: p.grad for kk, p in e64.named_parameters() if p.grad is not None}
    grads.update({"1." + kk: p.grad for kk, p in h64.named_parameters() if p.grad is not None})
    return loss.detach(), score.detach(), grads, pins


@pytest.mark.parametrize("act,som_k,M", [("relu", 9, 16), ("relu", 9, 64), ("elu", 9, 64),
                                         ("elu", 0, 16)])
def test_full_step_mixed_sizes_fp64(monkeypatch, act, som_k, M):
    sizes = [300, 1100, 57, 700, 1025]
    m, _ = _model(monkeypatch, "default", len(sizes), 512, k=3, node_num=M, som_k=som_k,
                  activation=act)
    pts, off, node, knn = _clouds(sizes, M, max(som_k, 1), seed=9)
    label = torch.tensor([1, 0, 4, 1, 9], dtype=torch.int64, device=DEV)
    loss64, score64, g64, pins = _fp64_step(m, pts, off, node, knn, label, 1)
    # test_gpu_train_parity.py's rule against fp64: 8x the error of a strict-fp32 run of the PyTorch
    # composition (the same restatement in fp32 on the GPU, TF32 off; its first layer is cuDNN's
    # convolution over the same k*T columns as the step's)
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    monkeypatch.setattr(train_ops, "ENABLED", False)
    try:
        _, score32, g32, _ = _fp64_step(m, pts, off, node, knn, label, 1, torch.float32, DEV, pins)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
        monkeypatch.setattr(train_ops, "ENABLED", True)
    torch.manual_seed(0)
    out = m.optimize_clouds(pts, off, label, node, knn, epoch=1)
    _, grads = _state(m)
    assert abs(float(out["loss"]) - float(loss64)) <= 1e-4 * max(1.0, abs(float(loss64)))
    assert _err(out["score"].cpu(), score64) <= max(1e-4, 8 * _err(score32.cpu(), score64))
    _check_grads({kk: g.cpu() for kk, g in grads.items()}, g64,
                 {kk: g.cpu() for kk, g in g32.items()})


# ---- 5. run behaviour ------------------------------------------------------------------------------
def test_deterministic(monkeypatch):
    """With PyTorch's deterministic algorithms on (the node-level stage's torch.gather backward is
    an atomic scatter otherwise, in optimize() too), two runs give the same bits."""
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        _deterministic(monkeypatch)
    finally:
        torch.use_deterministic_algorithms(False)


def _deterministic(monkeypatch):
    sizes, M = [333, 1200, 64], 64
    pts, off, node, knn = _clouds(sizes, M, 9, seed=4)
    label = torch.tensor([2, 5, 2], dtype=torch.int64, device=DEV)
    runs = []
    for _ in range(2):
        m, _ = _model(monkeypatch, "default", 3, 512)
        torch.manual_seed(0)
        out = [m.optimize_clouds(pts, off, label, node, knn, epoch=0) for _ in range(2)]
        runs.append((out, _state(m)))
    (o0, (s0, g0)), (o1, (s1, g1)) = runs
    for a, b in zip(o0, o1):
        assert torch.equal(a["loss"], b["loss"]) and torch.equal(a["score"], b["score"])
    assert all(torch.equal(s0[k], s1[k]) for k in s0)
    assert all(torch.equal(g0[k], g1[k]) for k in g0)


def test_interleaves_with_graphed_optimize(monkeypatch):
    """optimize_clouds between graphed optimize() steps re-captures nothing, and the graph's next
    replay equals an eager optimize() from the same state (parameters, running statistics and Adam
    state), to the state-dict bars."""
    B, N, M = 4, 256, 64
    pts, off, node, knn = _clouds([N] * B, M, 9, seed=6)
    label = torch.tensor([1, 2, 3, 4], dtype=torch.int64, device=DEV)
    pc = pts.view(B, N, 6).permute(0, 2, 1)
    rp, ro, rn, rk = _clouds([500, 90, 1300, 256], M, 9, seed=7)

    def bind(m):
        m.set_input(pc[:, :3].contiguous(), pc[:, 3:].contiguous(), label, node, knn)

    g, _ = _model(monkeypatch, "default", B, N)
    g.enable_train_graph(True)
    for _ in range(4):                       # each input set: an eager step, then capture + replay
        bind(g)
        g.optimize(epoch=0)
    graphs = {k: v["graph"] for k, v in g._train_graphs.items()}
    assert len(graphs) == 2 and all(v is not None for v in graphs.values())
    g.optimize_clouds(rp, ro, label, rn, rk, epoch=0)
    torch.cuda.synchronize()
    state, _ = _state(g)
    mods = (g.encoder, g.classifier)
    sds = [copy.deepcopy(mm.state_dict()) for mm in mods]
    osd = [copy.deepcopy(o.state_dict()) for o in g._optim]
    bind(g)
    g.optimize(epoch=0)                      # replays
    torch.cuda.synchronize()
    assert {k: v["graph"] for k, v in g._train_graphs.items()} == graphs
    got, g_got = _state(g)

    e, _ = _model(monkeypatch, "default", B, N)
    e.encoder.load_state_dict(sds[0])
    e.classifier.load_state_dict(sds[1])
    e._optim = e._make_optimizers()
    for o, sd in zip(e._optim, osd):
        o.load_state_dict(sd)
    bind(e)
    e.optimize(epoch=0)
    want, g_want = _state(e)
    _check_grads(g_got, g_want)
    _check_step(got, g_got, want, g_want, state, g.opt.lr)


def test_score_clouds_after_training(monkeypatch):
    sizes, M = [700, 123, 2000], 64
    pts, off, node, knn = _clouds(sizes, M, 9, seed=8)
    label = torch.tensor([0, 1, 2], dtype=torch.int64, device=DEV)
    m, _ = _model(monkeypatch, "default", 3, 512)
    m.encoder.eval()
    m.classifier.eval()
    s0 = m.score_clouds(pts, off, node, knn)
    torch.manual_seed(0)
    m.optimize_clouds(pts, off, label, node, knn, epoch=0)
    m.encoder.eval()
    m.classifier.eval()
    s1 = m.score_clouds(pts, off, node, knn)
    assert not torch.equal(s0, s1)
    fresh, _ = _model(monkeypatch, "default", 3, 512)
    fresh.encoder.load_state_dict(m.encoder.state_dict())
    fresh.classifier.load_state_dict(m.classifier.state_dict())
    fresh.encoder.eval()
    fresh.classifier.eval()
    assert torch.equal(fresh.score_clouds(pts, off, node, knn), s1)


def test_end_to_end_two_classes(monkeypatch):
    """full_batch(train=True) feeds 30 steps on a small seeded synthetic two-class set: spheres and
    cubes of 600 to 3000 points; the loss falls below half its first value."""
    rs = np.random.RandomState(0)
    points, labels, nodes = [], [], []
    for i in range(16):
        P = int(rs.randint(600, 3000))
        if i % 2 == 0:
            v = rs.normal(size=(P, 3))
            v /= np.linalg.norm(v, axis=1, keepdims=True)
            n = v.copy()
        else:
            v = rs.uniform(-1, 1, size=(P, 3))
            ax = rs.randint(0, 3, size=P)
            v[np.arange(P), ax] = np.sign(rs.uniform(-1, 1, size=P))
            n = np.zeros((P, 3))
            n[np.arange(P), ax] = v[np.arange(P), ax]
        points.append(np.concatenate([v, n], 1).astype(np.float32))
        labels.append(i % 2)
        nodes.append(v[rs.choice(P, 64, replace=False)].astype(np.float32))
    ds = augmentation.DeviceDataset(points, labels, nodes, device=DEV)
    m, _ = _model(monkeypatch, "default", 8, 512, classes=2, lr=1e-3, rot_horizontal=True)
    rng = np.random.RandomState(1)
    losses = []
    for step in range(30):
        idx = rng.choice(16, 8, replace=False)
        pts, off, label, som, knn = ds.full_batch(idx, m.opt, train=True, rng=rng, seed=step)
        losses.append(float(m.optimize_clouds(pts, off, label, som, knn, epoch=0)["loss"]))
    assert min(losses[-5:]) < 0.5 * losses[0], losses
