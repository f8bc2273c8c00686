"""Segmenter scores of every point of each shape (segmenter.Model.score_points) and the
full-resolution IoU (losses.compute_iou_full) on the GPU: consistency with the sampled forward,
a float64 restatement of the reference's per-point path, chunk and row independence, and the ragged
IoU kernel against its host twin and numpy."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import build_states
from sonet_b200 import losses, ops, segmenter, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _model(monkeypatch, tc="1", k=3, activation="relu", surface_normal=True, B=3, N=256, seed=5):
    monkeypatch.setenv("SONET_TC", tc)
    opt = synth.make_opt("segmenter", batch_size=B, input_pc_num=N, k=k, activation=activation,
                         surface_normal=surface_normal)
    st = build_states("segmenter", opt, seed)
    opt.device, opt.gpu_id = torch.device(DEV), 0
    m = segmenter.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.segmenter.load_state_dict(st["head"])
    return m, st


def _ragged(sizes, seed):
    """Clouds of the given sizes: points U(-1,1)^3 with unit normals, [sum P, 6]."""
    rs = np.random.RandomState(seed)
    clouds = []
    for P in sizes:
        xyz = rs.uniform(-1, 1, size=(P, 3)).astype(np.float32)
        n = rs.normal(size=(P, 3))
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        clouds.append(np.concatenate([xyz, n.astype(np.float32)], axis=1))
    return clouds


def _batch_from(clouds, N, M, seed):
    """The sampled batch of the clouds: N points each (with repeats when P < N), M loader nodes."""
    rs = np.random.RandomState(seed)
    pc, sn, node = [], [], []
    for c in clouds:
        sel = rs.choice(len(c), N, replace=len(c) < N)
        pc.append(c[sel, :3].T)
        sn.append(c[sel, 3:].T)
        nsel = rs.choice(len(c), M, replace=len(c) < M)
        node.append(c[nsel, :3].T + rs.normal(0, 1e-3, size=(3, M)).astype(np.float32))
    pc, sn = np.stack(pc).astype(np.float32), np.stack(sn).astype(np.float32)
    node = np.ascontiguousarray(np.stack(node), dtype=np.float32)
    d = ((node[:, :, :, None].astype(np.float64) - node[:, :, None, :]) ** 2).sum(axis=1)
    knn = np.argsort(d, axis=2, kind="stable")[:, :, :9].astype(np.int64)
    label = rs.randint(0, 16, size=len(clouds)).astype(np.int64)
    seg = np.zeros((len(clouds), N), dtype=np.int64)
    return [torch.from_numpy(a) for a in (pc, sn, label, seg, node, knn)]


def _run(m, batch):
    m.set_input(*batch)
    m.test_model()


def _sampled_as_ragged(m):
    pts = torch.cat((m.input_pc, m.input_sn), dim=1).permute(0, 2, 1).reshape(-1, 6).contiguous()
    B, N = m.input_pc.shape[0], m.input_pc.shape[2]
    return pts, torch.arange(0, B * N + 1, N, dtype=torch.int64, device=DEV)


# ---- 1. the sampled batch itself gives the sampled forward's scores --------------------------------
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("tc", ["0", "1", "fp16"])
@pytest.mark.parametrize("activation", ["relu", "elu"])
@pytest.mark.parametrize("surface_normal", [True, False])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_consistent_with_sampled_forward(monkeypatch, fused, tc, activation, surface_normal, k):
    # every route here is the same in both calls: pt / x_aug are the sampled forward's bits, the
    # first PointResNet and every head layer take the same kernel for k*rows >= 256 columns, and a
    # column's result does not depend on the other columns of its launch
    m, _ = _model(monkeypatch, tc=tc, k=k, activation=activation, surface_normal=surface_normal)
    m.encoder.fuse_pool = fused
    clouds = _ragged([300, 500, 256], seed=k)
    _run(m, _batch_from(clouds, 256, 64, seed=k))
    if fused:   # the fused-pool encoder route, reading first_pn_out lazily once
        m.encoder._fpo_demand = False
        m.test_model()
    pts, off = _sampled_as_ragged(m)
    got = m.score_points(pts, off)
    want = m.score_segmenter.permute(0, 2, 1).reshape(-1, m.opt.classes)
    assert torch.equal(got, want), float((got - want).abs().max())


# ---- 2. full ragged clouds against a float64 restatement ------------------------------------------
def _layer(x, st, name, act):
    y = torch.einsum("oc,cp->op", st[name + ".conv.weight"].double().squeeze(-1), x) \
        + st[name + ".conv.bias"].double()[:, None]
    if name + ".norm.weight" in st:
        g, b = st[name + ".norm.weight"].double(), st[name + ".norm.bias"].double()
        mu, var = st[name + ".norm.running_mean"].double(), st[name + ".norm.running_var"].double()
        y = (y - mu[:, None]) / torch.sqrt(var[:, None] + 1e-5) * g[:, None] + b[:, None]
        y = F.relu(y) if act == "relu" else F.elu(y)
    return y


def _oracle_cloud(st_e, st_h, opt, pts, node, cm, nfirst, nknn, nfinal, feature, label):
    """models/segmenter.py:90-98 + networks.py:259-341 for the points of one cloud, in float64:
    k nearest loader nodes (fp32 distances in the reference's order, lowest index on ties), the
    3356-channel concat from the sampled forward's node features, layers 1-5, the k-copy mean."""
    k, act = opt.k, opt.activation
    p32 = pts[:, :3]
    d = [(p32[:, c:c + 1] - node[c][None, :]).astype(np.float32) for c in range(3)]
    dist = (d[0] * d[0] + d[1] * d[1]).astype(np.float32) + d[2] * d[2]
    idx = np.argsort(dist.astype(np.float32), axis=1, kind="stable")[:, :k]     # [P, k]
    P = len(pts)
    outs = []
    x = torch.from_numpy(pts[:, :3].T).double()
    sn = torch.from_numpy(pts[:, 3:].T).double()
    onehot = torch.zeros(16, P, dtype=torch.float64)
    onehot[label] = 1
    for s in range(k):
        ids = torch.from_numpy(idx[:, s])
        ctr = cm[:, ids]
        xdec = (x.float() - ctr.float()).double()      # the fp32 subtraction of the encoder
        xin = torch.cat((xdec, sn)) if opt.surface_normal else xdec
        l0 = _layer(xin, st_e, "first_pointnet.layers.0", act)
        t = _layer(_layer(l0, st_e, "first_pointnet.layers.1", act), st_e,
                   "first_pointnet.layers.2", act)
        fpo = _layer(torch.cat((l0, t)), st_e, "first_pointnet.layers.3", act)
        parts = [xdec, x, ctr] + ([sn] if opt.surface_normal else []) + [onehot, fpo]
        parts += [nfirst[:, ids], nknn[:, ids], nfinal[:, ids], feature[:, None].expand(-1, P)]
        h = torch.cat(parts)
        for name in ("layer1", "layer2", "layer3"):
            h = _layer(h, st_h, name, act)
        outs.append(h)
    avg = outs[0] if k == 1 else (0.5 * (outs[0] + outs[1]) if k == 2
                                  else (1.0 / 3.0) * (outs[0] + outs[1] + outs[2]))
    return _layer(_layer(avg, st_h, "layer4", act), st_h, "layer5", act).t()


@pytest.mark.parametrize("k", [1, 2, 3])
def test_full_clouds_against_fp64(monkeypatch, k):
    sizes = [1, 200, 3001, 777]          # fewer points than N, and sizes off every tile
    m, st = _model(monkeypatch, k=k, B=len(sizes), seed=11 + k)
    clouds = _ragged(sizes, seed=20 + k)
    _run(m, _batch_from(clouds, 256, 64, seed=30 + k))
    pts = torch.from_numpy(np.concatenate(clouds)).to(DEV)
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device=DEV)
    got = m.score_points(pts, off).double().cpu()
    enc = m.encoder
    dd = lambda t: t.detach().double().cpu()  # noqa: E731
    node, cm = m.input_node.cpu().numpy(), dd(enc.som_node)
    for b, c in enumerate(clouds):
        ref = _oracle_cloud(st["encoder"], st["head"], m.opt, c, node[b], cm[b],
                            dd(enc.first_pn_out_masked_max[b]), dd(enc.knn_feature_1[b]),
                            dd(enc.final_pn_out[b]), dd(m.feature[b]), int(m.input_label[b]))
        g = got[int(off[b]):int(off[b + 1])]
        err = float(((g - ref).abs() / ref.abs().clamp(min=1)).max())
        assert err <= 1e-4, "cloud %d (%d points): rel err %.3e" % (b, len(c), err)


# ---- 3. chunking and 4. row independence ----------------------------------------------------------
def test_chunk_and_row_independence(monkeypatch):
    sizes = [1, 2999, 130, 2048]
    m, _ = _model(monkeypatch, B=len(sizes), seed=3)
    clouds = _ragged(sizes, seed=4)
    _run(m, _batch_from(clouds, 256, 64, seed=5))
    pts = torch.from_numpy(np.concatenate(clouds)).to(DEV)
    offs = np.concatenate([[0], np.cumsum(sizes)])
    off = torch.tensor(offs, dtype=torch.int64, device=DEV)
    ref = m.score_points(pts, off, chunk_rows=pts.shape[0])
    for chunk in (128, 300, 2999, None):      # one tile, a tile remainder, one cloud, default
        assert torch.equal(m.score_points(pts, off, chunk_rows=chunk), ref), chunk

    # points shuffled inside their clouds, cloud 1 given its points twice: the same rows' scores
    rs = np.random.RandomState(9)
    perm = [rs.permutation(P) for P in sizes]
    new = [c[p] for c, p in zip(clouds, perm)]
    new[1] = np.concatenate([new[1], new[1]])
    ref_rows = [ref[offs[b]:offs[b + 1]][torch.from_numpy(perm[b]).to(DEV)] for b in range(4)]
    ref_rows[1] = torch.cat([ref_rows[1], ref_rows[1]])
    noff = np.concatenate([[0], np.cumsum([len(c) for c in new])])
    got = m.score_points(torch.from_numpy(np.concatenate(new)).to(DEV),
                         torch.tensor(noff, dtype=torch.int64, device=DEV), chunk_rows=512)
    assert torch.equal(got, torch.cat(ref_rows))

    # cloud 2's points replaced: every other cloud's rows keep their bits
    new = list(clouds)
    new[2] = _ragged([77], seed=99)[0]
    noff = np.concatenate([[0], np.cumsum([len(c) for c in new])])
    got = m.score_points(torch.from_numpy(np.concatenate(new)).to(DEV),
                         torch.tensor(noff, dtype=torch.int64, device=DEV))
    for b in (0, 1, 3):
        assert torch.equal(got[noff[b]:noff[b + 1]], ref[offs[b]:offs[b + 1]]), b


# ---- 5. full-resolution IoU ----------------------------------------------------------------------
def _ref_iou(score, seg, label, offsets):
    out = []
    for b in range(len(label)):
        pred = np.argmax(score[offsets[b]:offsets[b + 1]], axis=1)
        gt = seg[offsets[b]:offsets[b + 1]]
        ious = []
        for p in ops.SHAPENET_PART_TABLE[label[b]]:
            i, u = np.sum((pred == p) & (gt == p)), np.sum((pred == p) | (gt == p))
            ious.append(1.0 if u == 0 else i / float(u + 0.0001))
        out.append(np.mean(ious))
    return np.asarray(out)


def test_compute_iou_full_device_host_numpy(monkeypatch):
    sizes = [1, 200, 3001, 777]
    m, _ = _model(monkeypatch, B=len(sizes), seed=8)
    clouds = _ragged(sizes, seed=8)
    _run(m, _batch_from(clouds, 256, 64, seed=8))
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device=DEV)
    score = m.score_points(torch.from_numpy(np.concatenate(clouds)).to(DEV), off)
    label = m.input_label.to(DEV)
    sc = score.cpu().numpy()
    offs = off.cpu().numpy()
    rs = np.random.RandomState(1)
    seg = np.empty(len(sc), dtype=np.int64)
    for b in range(len(sizes)):
        parts = ops.SHAPENET_PART_TABLE[int(label[b])]
        seg[offs[b]:offs[b + 1]] = rs.choice(parts, size=sizes[b])
    # shape 3: its first part absent from both prediction and ground truth
    parts = ops.SHAPENET_PART_TABLE[int(label[3])]
    sl = slice(offs[3], offs[4])
    seg[sl] = rs.choice(parts[1:] if len(parts) > 1 else parts, size=sizes[3])
    sc[sl, parts[0]] = -1e30
    score = torch.from_numpy(sc).to(DEV)
    segt = torch.from_numpy(seg)
    dev = losses.compute_iou_full(score, segt.to(DEV), label, off)
    host = losses.compute_iou_full(score.cpu(), segt, label.cpu(), off.cpu())
    np.testing.assert_array_equal(dev, host)
    np.testing.assert_array_equal(dev, _ref_iou(sc, seg, label.cpu().numpy(), offs))
