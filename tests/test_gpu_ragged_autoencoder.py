"""-m gpu: whole-cloud reconstruction. The ragged Chamfer kernel (ops.chamfer_ragged, csrc/chamfer.cu)
against the oracle's scan, the numpy restatement of its fixed summation order (chamfer_emu), the dense
entry at equal sizes and per cloud, across cloud boundaries, ties, non-finite inputs and
permutations; and autoencoder.Model.reconstruct_clouds against test_model() at equal sizes, the
reference golden, per-cloud dense Chamfer at mixed sizes, and the model state it must leave alone.
Every check of indices asserts their range before anything gathers with them."""
import math

import numpy as np
import pytest
import torch

import chamfer_emu
from helpers import assert_close, assert_golden, build_states, golden, golden_case
from sonet_b200 import augmentation, autoencoder, ops, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
KEYS = ("loss", "fwd_arr", "bwd_arr", "elem_fwd", "elem_bwd", "idx_fwd", "idx_bwd")


# ---- helpers ----------------------------------------------------------------------------------------
def _pred(rs, B, Mp):
    return torch.from_numpy(rs.uniform(-1, 1, size=(B, 3, Mp)).astype(np.float32)).to(DEV)


def _points(rs, sizes, ld=6):
    pts = rs.uniform(-1, 1, size=(sum(sizes), ld)).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return torch.from_numpy(pts).to(DEV), torch.from_numpy(off).to(DEV)


def _gt(points, off, b):
    o = off.tolist()
    return points[o[b]:o[b + 1], :3].t().contiguous()[None]       # [1,3,P_b]


def _ragged(pred, points, off, want_idx=True):
    r = ops.chamfer_ragged(pred, points, off, want_idx=want_idx)
    return {k: (v.cpu() if v is not None else None) for k, v in r.items()}


def _dense(pred, gt, want_idx=True):
    r = ops.chamfer(pred.contiguous(), gt.contiguous(), want_idx=want_idx)
    return {k: (v.cpu() if v is not None else None) for k, v in r.items()}


def _same(got, want, what):
    """Bit-equal: float32 compared as bit patterns, integers as values."""
    g = got.numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    w = want.numpy() if isinstance(want, torch.Tensor) else np.asarray(want)
    if g.dtype == np.float32:
        g, w = g.view(np.uint32), w.astype(np.float32).view(np.uint32)
    else:
        w = w.astype(g.dtype)
    ok = g == w
    if not ok.all():
        at = tuple(int(x) for x in np.argwhere(~ok)[0])
        raise AssertionError("%s: %d of %d differ, first at %s: got %r want %r"
                             % (what, int((~ok).sum()), ok.size, at, g[at], w[at]))


def _in_range(r, Mp, sizes):
    """idx_fwd of cloud b in [0, P_b), idx_bwd in [0, Mp)."""
    lim = torch.tensor(sizes, dtype=torch.int32)[:, None]
    f, b = r["idx_fwd"], r["idx_bwd"]
    assert bool(((f >= 0) & (f < lim)).all()), "idx_fwd outside its cloud"
    assert bool(((b >= 0) & (b < Mp)).all()), "idx_bwd outside [0, Mp)"


def _per_cloud_equals_dense(r, pred, points, off, what=""):
    """Cloud b's entries of the ragged result equal a dense B = 1 chamfer on that cloud."""
    o = off.tolist()
    for b in range(pred.shape[0]):
        d = _dense(pred[b:b + 1], _gt(points, off, b))
        sl = slice(o[b], o[b + 1])
        _same(r["idx_fwd"][b], d["idx_fwd"][0], "%sidx_fwd[%d]" % (what, b))
        _same(r["idx_bwd"][sl], d["idx_bwd"][0], "%sidx_bwd[%d]" % (what, b))
        _same(r["elem_fwd"][b], d["elem_fwd"][0], "%selem_fwd[%d]" % (what, b))
        _same(r["elem_bwd"][sl], d["elem_bwd"][0], "%selem_bwd[%d]" % (what, b))
        _same(r["fwd_arr"][b:b + 1], d["fwd_arr"], "%sfwd_arr[%d]" % (what, b))
        _same(r["bwd_arr"][b:b + 1], d["bwd_arr"], "%sbwd_arr[%d]" % (what, b))


# ---- 1. equal sizes: the dense entry's bits ---------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3, 300])
@pytest.mark.parametrize("Mp", [1, 127, 128, 129, 1280, 4352])
@pytest.mark.parametrize("N", [1, 255, 256, 257, 1023, 1024, 1025, 4097])
def test_equal_sizes_give_dense_bits(B, Mp, N):
    rs = np.random.RandomState(B * 7 + Mp * 3 + N)
    pred = _pred(rs, B, Mp)
    gt = torch.from_numpy(rs.uniform(-1, 1, size=(B, 3, N)).astype(np.float32)).to(DEV)
    pts = torch.cat([gt.permute(0, 2, 1).reshape(-1, 3),
                     torch.full((B * N, 3), float("nan"), device=DEV)], 1).contiguous()
    off = torch.arange(0, B * N + 1, N, dtype=torch.int64, device=DEV)
    for want_idx in (True, False):
        r, d = _ragged(pred, pts, off, want_idx), _dense(pred, gt, want_idx)
        if want_idx:
            _in_range(r, Mp, [N] * B)
        for k in KEYS:
            if d[k] is None:
                assert r[k] is None
                continue
            want = d[k].reshape(-1) if k in ("idx_bwd", "elem_bwd") else d[k]
            _same(r[k], want, k)


def test_row_stride_and_views():
    """[T,3] rows, [T,6] rows and the xyz view of [T,6] give the same bits."""
    rs = np.random.RandomState(1)
    pred = _pred(rs, 3, 300)
    pts6, off = _points(rs, [700, 1, 2100])
    a = _ragged(pred, pts6, off)
    b = _ragged(pred, pts6[:, :3], off)
    c = _ragged(pred, pts6[:, :3].contiguous(), off)
    for k in KEYS:
        _same(b[k], a[k], "view " + k)
        _same(c[k], a[k], "[T,3] " + k)


# ---- 2. the oracle's scan and the fixed-order sums --------------------------------------------------
@pytest.mark.parametrize("sizes,Mp", [([1, 1025, 300, 2048, 77], 1280), ([5000], 129),
                                      ([3, 1, 4097, 256, 1023], 1)])
def test_matches_oracle_and_restatement(oracle_mod, sizes, Mp):
    rs = np.random.RandomState(len(sizes) + Mp)
    pred = _pred(rs, len(sizes), Mp)
    pts, off = _points(rs, sizes)
    r = _ragged(pred, pts, off)
    _in_range(r, Mp, sizes)
    o = off.tolist()
    for b in range(len(sizes)):
        q = oracle_mod.chamfer(pred[b:b + 1].cpu(), _gt(pts, off, b).cpu())
        sl = slice(o[b], o[b + 1])
        _same(r["idx_fwd"][b], q["idx_fwd"][0].int(), "oracle idx_fwd[%d]" % b)
        _same(r["idx_bwd"][sl], q["idx_bwd"][0].int(), "oracle idx_bwd[%d]" % b)
        _same(r["elem_fwd"][b], oracle_mod.chamfer_elem(q["dist2_fwd"])[0], "oracle elem_fwd")
        _same(r["elem_bwd"][sl], oracle_mod.chamfer_elem(q["dist2_bwd"])[0], "oracle elem_bwd")
    e = chamfer_emu.chamfer_ragged(pred.cpu().numpy(), pts.cpu().numpy(), o)
    for k in ("elem_fwd", "elem_bwd", "fwd_arr", "bwd_arr", "loss"):
        _same(r[k], e[k], "restatement " + k)
    _same(r["idx_fwd"], e["idx_fwd"].astype(np.int32), "restatement idx_fwd")
    _same(r["idx_bwd"], e["idx_bwd"].astype(np.int32), "restatement idx_bwd")
    # the kernel's means against fp64 sums of its own terms
    for arr, el, P in (("fwd_arr", lambda b: r["elem_fwd"][b], lambda b: Mp),
                       ("bwd_arr", lambda b: r["elem_bwd"][o[b]:o[b + 1]], lambda b: sizes[b])):
        for b in range(len(sizes)):
            want = el(b).double().mean().item()
            err = abs(float(r[arr][b]) - want)
            assert err <= (math.ceil(P(b) / 1024) + 12) * U * want, (arr, b, err / want / U)
    B = len(sizes)
    for j, arr in ((0, "fwd_arr"), (1, "bwd_arr")):
        want = r[arr].double().mean().item()
        assert abs(float(r["loss"][j]) - want) <= (math.ceil(B / 256) + 10) * U * want


# ---- 3. mixed sizes, cloud boundaries ---------------------------------------------------------------
def test_mixed_sizes_match_each_cloud_alone():
    rs = np.random.RandomState(4)
    sizes = [2000 + int(x) for x in rs.randint(0, 8000, size=37)] + [1, 1024, 1025, 256]
    Mp = 1280
    pred = _pred(rs, len(sizes), Mp)
    pts, off = _points(rs, sizes)
    r = _ragged(pred, pts, off)
    _in_range(r, Mp, sizes)
    _per_cloud_equals_dense(r, pred, pts, off)


def test_cloud_boundaries_are_never_crossed():
    """A 1-point cloud between clouds of 1,025 and 2^20 points (none a multiple of 1024 after the
    first column tile, so a flat tiling would straddle them). Each cloud's predictions sit exactly
    on the first points of the NEXT cloud, which are closer than anything in their own cloud: they
    are never chosen."""
    rs = np.random.RandomState(5)
    sizes = [1025, 1, (1 << 20) + 3, 700]
    Mp = 300
    pts, off = _points(rs, sizes)
    o = off.tolist()
    pred = _pred(rs, len(sizes), Mp)
    for b in range(len(sizes)):
        pts[o[b]:o[b + 1], 0] += 10.0 * b                           # clouds 10 apart along x
    pred[-1, 0] += 10.0 * (len(sizes) - 1)
    for b in range(len(sizes) - 1):                                 # on cloud b+1's points
        nxt = pts[o[b + 1]:o[b + 1] + min(Mp, sizes[b + 1]), :3].t()
        pred[b, :, :nxt.shape[1]] = nxt
    r = _ragged(pred, pts, off)
    _in_range(r, Mp, sizes)
    _per_cloud_equals_dense(r, pred, pts, off)


def test_ties_across_tiles_resolve_to_the_lowest_index(oracle_mod):
    """Inside the second cloud of a ragged batch: duplicate gt points on both sides of its
    1024-column tiles and duplicate predictions on both sides of the 128-row tiles."""
    rs = np.random.RandomState(6)
    sizes = [77, 2100, 300]
    Mp = 300
    pts, off = _points(rs, sizes)
    o = off.tolist()
    pred = _pred(rs, len(sizes), Mp)
    g = pts[o[1]:o[2], :3]
    lo = torch.from_numpy(np.r_[1004:1024, 1050:1070, 0]).to(DEV)
    hi = torch.from_numpy(np.r_[1024:1044, 2048:2068, 2099]).to(DEV)
    g[hi] = g[lo]
    pred[1, :, :41] = g[lo].t()
    pred[1, :, 41:82] = g[lo].t() + 1e-3
    plo = torch.from_numpy(np.r_[100:128, 90:100]).to(DEV)
    phi = torch.from_numpy(np.r_[128:156, 260:270]).to(DEV)
    pred[1, :, phi] = pred[1, :, plo]
    g[200:238] = pred[1, :, plo].t()
    r = _ragged(pred, pts, off)
    _in_range(r, Mp, sizes)
    want = lo.int().cpu()
    assert torch.equal(r["idx_fwd"][1, :41], want)
    assert torch.equal(r["idx_fwd"][1, 41:82], want)
    assert bool((r["idx_bwd"][o[1] + 200:o[1] + 238] < 128).all())
    q = oracle_mod.chamfer(pred[1:2].cpu(), _gt(pts, off, 1).cpu())
    _same(r["idx_fwd"][1], q["idx_fwd"][0].int(), "oracle idx_fwd")
    _same(r["idx_bwd"][o[1]:o[2]], q["idx_bwd"][0].int(), "oracle idx_bwd")


@pytest.mark.parametrize("where", ["gt_nan", "gt_overflow", "pred_nan", "gt_all_nan"])
def test_non_finite_inputs_stay_in_their_cloud(oracle_mod, where):
    rs = np.random.RandomState(7)
    sizes = [400, 1500, 90]
    Mp = 200
    pts, off = _points(rs, sizes)
    o = off.tolist()
    pred = _pred(rs, len(sizes), Mp)
    clean = _ragged(pred, pts, off)
    pts2, pred2 = pts.clone(), pred.clone()
    if where == "gt_nan":
        pts2[o[1] + 17, 1] = float("nan")
    elif where == "gt_overflow":
        pts2[o[1] + 1100, :3] = 3e38
        pred2[1, :, 5] = -3e38
    elif where == "pred_nan":
        pred2[1, 2, 150] = float("nan")
    else:
        pts2[o[1]:o[2], 0] = float("nan")
    r = _ragged(pred2, pts2, off)
    _in_range(r, Mp, sizes)
    for b in (0, 2):                                          # other clouds: unchanged bits
        sl = slice(o[b], o[b + 1])
        for k in ("idx_fwd", "elem_fwd"):
            _same(r[k][b], clean[k][b], "%s[%d]" % (k, b))
        for k in ("idx_bwd", "elem_bwd"):
            _same(r[k][sl], clean[k][sl], "%s[%d]" % (k, b))
        for k in ("fwd_arr", "bwd_arr"):
            _same(r[k][b:b + 1], clean[k][b:b + 1], "%s[%d]" % (k, b))
    _per_cloud_equals_dense(r, pred2, pts2, off)             # the dense non-finite rule
    q = oracle_mod.chamfer(pred2[1:2].cpu(), _gt(pts2, off, 1).cpu())
    _same(r["idx_fwd"][1], q["idx_fwd"][0].int(), "oracle idx_fwd")
    _same(r["idx_bwd"][o[1]:o[2]], q["idx_bwd"][0].int(), "oracle idx_bwd")


def test_permuting_clouds_permutes_every_bit():
    rs = np.random.RandomState(8)
    sizes = [1, 3000, 1024, 517, 4097, 2]
    Mp = 1280
    pred = _pred(rs, len(sizes), Mp)
    pts, off = _points(rs, sizes)
    r = _ragged(pred, pts, off)
    perm = [4, 0, 5, 2, 1, 3]
    o = off.tolist()
    pts_p = torch.cat([pts[o[b]:o[b + 1]] for b in perm])
    sizes_p = [sizes[b] for b in perm]
    off_p = torch.tensor(np.concatenate([[0], np.cumsum(sizes_p)]), dtype=torch.int64, device=DEV)
    s = _ragged(pred[perm], pts_p, off_p)
    op = off_p.tolist()
    for i, b in enumerate(perm):
        for k in ("idx_fwd", "elem_fwd", "fwd_arr", "bwd_arr"):
            _same(s[k][i], r[k][b], "%s[%d]" % (k, b))
        for k in ("idx_bwd", "elem_bwd"):
            _same(s[k][op[i]:op[i + 1]], r[k][o[b]:o[b + 1]], "%s[%d]" % (k, b))


# ---- 4. the auto-encoder ----------------------------------------------------------------------------
def _ae(monkeypatch, tc="1", B=2, N=256, seed=3, **over):
    monkeypatch.setenv("SONET_TC", tc)
    opt = synth.make_opt("autoencoder", batch_size=B, input_pc_num=N, **over)
    st = build_states("autoencoder", opt, seed)
    opt.device, opt.gpu_id = torch.device(DEV), 0
    m = autoencoder.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.decoder.load_state_dict(st["head"])
    m.encoder.eval()
    m.decoder.eval()
    return m


def _as_ragged(pc, sn):
    B, _, N = pc.shape
    pts = torch.cat((pc, sn), dim=1).permute(0, 2, 1).reshape(-1, 6).contiguous().to(DEV)
    return pts, torch.arange(0, B * N + 1, N, dtype=torch.int64, device=DEV)


def _eq(a, b, what):
    assert (a is None) == (b is None), what
    if a is not None:
        assert torch.equal(a, b), what


AE_EQUAL = [(tc, act, fc, conv, som_k)
            for tc in ("1", "fp16") for act in ("relu", "elu")
            for fc, conv in ((256, 1024), (0, 4096), (256, 0)) for som_k in (0, 9)]


@pytest.mark.parametrize("tc,act,fc,conv,som_k", AE_EQUAL)
def test_equal_sizes_give_test_model_bits(monkeypatch, tc, act, fc, conv, som_k):
    B, N, M = 3, 512, 64
    m = _ae(monkeypatch, tc, B=B, N=N, activation=act, output_fc_pc_num=fc,
            output_conv_pc_num=conv, som_k=som_k)
    inp = synth.synth_inputs(B, N, M, max(som_k, 1), seed=som_k + fc + conv)
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    m.test_model()
    pts, off = _as_ragged(inp["pc"], inp["sn"])
    r = m.reconstruct_clouds(pts, off, inp["node"].to(DEV), inp["node_knn_I"].to(DEV))
    _eq(r["feature"], m.feature, "feature")
    _eq(r["predicted_pc"], m.predicted_pc, "predicted_pc")
    _eq(r["loss_chamfer"], m.loss_chamfer, "loss_chamfer")
    _eq(r["loss_chamfer_conv4"], getattr(m, "loss_chamfer_conv4", None) if conv else None, "conv4")
    _eq(r["loss_chamfer_conv5"], getattr(m, "loss_chamfer_conv5", None) if conv == 4096 else None,
        "conv5")
    _eq(r["loss"], m.loss, "loss")
    _eq(r["loss_array"], m.chamfer_criteria.loss_array, "loss_array")


def test_golden_clouds_as_ragged_set():
    g = golden("autoencoder_b2_n256")
    opt, inp, seed = golden_case(g, "autoencoder")
    st = build_states("autoencoder", opt, seed)
    opt.device, opt.gpu_id = torch.device(DEV), 0
    m = autoencoder.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.decoder.load_state_dict(st["head"])
    m.encoder.eval()
    m.decoder.eval()
    pts, off = _as_ragged(inp["pc"], inp["sn"])
    r = m.reconstruct_clouds(pts, off, inp["node"].to(DEV), inp["node_knn_I"].to(DEV))
    assert_golden(g, "predicted_pc", r["predicted_pc"])
    assert_close(r["loss_chamfer"], g["loss_chamfer"], "loss_chamfer")
    assert_close(r["loss_chamfer_conv4"], g["loss_chamfer_conv4"], "loss_chamfer_conv4")
    assert_close(r["loss"], g["loss"], "loss")
    assert_close(r["loss_array"], g["loss_array"], "loss_array")


def _clouds(sizes, M, som_k, seed):
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


@pytest.mark.parametrize("fc,conv", [(256, 1024), (0, 4096)])
def test_mixed_sizes_per_cloud_and_invariance(monkeypatch, fc, conv):
    sizes = [3000, 17, 1025, 8000, 640]
    m = _ae(monkeypatch, "1", B=len(sizes), N=256, output_fc_pc_num=fc, output_conv_pc_num=conv)
    pts, off, node, knn = _clouds(sizes, 64, 9, seed=11)
    r = m.reconstruct_clouds(pts, off, node, knn)
    o = off.tolist()
    with torch.no_grad():
        parts = m.decoder.outputs(r["feature"])[1]
    terms = [("loss_chamfer", r["predicted_pc"]), ("loss_chamfer_conv4", parts["conv_pc4"])]
    if conv == 4096:
        terms.append(("loss_chamfer_conv5", parts["conv_pc5"]))
    for b in range(len(sizes)):
        gt = pts[o[b]:o[b + 1], :3].t().contiguous()[None]
        d = ops.chamfer(r["predicted_pc"][b:b + 1].contiguous(), gt)
        assert torch.equal(r["loss_array"][b:b + 1], d["fwd_arr"] + d["bwd_arr"]), b
    for name, pc in terms:                                       # the batch term, cloud by cloud
        arr = []
        for b in range(len(sizes)):
            gt = pts[o[b]:o[b + 1], :3].t().contiguous()[None]
            d = ops.chamfer(pc[b:b + 1].contiguous(), gt)
            arr.append(d["fwd_arr"] + d["bwd_arr"])
        want = ops.chamfer_ragged(pc.contiguous(), pts, off)["loss"][2]
        assert torch.equal(r[name], want), name
        mean = float(torch.cat(arr).double().mean())
        assert abs(float(r[name]) - mean) <= 1e-5 * mean, name
    # permuting the clouds and chunking change no bit
    perm = [3, 0, 4, 2, 1]
    pts_p = torch.cat([pts[o[b]:o[b + 1]] for b in perm])
    off_p = torch.tensor(np.concatenate([[0], np.cumsum([sizes[b] for b in perm])]),
                         dtype=torch.int64, device=DEV)
    s = m.reconstruct_clouds(pts_p, off_p, node[perm], knn[perm])
    for k in ("feature", "predicted_pc", "loss_array"):
        assert torch.equal(s[k], r[k][perm]), k
    for chunk in (1, 1000, 9000):
        c = m.reconstruct_clouds(pts, off, node, knn, chunk_points=chunk)
        for k, v in r.items():
            _eq(c[k], v, "chunk %d %s" % (chunk, k))


def test_model_and_graph_state_untouched(monkeypatch):
    B, N, M = 3, 512, 64
    m = _ae(monkeypatch, "1", B=B, N=N)
    m.enable_cuda_graph(True)
    inp = synth.synth_inputs(B, N, M, 9, seed=21)
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    m.test_model()
    names = ("feature", "predicted_pc", "loss_chamfer", "loss_chamfer_conv4", "loss")
    dec_names = ("linear_pc", "conv_pc4", "conv_pc5", "conv_pc6")
    cc_names = ("forward_loss", "backward_loss", "forward_loss_array", "backward_loss_array",
                "loss_array")
    cd_names = ("pc4", "pc5", "pc6")

    def snap():
        return ({n: getattr(m, n) for n in names}, {n: getattr(m.decoder, n) for n in dec_names},
                {n: getattr(m.chamfer_criteria, n) for n in cc_names},
                {n: getattr(m.decoder.conv_decoder, n) for n in cd_names})
    ref = snap()
    vals = [{n: t.clone() for n, t in d.items()} for d in ref]
    pts, off, node, knn = _clouds([900, 3000, 12], M, 9, seed=5)
    m.reconstruct_clouds(pts, off, node)                   # node_knn_I computed
    after = snap()
    for d0, d1, v in zip(ref, after, vals):
        for n in d0:
            assert d1[n] is d0[n], "attribute %s rebound" % n
            assert torch.equal(d1[n], v[n]), "attribute %s changed" % n
    m.test_model()                                         # graph replay
    for d1, v in zip(snap(), vals):
        for n in d1:
            assert torch.equal(d1[n], v[n]), "replay: %s" % n
