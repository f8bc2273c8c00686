"""-m gpu: the Chamfer kernel (csrc/chamfer.cu) across its tile envelope, at scale extremes, on ties
across tile boundaries and on non-finite inputs, against plain references:

  the oracle's brute-force scan (oracle_c.c: oracle_nn_search), the same fp32 arithmetic as the
      kernel, so nearest-neighbour indices and the per-point terms sqrt(d + 1e-8) are compared
      bit for bit;
  fp64 distances, independent of that arithmetic: the selected pair is within fp32 rounding of
      the true nearest neighbour;
  fp64 sums of the kernel's own per-point terms for the per-cloud means and the losses;
  fp64 autograd of the reference's gather formulation for the training path's gradients.

Kernel geometry: a CTA covers CH_TM = 128 pred rows (grid.y) and 4 warps x 256 = 1024 gt columns
(grid.x); the last column CTA runs ceil((N mod 1024) / 256) live warps. Every check of indices
asserts their range first, before anything gathers with them."""
import math

import numpy as np
import pytest
import torch

from helpers import assert_close

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24          # unit roundoff of fp32
EPS = float(np.float32(1e-8))


# ---- inputs ------------------------------------------------------------------------------------------
def _cloud(rs, B, P, scale=1.0, offset=0.0):
    return torch.from_numpy((rs.uniform(-1, 1, size=(B, 3, P)) * scale + offset).astype(np.float32))


def _chamfer(pred, gt, want_idx=True):
    from sonet_b200 import ops
    r = ops.chamfer(pred.contiguous().to(DEV), gt.contiguous().to(DEV), want_idx=want_idx)
    return {k: (v.cpu() if v is not None else None) for k, v in r.items()}


# ---- checks ------------------------------------------------------------------------------------------
def _assert_idx_in_range(r, Mp, N):
    for k, n in (("idx_fwd", N), ("idx_bwd", Mp)):
        i = r[k]
        bad = (i < 0) | (i >= n)
        assert not bool(bad.any()), "%s: %d indices outside [0, %d), e.g. %d at %s" % (
            k, int(bad.sum()), n, int(i[bad][0]), tuple(int(x) for x in bad.nonzero()[0]))


def _assert_same_idx(got, want, what):
    got = got.long()
    diff = got != want
    assert not bool(diff.any()), "%s: %d of %d differ, first at %s: got %d want %d" % (
        what, int(diff.sum()), diff.numel(), tuple(int(x) for x in diff.nonzero()[0]),
        int(got[diff][0]), int(want[diff][0]))


def _assert_same_floats(got, want, what):
    """Bit-equal as values: NaN where the other is NaN, the same number everywhere else."""
    g, w = got.numpy(), want.numpy()
    ok = (g == w) | (np.isnan(g) & np.isnan(w))
    if not ok.all():
        at = tuple(int(x) for x in np.argwhere(~ok)[0])
        raise AssertionError("%s: %d of %d differ, first at %s: got %r want %r" % (
            what, int((~ok).sum()), ok.size, at, float(g[at]), float(w[at])))


def _assert_sums(r):
    """Per-cloud means and the three losses of the kernel against fp64 sums of its own per-point
    terms. All terms are positive, so a fixed-order fp32 sum is within (additions on the longest
    path + 1 for the division) * U of the exact mean, relatively: chamfer_cloud_kernel adds
    ceil(P/1024) terms per thread, then two 32-term trees; chamfer_final_kernel ceil(B/256) per
    thread, then a 256-term tree."""
    for e, arr in (("elem_fwd", "fwd_arr"), ("elem_bwd", "bwd_arr")):
        P = r[e].shape[1]
        want = r[e].double().mean(1)
        bound = (math.ceil(P / 1024) + 12) * U * want
        err = (r[arr].double() - want).abs()
        assert bool((err <= bound).all()), "%s: rel err %.3g U" % (arr, float((err / want).max() / U))
    B = r["fwd_arr"].shape[0]
    for j, arr in ((0, "fwd_arr"), (1, "bwd_arr")):
        want = float(r[arr].double().mean())
        err = abs(float(r["loss"][j]) - want)
        assert err <= (math.ceil(B / 256) + 10) * U * want, "loss[%d]: rel err %.3g U" % (j, err / want / U)
    assert float(r["loss"][2]) == float(np.float32(float(r["loss"][0])) + np.float32(float(r["loss"][1])))


def _check_vs_oracle(oracle_mod, pred, gt, sums=True):
    """ops.chamfer with indices against the oracle: indices in range, then equal; per-point terms
    bit for bit; the value-only path's terms equal the index path's. -> (kernel, oracle) dicts."""
    Mp, N = pred.shape[2], gt.shape[2]
    r = _chamfer(pred, gt)
    _assert_idx_in_range(r, Mp, N)
    o = oracle_mod.chamfer(pred, gt)
    _assert_same_idx(r["idx_fwd"], o["idx_fwd"], "idx_fwd")
    _assert_same_idx(r["idx_bwd"], o["idx_bwd"], "idx_bwd")
    _assert_same_floats(r["elem_fwd"], oracle_mod.chamfer_elem(o["dist2_fwd"]), "elem_fwd")
    _assert_same_floats(r["elem_bwd"], oracle_mod.chamfer_elem(o["dist2_bwd"]), "elem_bwd")
    v = _chamfer(pred, gt, want_idx=False)
    for k in ("elem_fwd", "elem_bwd", "fwd_arr", "bwd_arr", "loss"):
        _assert_same_floats(v[k], r[k], "value-only " + k)
    if sums:
        _assert_sums(r)
    return r, o


# ---- tile envelope -----------------------------------------------------------------------------------
# every N with a pred count <= 33 and one >= 127, every Mp with an N <= 257 and one >= 1024
ENVELOPE = [
    (1, 1280, 1), (3, 33, 1),
    (3, 31, 200), (3, 127, 200), (1, 129, 200), (1, 300, 200),
    (3, 1280, 256), (1, 33, 256),
    (3, 128, 257), (1, 1, 257),
    (1, 129, 1024), (3, 33, 1024),
    (3, 300, 1025), (1, 31, 1025),          # last CTA: one live warp, one column
    (1, 1280, 1324), (3, 1, 1324),          # two live warps
    (3, 129, 2648), (1, 1, 2648),           # three live warps
    (1, 127, 3072), (3, 31, 3072),
    (3, 128, 5000), (1, 1, 5000), (1, 300, 5000),
]


@pytest.mark.parametrize("B,Mp,N", ENVELOPE)
def test_chamfer_tile_envelope_vs_oracle(oracle_mod, B, Mp, N):
    rs = np.random.RandomState(7 * Mp + N + B)
    _check_vs_oracle(oracle_mod, _cloud(rs, B, Mp), _cloud(rs, B, N))


@pytest.mark.parametrize("B,Mp,N", [(2, 1025, 300), (3, 129, 2648), (1, 1, 5000), (2, 1280, 1324)])
def test_chamfer_symmetry(B, Mp, N):
    """chamfer(a, b) and chamfer(b, a) swap every output bit for bit ((p-g)^2 == (g-p)^2 in fp32):
    the row path (warp reduction + shared atomics) against the column path (registers)."""
    rs = np.random.RandomState(Mp * 3 + N)
    a, b = _cloud(rs, B, Mp), _cloud(rs, B, N)
    r, s = _chamfer(a, b), _chamfer(b, a)
    _assert_idx_in_range(r, Mp, N)
    _assert_idx_in_range(s, N, Mp)
    for x, y in (("elem_fwd", "elem_bwd"), ("idx_fwd", "idx_bwd"), ("fwd_arr", "bwd_arr")):
        assert torch.equal(r[x], s[y]), x
        assert torch.equal(r[y], s[x]), y
    assert torch.equal(r["loss"][[1, 0, 2]], s["loss"])


# ---- fp64 reference -----------------------------------------------------------------------------------
@pytest.mark.parametrize("scale,offset", [(1e-4, 0.0), (1.0, 0.0), (1e3, 0.0), (1e15, 0.0), (1.0, 1e4)])
def test_chamfer_fp64_reference(oracle_mod, scale, offset):
    """Selected pairs against fp64 distances. All terms of d are non-negative, so the fp32
    d = ((dx*dx + dy*dy) + dz*dz) of a pair is within 6 U of its fp64 value (relative); the selected
    pair is then within 12 U of the fp64 minimum over all candidates, and the term sqrt(d + 1e-8)
    within 5 U of its fp64 value. Scale 1e-4 puts squared distances near the 1e-8 epsilon, 1e15
    near 1e30; offset 1e4 makes every difference cancel."""
    rs = np.random.RandomState(11)
    B, Mp, N = 2, 300, 1324
    pred, gt = _cloud(rs, B, Mp, scale, offset), _cloud(rs, B, N, scale, offset)
    r = _chamfer(pred, gt)
    _assert_idx_in_range(r, Mp, N)
    p64, g64 = pred.double().to(DEV), gt.double().to(DEV)
    D = ((p64[:, :, :, None] - g64[:, :, None, :]) ** 2).sum(1)                 # [B, Mp, N]
    for what, Dq, q, db, idx, elem in (("fwd", D, pred, gt, r["idx_fwd"], r["elem_fwd"]),
                                       ("bwd", D.transpose(1, 2), gt, pred, r["idx_bwd"], r["elem_bwd"])):
        idx = idx.long()
        sel = Dq.gather(2, idx.to(DEV)[:, :, None])[:, :, 0].cpu()
        dmin = Dq.min(2)[0].cpu()
        sel_db = torch.gather(db, 2, idx[:, None, :].expand(-1, 3, -1))
        d32 = torch.stack([oracle_mod.pair_dist2(q[b], sel_db[b]) for b in range(B)]).double()
        assert bool(((d32 - sel).abs() <= 6 * U * sel).all()), "%s: fp32 distance vs fp64" % what
        assert bool((sel <= dmin * (1 + 12 * U)).all()), "%s: not the nearest neighbour" % what
        want = (sel + EPS).sqrt()
        err = (elem.double() - want).abs() / want
        assert float(err.max()) <= 5 * U, "%s: term rel err %.3g U" % (what, float(err.max()) / U)
    _assert_sums(r)


# ---- ties across tile boundaries ---------------------------------------------------------------------
def test_chamfer_ties_across_column_ctas(oracle_mod):
    """Duplicate gt points on both sides of the 1024-column CTA boundaries; pred points on them
    (distance 0) or 1e-3 off them (equal non-zero distances): the lowest column wins."""
    rs = np.random.RandomState(21)
    B, Mp, N = 2, 300, 2100
    pred, gt = _cloud(rs, B, Mp), _cloud(rs, B, N)
    lo = torch.from_numpy(np.r_[1004:1024, 1050:1070, 0])      # CTA 0 | 1, CTA 1 | 2, CTA 0 | 2
    hi = torch.from_numpy(np.r_[1024:1044, 2048:2068, 2099])
    gt[:, :, hi] = gt[:, :, lo]
    pred[:, :, :41] = gt[:, :, lo]
    pred[:, :, 41:82] = gt[:, :, lo] + 1e-3
    r, _ = _check_vs_oracle(oracle_mod, pred, gt)
    want = lo.int()
    assert torch.equal(r["idx_fwd"][:, :41], want.expand(B, -1))
    assert torch.equal(r["idx_fwd"][:, 41:82], want.expand(B, -1))


def test_chamfer_ties_across_row_tiles(oracle_mod):
    """Duplicate pred points on both sides of the 128-row tile boundaries (and two tiles apart);
    gt points on them or 1e-3 off them: the lowest row wins."""
    rs = np.random.RandomState(22)
    B, Mp, N = 2, 300, 1324
    pred, gt = _cloud(rs, B, Mp), _cloud(rs, B, N)
    lo = torch.from_numpy(np.r_[100:128, 90:100, 0])           # tile 0 | 1, tile 0 | 2, tile 0 | 2
    hi = torch.from_numpy(np.r_[128:156, 260:270, 299])
    pred[:, :, hi] = pred[:, :, lo]
    gt[:, :, :39] = pred[:, :, lo]
    gt[:, :, 1200:1239] = pred[:, :, lo] + 1e-3
    r, _ = _check_vs_oracle(oracle_mod, pred, gt)
    want = lo.int()
    assert torch.equal(r["idx_bwd"][:, :39], want.expand(B, -1))
    assert torch.equal(r["idx_bwd"][:, 1200:1239], want.expand(B, -1))


@pytest.mark.parametrize("B,Mp,N", [(3, 1280, 2648), (2, 129, 5000)])
def test_chamfer_quantised_mass_ties(oracle_mod, B, Mp, N):
    """Coordinates on a 1/8 grid (17^3 sites): many points have several equidistant neighbours,
    and duplicates land in every tile."""
    rs = np.random.RandomState(B + Mp)
    pred = torch.from_numpy(np.round(rs.uniform(-1, 1, size=(B, 3, Mp)) * 8).astype(np.float32) / 8)
    gt = torch.from_numpy(np.round(rs.uniform(-1, 1, size=(B, 3, N)) * 8).astype(np.float32) / 8)
    _check_vs_oracle(oracle_mod, pred, gt)
    p64, g64 = pred.double().to(DEV), gt.double().to(DEV)
    D = ((p64[:, :, :, None] - g64[:, :, None, :]) ** 2).sum(1)
    ties = (D == D.min(2, keepdim=True)[0]).sum(2)
    assert int((ties > 1).sum()) > B * Mp // 4          # the case is what it says


# ---- non-finite inputs --------------------------------------------------------------------------------
NONFINITE = ["nan_pred_point", "nan_gt_point", "nan_pred_cloud", "nan_gt_cloud", "overflow_all",
             "overflow_point", "far_points", "nan_or_overflow", "overflow_or_nan"]


def _nonfinite_case(kind):
    rs = np.random.RandomState(NONFINITE.index(kind))
    B, Mp, N = 2, 300, 1324
    pred, gt = _cloud(rs, B, Mp), _cloud(rs, B, N)
    nan = float("nan")
    if kind == "nan_pred_point":
        pred[1, 1, 129] = nan                       # first row of the second tile
    elif kind == "nan_gt_point":
        gt[0, 2, 1025] = nan                        # a column of the last (partial) CTA
    elif kind == "nan_pred_cloud":
        pred[1] = nan
    elif kind == "nan_gt_cloud":
        gt[0] = nan
    elif kind == "overflow_all":                    # every squared distance overflows to +inf
        pred = pred.abs() * 1e20 + 1e20
        gt = -(gt.abs() * 1e20 + 1e20)
    elif kind == "overflow_point":                  # one point far away: nobody's neighbour
        pred[0, :, 7] = 1e20
        gt[1, :, 1300] = -1e20
    elif kind == "far_points":                      # where a finite tile padding would be nearest
        pred[0, :, 5] = -1e30
        gt[1, :, 9] = 1e30
    elif kind == "nan_or_overflow":                 # every candidate NaN or +inf; gt point 0 NaN
        gt[:, :, 0] = nan
        gt[:, :, 1:] = 1e20
    elif kind == "overflow_or_nan":                 # gt point 0 overflows, every other one NaN
        gt[:, :, 0] = 1e20
        gt[:, :, 1:] = nan
    return pred, gt


@pytest.mark.parametrize("kind", NONFINITE)
def test_chamfer_nonfinite_inputs(oracle_mod, kind):
    """A point with no finite nearest neighbour gets index 0 and the term of the pair (point,
    other cloud's point 0), as the oracle's scan from (+inf, 0) does: NaN with a NaN, +inf on
    overflow. Indices stay in range; per-cloud means and losses are NaN / inf exactly where the
    oracle's are."""
    pred, gt = _nonfinite_case(kind)
    r, o = _check_vs_oracle(oracle_mod, pred, gt, sums=False)
    for got, want in ((r["fwd_arr"], o["forward_loss_array"]), (r["bwd_arr"], o["backward_loss_array"]),
                      (r["loss"], torch.stack([o["forward_loss"], o["backward_loss"], o["loss"]]))):
        assert torch.equal(got.isnan(), want.isnan()), (got, want)
        assert torch.equal(got.isinf(), want.isinf()), (got, want)
        fin = got.isfinite()
        if bool(fin.any()):
            assert_close(got[fin], want[fin], "finite means")
    if kind == "nan_pred_point":
        assert int(r["idx_fwd"][1, 129]) == 0 and math.isnan(float(r["elem_fwd"][1, 129]))
        assert bool(r["elem_bwd"].isfinite().all())
    if kind == "nan_or_overflow":
        assert bool((r["idx_fwd"] == 0).all()) and bool(r["elem_fwd"].isnan().all())


def test_chamfer_training_path_nan_point_gives_nan_loss():
    """One NaN in the decoder output makes the training loss NaN instead of an out-of-range
    gather: the clouds without it keep finite losses."""
    from sonet_b200 import losses, synth
    pred, gt = _nonfinite_case("nan_pred_point")
    r = _chamfer(pred, gt)
    _assert_idx_in_range(r, pred.shape[2], gt.shape[2])          # before ChamferLoss gathers
    crit = losses.ChamferLoss(synth.make_opt("autoencoder"))
    p = pred.to(DEV).requires_grad_(True)
    with torch.enable_grad():
        loss = crit(p, gt.to(DEV))
        loss.backward()
    assert math.isnan(float(loss.detach()))
    arr = crit.loss_array.detach().cpu()
    assert math.isfinite(float(arr[0])) and math.isnan(float(arr[1]))
    assert torch.equal(crit.nn_idx_fwd.cpu(), r["idx_fwd"]) and torch.equal(crit.nn_idx_bwd.cpu(), r["idx_bwd"])
    assert bool(p.grad[0].isfinite().all())


# ---- reductions ---------------------------------------------------------------------------------------
def test_chamfer_batch_beyond_final_kernel_threads(oracle_mod):
    """B = 300 > the 256 threads of chamfer_final_kernel: losses against fp64 means."""
    rs = np.random.RandomState(300)
    pred, gt = _cloud(rs, 300, 129), _cloud(rs, 300, 257)
    _check_vs_oracle(oracle_mod, pred, gt)


def test_chamfer_batch_slices_and_repeats_are_bit_identical():
    rs = np.random.RandomState(5)
    pred, gt = _cloud(rs, 12, 1280), _cloud(rs, 12, 2648)
    r = _chamfer(pred, gt)
    again = _chamfer(pred, gt)
    for k in r:
        assert torch.equal(r[k], again[k]), k
    s = _chamfer(pred[5:9], gt[5:9])
    for k in ("idx_fwd", "idx_bwd", "elem_fwd", "elem_bwd", "fwd_arr", "bwd_arr"):
        assert torch.equal(s[k], r[k][5:9]), k


# ---- production shapes --------------------------------------------------------------------------------
@pytest.mark.parametrize("B,Mp,N", [(32, 256, 5000), (32, 1280, 5000), (8, 4352, 5000)])
def test_chamfer_production_shapes_vs_oracle(oracle_mod, B, Mp, N):
    """The auto-encoder's calls: conv_pc4 (256) and predicted_pc (1280) against 5000-point clouds
    at B = 32, and the output_conv_pc_num=4096 option's 4352 points."""
    rs = np.random.RandomState(Mp)
    _check_vs_oracle(oracle_mod, _cloud(rs, B, Mp), _cloud(rs, B, N))


# ---- training path -----------------------------------------------------------------------------------
def _fp64_chamfer_grads(pred, gt, i_f, i_b, gt_grad):
    """fp64 autograd of the reference's formulation (losses.py:269-289) with the given indices, and
    per element the sum of the absolute values of the terms its gradient adds up, and how many."""
    B, _, Mp = pred.shape
    N = gt.shape[2]
    p = pred.detach().double().requires_grad_(True)
    g = gt.detach().double().requires_grad_(gt_grad)
    ef, eb = i_f.long()[:, None, :].expand(-1, 3, -1), i_b.long()[:, None, :].expand(-1, 3, -1)
    vf, vb = g.gather(2, ef) - p, p.gather(2, eb) - g
    f = ((vf ** 2).sum(1) + EPS).sqrt()
    b = ((vb ** 2).sum(1) + EPS).sqrt()
    (f.mean() + b.mean()).backward()
    with torch.no_grad():
        tf = vf.abs() / f[:, None, :] / (B * Mp)
        tb = vb.abs() / b[:, None, :] / (B * N)
        mag_p = tf + torch.zeros_like(tf).scatter_add_(2, eb, tb)
        mag_g = tb + torch.zeros_like(tb).scatter_add_(2, ef, tf)
        cnt_p = 1 + torch.zeros_like(tf).scatter_add_(2, eb, torch.ones_like(tb))
        cnt_g = 1 + torch.zeros_like(tb).scatter_add_(2, ef, torch.ones_like(tf))
    return p.grad, (g.grad if gt_grad else None), (mag_p, cnt_p), (mag_g, cnt_g)


@pytest.mark.parametrize("B,Mp,N,gt_grad", [(2, 300, 1025, False), (3, 129, 2648, True),
                                            (1, 1280, 5000, True), (4, 33, 257, True)])
def test_chamfer_training_path_vs_fp64(B, Mp, N, gt_grad):
    """ChamferLoss with gradients: the search is the kernel's, the loss a differentiable gather.
    Its loss and per-cloud arrays agree with the eval path's (two fixed-order fp32 sums of the same
    positive terms: 48 U covers either's worst-case rounding), its indices are the kernel's, and
    each gradient element is within (32 + terms) U of fp64 autograd relative to the sum of the
    absolute values of its terms."""
    from sonet_b200 import losses, synth
    rs = np.random.RandomState(B * Mp + N)
    pred, gt = _cloud(rs, B, Mp), _cloud(rs, B, N)
    r = _chamfer(pred, gt)
    _assert_idx_in_range(r, Mp, N)                                   # before ChamferLoss gathers
    crit = losses.ChamferLoss(synth.make_opt("autoencoder"))
    with torch.no_grad():
        ev = float(crit(pred.to(DEV), gt.to(DEV)))
        ev_f, ev_b = crit.forward_loss_array.cpu(), crit.backward_loss_array.cpu()
    p = pred.to(DEV).requires_grad_(True)
    g = gt.to(DEV).requires_grad_(gt_grad)
    with torch.enable_grad():
        loss = crit(p, g)
        loss.backward()
    assert torch.equal(crit.nn_idx_fwd.cpu(), r["idx_fwd"]) and torch.equal(crit.nn_idx_bwd.cpu(), r["idx_bwd"])
    assert abs(float(loss.detach()) - ev) <= 48 * U * ev
    for got, want in ((crit.forward_loss_array.detach().cpu(), ev_f),
                      (crit.backward_loss_array.detach().cpu(), ev_b)):
        assert bool(((got.double() - want.double()).abs() <= 48 * U * want.double()).all())
    gp, gg, (mp, cp), (mg, cg) = _fp64_chamfer_grads(pred, gt, r["idx_fwd"], r["idx_bwd"], gt_grad)
    for what, got, want, mag, cnt in (("d pred", p.grad, gp, mp, cp), ("d gt", g.grad, gg, mg, cg)):
        if want is None:
            assert got is None
            continue
        err = (got.cpu().double() - want).abs()
        bound = (32 + cnt) * U * mag
        assert bool((err <= bound).all()), "%s: %.3g x the bound" % (what, float((err / bound).max()))
