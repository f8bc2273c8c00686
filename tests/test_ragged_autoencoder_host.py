"""Whole-cloud reconstruction (losses.chamfer_ragged, ops.chamfer_ragged,
autoencoder.Model.reconstruct_clouds) without a GPU: the C-ABI exports the ragged Chamfer entry with
a header-derived signature and refuses bad arguments before any launch, every Python refusal fires
before any launch, and the numpy restatement of the kernels' contract (tests/chamfer_emu.py) agrees
with the oracle's brute-force scan."""
import ctypes

import numpy as np
import pytest
import torch

import chamfer_emu
from sonet_b200 import _C, autoencoder, losses, ops, synth

ENTRY = "sonet_chamfer_ragged_f32"


@pytest.fixture
def no_launch(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(ops, "_call", refuse)


# ---- C-ABI ----------------------------------------------------------------------------------------
def test_cabi_has_the_entry(lib_built):
    h = ctypes.CDLL(lib_built)
    assert hasattr(h, ENTRY) and ENTRY in _C._SIGNATURES
    assert ENTRY not in _C.ACT_ENTRIES and ENTRY not in _C.F16_ENTRIES
    sig = _C._SIGNATURES[ENTRY]
    assert len(sig) == 17
    assert sig[1] is ctypes.c_int and sig[2] is ctypes.c_int          # B, Mp
    assert sig[4] is ctypes.c_longlong and sig[5] is ctypes.c_longlong  # T, ld
    assert all(sig[i] is ctypes.c_void_p for i in (0, 3, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16))
    assert _C._RESTYPE[ENTRY] is ctypes.c_int


def _call(B=3, Mp=4, T=None, ld=6, offsets=(0, 2, 5, 9), idx=True, null=None):
    """The entry with dummy (never dereferenced on the device) pointers and a real host offsets
    array; `null` names the argument passed as NULL."""
    lib = _C.lib()
    off = np.asarray(offsets, dtype=np.int64)
    T = int(off[-1]) if T is None else T
    fake = 256                                   # a non-null address: refusals come first
    args = dict(pred=fake, points=fake, offsets=fake, offsets_host=off.ctypes.data, tile_start=fake,
                idx_fwd=fake if idx else None, idx_bwd=fake if idx else None, elem_fwd=fake,
                elem_bwd=fake, fwd=fake, bwd=fake, loss=fake)
    if null:
        args[null] = None
    rc = lib.sonet_chamfer_ragged_f32(args["pred"], B, Mp, args["points"], T, ld, args["offsets"],
                                      args["offsets_host"], args["tile_start"], args["idx_fwd"],
                                      args["idx_bwd"], args["elem_fwd"], args["elem_bwd"],
                                      args["fwd"], args["bwd"], args["loss"], None)
    return rc, _C.last_error()


@pytest.mark.parametrize("null", ["pred", "points", "offsets", "offsets_host", "tile_start",
                                  "elem_fwd", "elem_bwd", "fwd", "bwd", "loss"])
def test_cabi_refuses_null_pointers(lib_built, null):
    rc, err = _call(null=null)
    assert rc == -1 and "null" in err


@pytest.mark.parametrize("case,kw,msg", [
    ("B0", dict(B=0, offsets=(0,)), "B=0"),
    ("Mp0", dict(Mp=0), "Mp=0"),
    ("ld2", dict(ld=2), "stride"),
    ("idx_fwd_alone", dict(null="idx_bwd"), "together"),
    ("idx_bwd_alone", dict(null="idx_fwd"), "together"),
    ("start", dict(offsets=(1, 2, 5, 9)), "from 0"),
    ("end", dict(offsets=(0, 2, 5, 9), T=10), "from 0"),
    ("empty_first", dict(offsets=(0, 0, 5, 9)), "cloud 0 has no points"),
    ("empty_mid", dict(offsets=(0, 2, 2, 9)), "cloud 1 has no points"),
    ("decreasing", dict(offsets=(0, 6, 5, 9)), "cloud 1 has no points"),
    ("too_large", dict(B=2, offsets=(0, 1, 1 + (1 << 24))), "cloud 1 has 16777216 points"),
])
def test_cabi_argument_checks(lib_built, case, kw, msg):
    rc, err = _call(**kw)
    assert rc == -1 and msg in err, (case, err)


# ---- Python refusals --------------------------------------------------------------------------------
def _ragged(B=3, Mp=8):
    pts = torch.zeros(9, 6)
    off = torch.tensor([0, 2, 5, 9], dtype=torch.int64)
    return torch.zeros(B, 3, Mp), pts, off


@pytest.mark.parametrize("case", ["pred_device", "pred_dtype", "points_device", "points_dtype",
                                  "offsets_device"])
def test_chamfer_ragged_refusals_before_any_launch(no_launch, case):
    pred, pts, off = _ragged()
    if case == "pred_dtype":
        pred = pred.double()
    elif case == "points_dtype":
        pts = pts.double()
    elif case == "offsets_device":
        pass                                     # everything on the CPU: refused as not CUDA
    with pytest.raises(RuntimeError, match="CUDA|dtype|float32"):
        ops.chamfer_ragged(pred, pts, off)


@pytest.mark.parametrize("which", ["predict_pc", "points"])
def test_losses_chamfer_ragged_refuses_gradients(no_launch, which):
    pred, pts, off = _ragged()
    (pred if which == "predict_pc" else pts).requires_grad_(True)
    with pytest.raises(RuntimeError, match="evaluation only"):
        losses.chamfer_ragged(pred, pts, off)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):
        losses.chamfer_ragged(pred, pts, off)       # grad mode off: on to the device check


def _ae(**over):
    opt = synth.make_opt("autoencoder", batch_size=3, input_pc_num=10, **over)
    m = autoencoder.Model(opt)
    m.encoder.eval()
    m.decoder.eval()
    return m


def _ae_args(B=3, M=64, som_k=9):
    pts = torch.zeros(30, 6)
    off = torch.tensor([0, 10, 20, 30], dtype=torch.int64)
    return pts, off, torch.zeros(B, 3, M), torch.zeros(B, M, som_k, dtype=torch.int64)


@pytest.mark.parametrize("case", ["train_encoder", "train_decoder", "instance", "points_dtype",
                                  "points_cols", "node_shape", "offsets_dtype", "offsets_end",
                                  "offsets_decrease", "knn_shape", "device", "chunk", "empty"])
def test_reconstruct_clouds_refusals_before_any_launch(no_launch, case):
    m = _ae(normalization="instance" if case == "instance" else "batch")
    if case == "train_encoder":
        m.encoder.train()
    elif case == "train_decoder":
        m.decoder.train()
    pts, off, node, knn = _ae_args()
    kw = {}
    err = RuntimeError
    if case == "points_dtype":
        pts = pts.double()
    elif case == "points_cols":
        pts = torch.zeros(30, 3)
    elif case == "node_shape":
        node = torch.zeros(3, 2, 64)
    elif case == "offsets_dtype":
        off = off.int()
    elif case == "offsets_end":
        off = torch.tensor([0, 10, 20, 29])
    elif case == "offsets_decrease":
        off = torch.tensor([0, 20, 10, 30])
    elif case == "knn_shape":
        knn = torch.zeros(3, 64, 2, dtype=torch.int64)
    elif case == "device":
        pts = pts.to("meta")
    elif case == "chunk":
        kw["chunk_points"] = 0
    elif case == "empty":
        off = torch.tensor([0, 10, 10, 30])
        err = ValueError
    with pytest.raises(err, match="reconstruct_clouds|offsets"):
        m.reconstruct_clouds(pts, off, node, knn, **kw)


# ---- the numpy restatement --------------------------------------------------------------------------
def _cloud(rs, P, scale=1.0):
    return (rs.uniform(-1, 1, size=(3, P)) * scale).astype(np.float32)


@pytest.mark.parametrize("Mp,N", [(1, 1), (7, 300), (130, 65), (40, 1100)])
def test_restatement_matches_the_oracle_scan(oracle_mod, Mp, N):
    rs = np.random.RandomState(Mp * 7 + N)
    pred, gt = _cloud(rs, Mp), _cloud(rs, N)
    gt[:, N // 2:N // 2 + 3] = gt[:, :3] if N > 6 else gt[:, N // 2:N // 2 + 3]   # ties
    o = oracle_mod.chamfer(torch.from_numpy(pred[None]), torch.from_numpy(gt[None]))
    e = chamfer_emu.chamfer_cloud(pred, gt)
    assert np.array_equal(e["idx_fwd"], o["idx_fwd"][0].numpy().astype(np.int64))
    assert np.array_equal(e["idx_bwd"], o["idx_bwd"][0].numpy().astype(np.int64))
    for k, d in (("elem_fwd", "dist2_fwd"), ("elem_bwd", "dist2_bwd")):
        want = oracle_mod.chamfer_elem(o[d])[0].numpy()
        assert np.array_equal(e[k].view(np.uint32), want.view(np.uint32)), k
    for k, a in (("fwd", "forward_loss_array"), ("bwd", "backward_loss_array")):
        assert abs(float(e[k]) - float(o[a][0])) <= 1e-6 * float(o[a][0]), k


def test_restatement_non_finite_rule(oracle_mod):
    """NaN and overflowing coordinates: the scan's (+inf, index 0) rule, as the oracle applies it."""
    rs = np.random.RandomState(3)
    pred, gt = _cloud(rs, 20), _cloud(rs, 50)
    pred[0, 3] = np.nan
    pred[:, 4] = 3e38
    gt[1, 7] = np.nan
    gt[:, 9] = -3e38
    o = oracle_mod.chamfer(torch.from_numpy(pred[None]), torch.from_numpy(gt[None]))
    e = chamfer_emu.chamfer_cloud(pred, gt)
    assert np.array_equal(e["idx_fwd"], o["idx_fwd"][0].numpy().astype(np.int64))
    assert np.array_equal(e["idx_bwd"], o["idx_bwd"][0].numpy().astype(np.int64))
    assert e["idx_fwd"][3] == 0 and e["idx_fwd"][4] == 0
    want = oracle_mod.chamfer_elem(o["dist2_fwd"])[0].numpy()
    assert np.array_equal(np.isnan(e["elem_fwd"]), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.array_equal(e["elem_fwd"][ok], want[ok])


@pytest.mark.parametrize("P", [1, 31, 32, 1023, 1024, 1025, 5000])
def test_fixed_order_sums_within_fp64_bounds(P):
    """cloud_mean / final_loss of positive terms against fp64: within (chain + 12) ulps."""
    rs = np.random.RandomState(P)
    e = rs.uniform(0.1, 2, size=P).astype(np.float32)
    got = float(chamfer_emu.cloud_mean(e))
    want = e.astype(np.float64).mean()
    assert abs(got - want) <= (-(-P // 1024) + 12) * 2.0 ** -24 * want
    a, b = e[:min(P, 700)], e[::-1][:min(P, 700)]
    loss = chamfer_emu.final_loss(a, b)
    for j, x in ((0, a), (1, b)):
        w = x.astype(np.float64).mean()
        assert abs(float(loss[j]) - w) <= (-(-len(x) // 256) + 10) * 2.0 ** -24 * w
    assert loss[2] == np.float32(loss[0] + loss[1])


def test_ragged_restatement_is_per_cloud():
    rs = np.random.RandomState(9)
    sizes = [1, 1025, 300]
    pts = rs.uniform(-1, 1, size=(sum(sizes), 6)).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(sizes)])
    pred = rs.uniform(-1, 1, size=(3, 3, 40)).astype(np.float32)
    r = chamfer_emu.chamfer_ragged(pred, pts, off)
    for b in range(3):
        c = chamfer_emu.chamfer_cloud(pred[b], pts[off[b]:off[b + 1], :3].T)
        assert np.array_equal(r["idx_bwd"][off[b]:off[b + 1]], c["idx_bwd"])
        assert np.array_equal(r["idx_fwd"][b], c["idx_fwd"])
        assert (r["idx_fwd"][b] < sizes[b]).all() and (r["idx_bwd"] < 40).all()
        assert r["fwd_arr"][b] == c["fwd"] and r["bwd_arr"][b] == c["bwd"]
