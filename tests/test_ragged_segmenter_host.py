"""Whole-shape part segmentation (segmenter.Model.segment_clouds, losses.seg_loss_ragged,
ops.seg_loss_ragged) without a GPU: the C-ABI exports the ragged loss entry and its scratch size with
header-derived signatures and refuses bad arguments before touching a device, and every Python
refusal fires before any launch."""
import ctypes
import re

import numpy as np
import pytest
import torch

from sonet_b200 import _C, losses, ops, segmenter, synth

ENTRY = "sonet_seg_loss_ragged_f32"
SCRATCH = "sonet_seg_loss_ragged_scratch_bytes"


@pytest.fixture
def no_launch(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(ops, "_call", refuse)


# ---- C-ABI ----------------------------------------------------------------------------------------
def test_cabi_has_the_entries(lib_built):
    h = ctypes.CDLL(lib_built)
    for name in (ENTRY, SCRATCH):
        assert hasattr(h, name) and name in _C._SIGNATURES
        assert name not in _C.ACT_ENTRIES and name not in _C.F16_ENTRIES
    sig = _C._SIGNATURES[ENTRY]
    assert len(sig) == 11
    assert sig[4] is ctypes.c_int and sig[5] is ctypes.c_int and sig[6] is ctypes.c_longlong
    assert all(sig[i] is ctypes.c_void_p for i in (0, 1, 2, 3, 7, 8, 9, 10))
    assert _C._RESTYPE[ENTRY] is ctypes.c_int
    assert tuple(_C._SIGNATURES[SCRATCH]) == (ctypes.c_int, ctypes.c_longlong)
    assert _C._RESTYPE[SCRATCH] is ctypes.c_longlong


def _tiles(sizes):
    return sum(-(-P // 256) for P in sizes)


@pytest.mark.parametrize("sizes", [[0], [1], [255], [256], [257], [1, 1, 1, 1], [0, 0, 5],
                                   [3000, 17, 1 << 20], [256] * 64, [255, 1] * 33])
def test_scratch_bytes(lib_built, sizes):
    """(T / 256 + B) partials of a double and an int, B + 1 tile starts and 16 bytes: enough for
    every cloud's tiles, however the T points split into B clouds."""
    lib = _C.lib()
    B, T = len(sizes), sum(sizes)
    got = lib.sonet_seg_loss_ragged_scratch_bytes(B, T)
    assert got == (T // 256 + B) * 12 + 4 * (B + 1) + 16
    assert got >= _tiles(sizes) * 12 + 4 * (B + 1)


def test_scratch_bytes_refuses_negative_sizes(lib_built):
    lib = _C.lib()
    assert lib.sonet_seg_loss_ragged_scratch_bytes(-1, 5) == -1
    assert lib.sonet_seg_loss_ragged_scratch_bytes(2, -1) == -1
    assert lib.sonet_seg_loss_ragged_scratch_bytes(0, 0) == 4 + 16


def _call(B=3, C=50, T=None, offsets=(0, 2, 5, 9), null=None):
    """The entry with dummy (never dereferenced on the device) pointers and a real host offsets
    array; `null` names the argument passed as NULL."""
    lib = _C.lib()
    off = np.asarray(offsets, dtype=np.int64)
    T = int(off[-1]) if T is None else T
    fake = 256                                   # a non-null address: refusals come first
    args = dict(score=fake, target=fake, offsets=fake, offsets_host=off.ctypes.data, scratch=fake,
                loss=fake, loss_array=fake)
    if null:
        args[null] = None
    rc = lib.sonet_seg_loss_ragged_f32(args["score"], args["target"], args["offsets"],
                                       args["offsets_host"], B, C, T, args["scratch"], args["loss"],
                                       args["loss_array"], None)
    return rc, _C.last_error()


@pytest.mark.parametrize("null", ["score", "target", "offsets", "offsets_host", "scratch", "loss",
                                  "loss_array"])
def test_cabi_refuses_null_pointers(lib_built, null):
    rc, err = _call(null=null)
    assert rc == -1 and "null" in err


BIG = (1 << 31) - 257                            # the largest cloud the entry takes


@pytest.mark.parametrize("case,kw,msg", [
    ("B0", dict(B=0, offsets=(0,)), "B=0"),
    ("C0", dict(C=0), "C=0"),
    ("T_negative", dict(T=-1, offsets=(0, 0, 0, -1)), "negative"),
    ("start", dict(offsets=(1, 2, 5, 9)), "from 0"),
    ("end", dict(offsets=(0, 2, 5, 9), T=10), "from 0"),
    ("decreasing", dict(offsets=(0, 6, 5, 9)), "decrease at cloud 1"),
    ("cloud_too_large", dict(B=2, offsets=(0, 1, 2 + BIG)), "cloud 1 has 2147483392 points"),
    ("partials", dict(B=300, offsets=tuple(range(0, 301 * BIG, BIG))), "partials, 2^31"),
])
def test_cabi_argument_checks(lib_built, case, kw, msg):
    rc, err = _call(**kw)
    assert rc == -1 and msg in err, (case, err)


# ---- Python refusals --------------------------------------------------------------------------------
def _loss_args():
    return torch.zeros(9, 50), torch.zeros(9, dtype=torch.int64), \
        torch.tensor([0, 2, 5, 9], dtype=torch.int64)


@pytest.mark.parametrize("case", ["score_device", "score_dtype", "target_dtype", "offsets_dtype"])
def test_seg_loss_ragged_refusals_before_any_launch(no_launch, case):
    score, target, off = _loss_args()
    if case == "score_dtype":
        score = score.double()
    elif case == "target_dtype":
        target = target.int()
    elif case == "offsets_dtype":
        off = off.int()
    with pytest.raises(RuntimeError, match="CUDA|dtype"):
        ops.seg_loss_ragged(score, target, off)


def test_losses_seg_loss_ragged_refuses_gradients(no_launch):
    score, target, off = _loss_args()
    score.requires_grad_(True)
    with pytest.raises(RuntimeError, match="evaluation only"):
        losses.seg_loss_ragged(score, target, off)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):
        losses.seg_loss_ragged(score, target, off)       # grad mode off: on to the device check


def _seg(**over):
    opt = synth.make_opt("segmenter", batch_size=3, input_pc_num=10, **over)
    m = segmenter.Model(opt)
    m.encoder.eval()
    m.segmenter.eval()
    return m


def _seg_args(B=3, M=64, som_k=9):
    pts = torch.zeros(30, 6)
    off = torch.tensor([0, 10, 20, 30], dtype=torch.int64)
    return pts, off, torch.tensor([0, 4, 15]), torch.zeros(B, 3, M), \
        torch.zeros(B, M, som_k, dtype=torch.int64), torch.zeros(30, dtype=torch.int64)


CASES = {   # case -> what its message says
    "train_encoder": "train mode", "train_head": "train mode", "instance": "instance",
    "som_k1": "som_k >= 2", "points_dtype": "points", "points_cols": "points",
    "node_shape": "node", "offsets_dtype": "offsets", "offsets_end": "offsets",
    "offsets_decrease": "offsets", "knn_shape": "node_knn_I", "device": "device", "chunk": "chunk",
    "empty": "no points", "label_dtype": "label must be an int64", "label_shape": "label must be",
    "label_device": "label must be on", "label_range": "outside \\[0, 16\\)",
    "label_list": "label must be", "seg_dtype": "seg must be an int64", "seg_shape": "seg must be",
    "seg_device": "seg must be on",
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_segment_clouds_refusals_before_any_launch(no_launch, case):
    over = {}
    if case == "instance":
        over["normalization"] = "instance"
    if case == "som_k1":
        over["som_k"] = 1
    m = _seg(**over)
    if case == "train_encoder":
        m.encoder.train()
    elif case == "train_head":
        m.segmenter.train()
    pts, off, label, node, knn, seg = _seg_args(som_k=1 if case == "som_k1" else 9)
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
    elif case == "label_dtype":
        label = label.int()
    elif case == "label_shape":
        label = torch.zeros(2, dtype=torch.int64)
    elif case == "label_device":
        label = label.to("meta")
    elif case == "label_range":
        label = torch.tensor([0, 16, 1])
    elif case == "label_list":
        label = [0, 1, 2]
    elif case == "seg_dtype":
        seg = seg.int()
    elif case == "seg_shape":
        seg = torch.zeros(29, dtype=torch.int64)
    elif case == "seg_device":
        seg = seg.to("meta")
    with pytest.raises(err, match="segment_clouds|offsets") as e:
        m.segment_clouds(pts, off, label, node, knn, seg=seg, **kw)
    assert re.search(CASES[case], str(e.value)), (case, str(e.value))


def test_segment_clouds_without_refusal_reaches_the_device(no_launch):
    """The same arguments unchanged pass every refusal: the first thing that stops them on a
    host-only model is a CUDA requirement further in, not a segment_clouds refusal."""
    m = _seg()
    pts, off, label, node, knn, seg = _seg_args()
    with pytest.raises((RuntimeError, ValueError, AssertionError)) as e:
        m.segment_clouds(pts, off, label, node, knn, seg=seg)
    assert "segment_clouds" not in str(e.value)
