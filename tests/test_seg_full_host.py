"""Full-resolution part segmentation without a GPU: the C-ABI of the ragged SOM assignment and the
ragged IoU (declared, exported, argument checks), the host twin of the ragged IoU against a numpy
restatement of the reference's compute_iou rule, and score_points' refusals."""
import ctypes

import numpy as np
import pytest
import torch

from sonet_b200 import _C, losses, ops, segmenter, synth

ENTRIES = ("sonet_seg_points_assign_f32", "sonet_seg_iou_ragged_f32", "sonet_seg_iou_ragged_cpu_f32")


def _ref_iou(score, seg, label, offsets, table=ops.SHAPENET_PART_TABLE):
    """models/losses.py:119-189 per shape, over all its points: argmax over all classes, then
    I / (U + 0.0001) per part of the category (1.0 for an empty union), mean over the parts."""
    out = []
    for b in range(len(label)):
        sc = score[offsets[b]:offsets[b + 1]]
        pred = np.argmax(sc, axis=1)
        gt = seg[offsets[b]:offsets[b + 1]]
        ious = []
        for p in table[label[b]]:
            i = np.sum((pred == p) & (gt == p))
            u = np.sum((pred == p) | (gt == p))
            ious.append(1.0 if u == 0 else i / float(u + 0.0001))
        out.append(np.mean(ious))
    return np.asarray(out)


def _ragged_case(seed, sizes):
    rs = np.random.RandomState(seed)
    T = int(sum(sizes))
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    label = rs.randint(0, 16, size=len(sizes)).astype(np.int64)
    score = rs.normal(size=(T, 50)).astype(np.float32)
    seg = np.empty(T, dtype=np.int64)
    for b, lab in enumerate(label):
        parts = ops.SHAPENET_PART_TABLE[lab]
        n = sizes[b]
        # the category's first part is absent from the ground truth and never predicted
        seg[offsets[b]:offsets[b + 1]] = rs.choice(parts[1:] if len(parts) > 1 else parts, size=n)
        sc = score[offsets[b]:offsets[b + 1]]
        sc[:, parts[0]] = -1e9
        sc[np.arange(n), seg[offsets[b]:offsets[b + 1]]] += rs.uniform(0, 3, size=n).astype(np.float32)
    return score, seg, label, offsets


def test_entries_declared_and_exported(lib_built):
    lib = _C.lib()
    for name in ENTRIES:
        assert name in _C.EXPORTED_SYMBOLS, name
        assert getattr(lib, name).restype is ctypes.c_int


@pytest.mark.parametrize("sizes", [[1], [5, 0, 3000, 17], [2048, 2999, 2500]])
def test_compute_iou_full_host_matches_numpy(lib_built, sizes):
    score, seg, label, offsets = _ragged_case(len(sizes), sizes)
    got = losses.compute_iou_full(torch.from_numpy(score), torch.from_numpy(seg),
                                  torch.from_numpy(label), torch.from_numpy(offsets))
    ref = _ref_iou(score, seg, label, offsets)
    np.testing.assert_array_equal(got, ref)


def _assign(points=True, offsets=True, node=True, cm=True, B=2, M=16, k=3, rows=4, rows_pad=256,
            total=8, row0=0, with_sn=1):
    """sonet_seg_points_assign_f32 with host buffers: every check fails before a CUDA call."""
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    lib = _C.lib()
    return lib.sonet_seg_points_assign_f32(p if points else None, total, p if offsets else None, B,
                                           p if node else None, p if cm else None, M, k, with_sn, row0,
                                           rows, rows_pad, p, p, p, None)


@pytest.mark.parametrize("kw, msg", [
    (dict(points=False), "null pointer"), (dict(offsets=False), "null pointer"),
    (dict(node=False), "null pointer"), (dict(cm=False), "null pointer"),
    (dict(k=0), "k=0"), (dict(k=5), "k=5"), (dict(M=2, k=3), "k=3"), (dict(M=0), "M=0"),
    (dict(M=257), "M=257"), (dict(B=0), "bad dimension"), (dict(rows=300, rows_pad=256), "bad dimension"),
    (dict(row0=6, rows=4), "outside"), (dict(row0=-1), "bad dimension"), (dict(with_sn=2), "with_sn"),
])
def test_seg_points_assign_argument_checks(lib_built, kw, msg):
    rc = _assign(**kw)
    assert rc == _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    assert msg in _C.last_error()


def _iou_cpu(score, seg, label, offsets, B=None, T=None, null=False):
    poff, ids, K = ops.part_table_csr(None, 50, "cpu")
    iou = np.zeros(len(label), dtype=np.float64)
    P = lambda a: None if null else a.ctypes.data  # noqa: E731
    return _C.lib().sonet_seg_iou_ragged_cpu_f32(
        P(score), seg.ctypes.data, label.ctypes.data, offsets.ctypes.data,
        len(label) if B is None else B, 50, score.shape[0] if T is None else T, poff.data_ptr(),
        ids.data_ptr(), K, iou.ctypes.data, None, None, 1), iou


def test_seg_iou_ragged_cpu_argument_checks(lib_built):
    score, seg, label, offsets = _ragged_case(3, [4, 6, 2])
    bad = _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    assert _iou_cpu(score, seg, label, offsets)[0] == 0
    assert _iou_cpu(score, seg, label, offsets, null=True)[0] == bad
    assert "null pointer" in _C.last_error()
    dec = offsets.copy()
    dec[1], dec[2] = 8, 3                      # non-monotone
    assert _iou_cpu(score, seg, label, dec)[0] == bad
    assert "decrease" in _C.last_error()
    assert _iou_cpu(score, seg, label, offsets, T=11)[0] == bad     # last offset != T
    assert "offsets must run" in _C.last_error()
    lab = label.copy()
    lab[1] = 16
    assert _iou_cpu(score, seg, lab, offsets)[0] == bad
    assert "outside the part table" in _C.last_error()


def test_seg_iou_ragged_device_argument_checks(lib_built):
    lib = _C.lib()
    bad = _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    assert lib.sonet_seg_iou_ragged_f32(None, None, None, None, 2, 50, 10, None, None, 16, None,
                                        None, None, None) == bad
    assert "null pointer" in _C.last_error()
    assert lib.sonet_seg_iou_ragged_f32(None, None, None, None, 2, 0, 10, None, None, 16, None,
                                        None, None, None) == bad
    assert "bad dimension" in _C.last_error()
    assert lib.sonet_seg_iou_ragged_f32(None, None, None, None, 0, 50, 0, None, None, 16, None,
                                        None, None, None) == 0      # nothing to do


def test_ragged_offsets_checks():
    ok = torch.tensor([0, 3, 3, 7])
    assert list(ops.ragged_offsets(ok, 7, 3)) == [0, 3, 3, 7]
    for off, T, B, msg in [(torch.tensor([0, 3, 2, 7]), 7, 3, "without decreasing"),
                           (torch.tensor([1, 3, 7]), 7, 2, "without decreasing"),
                           (torch.tensor([0, 3, 6]), 7, 2, "without decreasing"),
                           (ok, 7, 2, "B\\+1 = 3"),
                           (ok.int(), 7, 3, "int64")]:
        with pytest.raises(RuntimeError, match=msg):
            ops.ragged_offsets(off, T, B)


def _cpu_model(**over):
    opt = synth.make_opt("segmenter", batch_size=2, input_pc_num=64, **over)
    m = segmenter.Model(opt)
    m.encoder.eval()
    m.segmenter.eval()
    return m


def test_score_points_refusals(lib_built):
    pts = torch.zeros(10, 6)
    off = torch.tensor([0, 4, 10])
    m = _cpu_model()
    with pytest.raises(RuntimeError, match="not been evaluated"):
        m.score_points(pts, off)
    m._evaluated = True        # as after test_model(): the host-side checks that follow
    with pytest.raises(RuntimeError, match="B\\+1 = 3"):
        m.score_points(pts, torch.tensor([0, 10]))
    with pytest.raises(RuntimeError, match="without decreasing"):
        m.score_points(pts, torch.tensor([0, 4, 9]))
    with pytest.raises(RuntimeError, match="float32 \\[T, 6\\]"):
        m.score_points(torch.zeros(10, 3), off)
    with pytest.raises(RuntimeError, match="model's device"):
        m.score_points(pts, off)
    m.segmenter.train()
    with pytest.raises(RuntimeError, match="train mode"):
        m.score_points(pts, off)
    m.set_input(*[t for t in (torch.zeros(2, 3, 64), torch.zeros(2, 3, 64), torch.zeros(2).long(),
                              torch.zeros(2, 64).long(), torch.zeros(2, 3, 64),
                              torch.zeros(2, 64, 9).long())])
    m.segmenter.eval()
    with pytest.raises(RuntimeError, match="not been evaluated"):
        m.score_points(pts, off)
    with pytest.raises(RuntimeError, match="instance"):
        _cpu_model(normalization="instance").score_points(pts, off)
    with pytest.raises(RuntimeError, match="som_k >= 2"):
        _cpu_model(som_k=1).score_points(pts, off)


def test_device_dataset_full_clouds():
    from sonet_b200.augmentation import DeviceDataset
    rs = np.random.RandomState(0)
    sizes = [3, 5, 2, 4]
    pts = [rs.normal(size=(P, 6)).astype(np.float32) for P in sizes]
    seg = [rs.randint(0, 50, size=P) for P in sizes]
    ds = DeviceDataset(pts, np.zeros(4), [np.zeros((4, 3))] * 4, seg=seg, device="cpu")
    for index in ([1, 2], [3, 0, 3], [2]):
        p, off, s = ds.full_clouds(index)
        np.testing.assert_array_equal(p.numpy(), np.concatenate([pts[i] for i in index]))
        np.testing.assert_array_equal(off.numpy(), np.cumsum([0] + [sizes[i] for i in index]))
        np.testing.assert_array_equal(s.numpy(), np.concatenate([seg[i] for i in index]))
        assert s.dtype == torch.int64
    assert ds.full_clouds([1, 2])[0]._base is ds.data      # consecutive clouds: a view
    with pytest.raises(ValueError, match="index"):
        ds.full_clouds([4])
