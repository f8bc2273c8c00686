"""Training on whole clouds (classifier.Model.optimize_clouds, networks.Encoder.forward_ragged_train)
without a GPU: every refusal fires before any launch, the four new C-ABI entries are bound from the
header and refuse bad arguments before touching a device, and a numpy restatement of the ragged
BatchNorm fold matches the fp64 statistics of the data and, at equal sizes, the dense fold."""
import ctypes

import numpy as np
import pytest
import torch

from sonet_b200 import _C, classifier, ops, synth, train_ops

ENTRIES = {
    "sonet_bn_cloud_partials_ragged_f32": 14,
    "sonet_bn_ragged_forward_f32": 15,
    "sonet_bn_ragged_backward_f32": 16,
    "sonet_index_max_ragged_backward_f32": 9,
    "sonet_augment_ragged_f32": 21,
}


@pytest.fixture
def no_launch(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(ops, "_call", refuse)


# ---- C-ABI ----------------------------------------------------------------------------------------
def test_cabi_has_the_entries(lib_built):
    h = ctypes.CDLL(lib_built)
    for name, n in ENTRIES.items():
        assert hasattr(h, name) and name in _C._SIGNATURES, name
        assert len(_C._SIGNATURES[name]) == n, name
        assert _C._RESTYPE[name] is ctypes.c_int
    sig = _C._SIGNATURES["sonet_bn_cloud_partials_ragged_f32"]
    assert sig[6] is ctypes.c_int and sig[7] is ctypes.c_longlong and sig[8] is ctypes.c_void_p
    assert sig[9] is ctypes.c_int
    sig = _C._SIGNATURES["sonet_augment_ragged_f32"]
    assert sig[1] is ctypes.c_longlong and sig[11] is ctypes.c_double and sig[17] is ctypes.c_ulonglong


P = 0x1000    # a non-null pointer the checks never dereference


def _partials(**kw):
    a = dict(x=P, dy=None, mean=None, invstd=None, gamma=None, beta=None, C=4, ld=10, cols=P, B=2,
             act=0, backward=0, rec=P)
    a.update(kw)
    return _C.lib().sonet_bn_cloud_partials_ragged_f32(*a.values(), None)


def _forward(**kw):
    a = dict(rec=P, cols=P, B=2, x=P, gamma=None, beta=None, C=4, L=10, eps=1e-5, act=1, y=P, mean=P,
             var=P, invstd=P)
    a.update(kw)
    return _C.lib().sonet_bn_ragged_forward_f32(*a.values(), None)


def _backward(**kw):
    a = dict(rec=P, cols=P, B=2, dy=P, x=P, mean=P, invstd=P, gamma=None, beta=None, C=4, L=10, act=1,
             dx=P, dgamma=P, dbeta=P)
    a.update(kw)
    return _C.lib().sonet_bn_ragged_backward_f32(*a.values(), None)


def _pool(**kw):
    a = dict(go=P, idx=P, cols=P, B=2, C=4, M=64, ld=10, grad=P)
    a.update(kw)
    return _C.lib().sonet_index_max_ragged_backward_f32(*a.values(), None)


def _augment(**kw):
    a = dict(points=P, T=10, ld=6, offsets=P, B=2, som=P, M=4, rot1=None, rot2=None, scale=None,
             shift=None, s0=0.01, c0=0.05, s1=0.01, c1=0.05, s2=0.04, c2=0.1, seed=0, out=P, som_out=P)
    a.update(kw)
    return _C.lib().sonet_augment_ragged_f32(*a.values(), None)


BAD = [
    (_partials, dict(B=0)), (_partials, dict(B=65536)), (_partials, dict(C=0)),
    (_partials, dict(C=65536)), (_partials, dict(ld=0)), (_partials, dict(ld=1 << 31)),
    (_partials, dict(act=7)), (_partials, dict(x=None)), (_partials, dict(cols=None)),
    (_partials, dict(rec=None)), (_partials, dict(backward=1)),
    (_forward, dict(B=0)), (_forward, dict(C=65536)), (_forward, dict(L=0)),
    (_forward, dict(L=1 << 31)), (_forward, dict(act=-1)), (_forward, dict(rec=None)),
    (_forward, dict(cols=None)), (_forward, dict(y=None)),
    (_backward, dict(B=65536)), (_backward, dict(C=0)), (_backward, dict(L=1 << 31)),
    (_backward, dict(act=3)), (_backward, dict(dy=None)), (_backward, dict(dgamma=None)),
    (_pool, dict(B=0)), (_pool, dict(C=0)), (_pool, dict(M=0)), (_pool, dict(M=257)),
    (_pool, dict(ld=0)), (_pool, dict(ld=1 << 31)), (_pool, dict(grad=None)), (_pool, dict(cols=None)),
    (_augment, dict(B=0)), (_augment, dict(B=65536)), (_augment, dict(T=-1)),
    (_augment, dict(T=1 << 31)), (_augment, dict(ld=5)), (_augment, dict(offsets=None)),
    (_augment, dict(out=None)), (_augment, dict(som_out=None)), (_augment, dict(c0=0.0)),
    (_augment, dict(c2=-1.0)),
]


@pytest.mark.parametrize("fn,kw", BAD, ids=["%s-%s" % (f.__name__, "-".join("%s=%s" % i for i in k.items()))
                                              for f, k in BAD])
def test_cabi_refuses_bad_arguments(lib_built, fn, kw):
    assert fn(**kw) == _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    assert "ragged" in _C.lib().sonet_last_error_string().decode()


def test_cabi_refuses_aliasing_with_a_wide_row(lib_built):
    assert _augment(ld=7, out=P) == _C.CONSTANTS["SONET_ERR_BAD_ARG"]


# ---- Python refusals -------------------------------------------------------------------------------
def _model(**over):
    opt = synth.make_opt("classifier", batch_size=2, input_pc_num=64, **over)
    return classifier.Model(opt)


def _batch(sizes=(5, 7), M=64, som_k=9):
    T = sum(sizes)
    off = torch.tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64)
    return (torch.zeros(T, 6), off, torch.zeros(len(sizes), dtype=torch.int64),
            torch.zeros(len(sizes), 3, M), torch.zeros(len(sizes), M, max(som_k, 1), dtype=torch.int64))


def _refused(m, args, exc=RuntimeError, match=None):
    with pytest.raises(exc, match=match):
        m.optimize_clouds(*args)


def test_refusals_of_check_ragged(no_launch):
    m = _model()
    pts, off, lab, node, knn = _batch()
    _refused(m, (pts, torch.tensor([0, 5, 5, 12]), torch.zeros(3, dtype=torch.int64),
                 torch.zeros(3, 3, 64), None), ValueError, "no points")
    _refused(m, (pts, torch.tensor([0, 7, 5]), lab, node, knn), match="offsets")
    _refused(m, (pts, torch.tensor([0, 5, 11]), lab, node, knn), match="offsets")
    _refused(m, (pts.double(), off, lab, node, knn), match="points")
    _refused(m, (pts, off.int(), lab, node, knn), match="offsets")
    _refused(m, (pts[:, :3].contiguous(), off, lab, node, knn), match=r"\[T, 6\]")
    _refused(m, (pts, off, lab, torch.zeros(2, 3, 289), torch.zeros(2, 289, 9, dtype=torch.int64)),
             match="M=289")
    _refused(m, (pts, off, lab, node, knn[:, :, :3]), match="node_knn_I")
    _refused(_model(k=5), (pts, off, lab, node, knn), match="k=5")
    _refused(_model(k=0), (pts, off, lab, node, knn), match="k=0")


def test_refuses_a_cloud_of_2_24_points(no_launch):
    m = _model()
    T = 1 << 24
    pts = torch.zeros(1, 6).expand(T + 3, 6)
    off = torch.tensor([0, 3, T + 3])
    _refused(m, (pts, off, torch.zeros(2, dtype=torch.int64), torch.zeros(2, 3, 64), None),
             match="more than")


def test_refuses_2_31_stacked_columns(no_launch):
    m = _model(k=4)
    T = 1 << 29
    per = (1 << 24) - 1
    off = list(range(0, T, per)) + [T]
    B = len(off) - 1
    pts = torch.zeros(1, 6).expand(T, 6)
    _refused(m, (pts, torch.tensor(off), torch.zeros(B, dtype=torch.int64), torch.zeros(B, 3, 64),
                 None), match="2\\^31")


def test_refusals_of_the_train_step(no_launch, monkeypatch):
    args = _batch()
    _refused(_model(normalization="instance"), args, match="instance")
    _refused(_model(random_pc_dropout_lower_limit=0.5), args, match="dropout")
    monkeypatch.setattr(train_ops, "ENABLED", False)
    _refused(_model(), args, match="ENABLED")
    monkeypatch.setattr(train_ops, "ENABLED", True)
    monkeypatch.setattr(train_ops, "EXCHANGE", object())
    _refused(_model(), args, match="DataParallelTraining")


def test_refusals_of_the_label(no_launch):
    m = _model()
    pts, off, lab, node, knn = _batch()
    _refused(m, (pts, off, lab.int(), node, knn), match="label")
    _refused(m, (pts, off, lab[:1], node, knn), match="label")
    _refused(m, (pts, off, [0, 1], node, knn), match="label")
    _refused(m, (pts, off, torch.tensor([0, 40]), node, knn), match=r"\[0, 40\)")
    _refused(m, (pts, off, torch.tensor([-1, 0]), node, knn), match=r"\[0, 40\)")


def test_forward_ragged_train_refuses_eval_mode(no_launch):
    m = _model()
    m.encoder.eval()
    pts, off, _, node, knn = _batch()
    with pytest.raises(RuntimeError, match="eval mode"):
        m.encoder.forward_ragged_train(pts, off, node, knn)


def test_norm_act_train_refuses_cols_with_instance_norm_or_an_exchange(no_launch, monkeypatch):
    y0 = torch.zeros(1, 4, 10)
    cols = torch.tensor([0, 4, 10])
    inorm = torch.nn.InstanceNorm1d(4, affine=True)
    with pytest.raises(RuntimeError, match="instance"):
        train_ops.norm_act_train(y0, inorm, "relu", cols=cols)
    monkeypatch.setattr(train_ops, "EXCHANGE", object())
    with pytest.raises(RuntimeError, match="exchange"):
        train_ops.norm_act_train(y0, None, "relu", cols=cols)


# ---- the fold, restated -----------------------------------------------------------------------------
def _records(x, cols):
    """The forward records {pivot, sum d, sum d^2} per (cloud, channel) in fp64 (sequential sums:
    the restatement of the fold only, not of the kernels' summation order)."""
    C = x.shape[0]
    rec = np.empty((len(cols) - 1, C, 3))
    for b in range(len(cols) - 1):
        seg = x[:, cols[b]:cols[b + 1]].astype(np.float64)
        d = seg - seg[:, :1]
        rec[b, :, 0], rec[b, :, 1], rec[b, :, 2] = seg[:, 0], d.sum(1), (d * d).sum(1)
    return rec


def _fold(rec, counts, n):
    """sonet_bn_ragged_forward_f32's fold: record b with its own count onto cloud 0's pivot."""
    p = rec[0, :, 0]
    s1 = np.zeros_like(p)
    s2 = np.zeros_like(p)
    for b in range(rec.shape[0]):
        nb = float(counts[b])
        s = rec[b, :, 0] - p
        s1 = s1 + (rec[b, :, 1] + nb * s)
        s2 = s2 + (rec[b, :, 2] + 2.0 * s * rec[b, :, 1] + nb * s * s)
    md = s1 / n
    v = np.maximum(s2 / n - md * md, 0.0)
    return p + md, v


@pytest.mark.parametrize("sizes", [[1], [1025, 3], [1, 40, 1025, 2, 3000, 7], [64] * 9])
def test_fold_restatement_gives_the_statistics(sizes):
    rs = np.random.RandomState(len(sizes))
    L = sum(sizes)
    x = (rs.normal(size=(5, L)) * 2 + 0.5).astype(np.float32)
    x[0] += 3e3
    cols = np.concatenate([[0], np.cumsum(sizes)])
    mean, var = _fold(_records(x, cols), np.diff(cols), float(L))
    xd = x.astype(np.float64)
    np.testing.assert_allclose(mean, xd.mean(1), rtol=1e-12)
    np.testing.assert_allclose(var, xd.var(1), rtol=1e-9, atol=1e-12)


def test_fold_at_equal_sizes_is_the_dense_fold():
    """With B clouds of P values each cloud stands for P values and n = B*P: the dense fold's
    operations on the same records, so the same bits."""
    rs = np.random.RandomState(3)
    B, P = 6, 37
    x = rs.normal(size=(4, B * P)).astype(np.float32)
    rec = _records(x, np.arange(0, B * P + 1, P))
    mean, var = _fold(rec, [P] * B, float(B) * P)
    p = rec[0, :, 0]
    s1 = np.zeros_like(p)
    s2 = np.zeros_like(p)
    nb = float(P)
    for b in range(B):
        s = rec[b, :, 0] - p
        s1 = s1 + (rec[b, :, 1] + nb * s)
        s2 = s2 + (rec[b, :, 2] + 2.0 * s * rec[b, :, 1] + nb * s * s)
    md = s1 / (float(B) * P)
    assert np.array_equal(mean, p + md)
    assert np.array_equal(var, np.maximum(s2 / (float(B) * P) - md * md, 0.0))
