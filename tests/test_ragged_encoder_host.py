"""Whole clouds of any size (networks.Encoder.forward_ragged, classifier.Model.score_clouds) without
a GPU: every refusal comes before any launch, the numpy restatement of the ragged assignment, sort
and cluster statistics meets its definitions, and the C-ABI exports and checks the new entries."""
import numpy as np
import pytest
import torch

import ragged_emu
from sonet_b200 import _C, networks, ops, synth

NEW_ENTRIES = ("sonet_som_assign_ragged_f32", "sonet_som_group_decenter_ragged_f32",
               "sonet_som_decenter_ragged_f32", "sonet_pointresnet_tc_pool_ragged_forward",
               "sonet_index_max_ragged_f32")


def _clouds(sizes, M=16, seed=0):
    rs = np.random.RandomState(seed)
    pts = rs.uniform(-1, 1, size=(sum(sizes), 6)).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    node = rs.uniform(-1, 1, size=(len(sizes), 3, M)).astype(np.float32)
    return pts, off, node


@pytest.fixture
def no_launch(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a kernel was launched")
    monkeypatch.setattr(ops, "_call", refuse)


def _encoder(**over):
    opt = synth.make_opt("classifier", **over)
    return networks.Encoder(opt).eval()


def _args(B=3, M=64, T=30, som_k=9):
    pts = torch.zeros(T, 6)
    off = torch.tensor([0, 10, 20, 30][:B + 1], dtype=torch.int64)
    node = torch.zeros(B, 3, M)
    knn = torch.zeros(B, M, som_k, dtype=torch.int64)
    return pts, off, node, knn


@pytest.mark.parametrize("case", ["train", "instance", "k5", "m257", "m_lt_k", "points_dtype",
                                  "points_cols", "node_shape", "offsets_dtype", "offsets_len",
                                  "offsets_start", "offsets_end", "offsets_decrease", "knn_shape",
                                  "knn_dtype", "device", "chunk", "empty"])
def test_refusals_before_any_launch(no_launch, case):
    enc = _encoder(normalization="instance" if case == "instance" else "batch",
                   k=5 if case == "k5" else 3)
    if case == "train":
        enc.train()
    pts, off, node, knn = _args()
    kw = {}
    err = RuntimeError
    if case == "m257":
        node, knn = torch.zeros(3, 3, 257), torch.zeros(3, 257, 9, dtype=torch.int64)
    elif case == "m_lt_k":
        node, knn = torch.zeros(3, 3, 2), torch.zeros(3, 2, 9, dtype=torch.int64)
    elif case == "points_dtype":
        pts = pts.double()
    elif case == "points_cols":
        pts = torch.zeros(30, 3)
    elif case == "node_shape":
        node = torch.zeros(3, 2, 64)
    elif case == "offsets_dtype":
        off = off.int()
    elif case == "offsets_len":
        off = off[:3]
    elif case == "offsets_start":
        off = torch.tensor([1, 10, 20, 30])
    elif case == "offsets_end":
        off = torch.tensor([0, 10, 20, 29])
    elif case == "offsets_decrease":
        off = torch.tensor([0, 15, 12, 30])
    elif case == "knn_shape":
        knn = torch.zeros(3, 64, 2, dtype=torch.int64)
    elif case == "knn_dtype":
        knn = knn.int()
    elif case == "device":
        pts = torch.zeros(30, 6, device="meta")
    elif case == "chunk":
        kw["chunk_points"] = 0
    elif case == "empty":
        off = torch.tensor([0, 10, 10, 30])
        err = ValueError
    with pytest.raises(err) as e:
        enc.forward_ragged(pts, off, node, knn, **kw)
    if case == "empty":
        assert "cloud 1" in str(e.value)


def test_valid_arguments_pass_the_checks():
    enc = _encoder()
    off = enc.check_ragged(*_args())
    assert off.tolist() == [0, 10, 20, 30]
    assert enc.check_ragged(*_args()[:3], None).tolist() == [0, 10, 20, 30]   # knn computed later


def test_score_clouds_refuses_train_mode(no_launch):
    from sonet_b200 import classifier
    opt = synth.make_opt("classifier", batch_size=3, input_pc_num=10)
    m = classifier.Model(opt)
    m.encoder.train()
    with pytest.raises(RuntimeError, match="train mode"):
        m.score_clouds(*_args()[:3])
    m.encoder.eval()
    m.classifier.eval()
    with pytest.raises(RuntimeError, match="offsets"):
        m.score_clouds(_args()[0], torch.tensor([0, 10, 20, 31]), _args()[2])


def test_chunks_are_runs_of_whole_clouds():
    off = np.array([0, 5, 7, 20, 21, 30])
    assert list(networks._ragged_chunks(off, 1)) == [(0, 1), (1, 2), (2, 3), (3, 4), (4, 5)]
    assert list(networks._ragged_chunks(off, 10)) == [(0, 2), (2, 3), (3, 5)]
    assert list(networks._ragged_chunks(off, 100)) == [(0, 5)]


@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_emulator_meets_the_definitions(k):
    sizes = [1, max(k - 1, 1), 63, 200]
    M = 16
    pts, off, node = _clouds(sizes, M, seed=k)
    idx, count = ragged_emu.assign(pts, off, node, k)
    order, ns, pos0, cm = ragged_emu.group(pts, off, idx, M, k)
    for b, P in enumerate(sizes):
        lo, hi = off[b], off[b + 1]
        blk = idx[k * lo:k * hi].reshape(k, P)
        # k distinct nearest nodes per point, ascending distance (float64 check of the fp32 order)
        d = ((pts[lo:hi, None, :3].astype(np.float64) - node[b].T[None].astype(np.float64)) ** 2).sum(2)
        for n in range(P):
            assert len(set(blk[:, n])) == k
            assert np.all(np.diff(d[n, blk[:, n]]) >= -1e-6)
        assert count[b].sum() == k * P
        assert np.array_equal(count[b], np.bincount(blk.reshape(-1), minlength=M))
        # sorted order: grouped by node, ascending stacked column inside a node, cloud's own block
        cols = order[k * lo:k * hi]
        assert sorted(cols.tolist()) == list(range(k * lo, k * hi))
        keys = ns[k * lo:k * hi]
        assert np.all(np.diff(keys) >= 0) and np.all(keys // M == b)
        same = np.diff(keys) == 0
        assert np.all(np.diff(cols)[same] > 0)
        assert order[pos0[b]] == k * lo                       # pos0: sorted position of copy 0
        # cluster means: the mean of the node's copies (float64), empty nodes 0
        x64 = pts[lo:hi, :3].astype(np.float64)
        for m in range(M):
            pts_m = np.tile(np.arange(P), k)[blk.reshape(-1) == m]
            want = x64[pts_m].sum(0) / (len(pts_m) + 1e-5)
            assert np.allclose(cm[b, :, m], want, rtol=1e-5, atol=1e-6)


def test_emulator_clouds_are_independent():
    """A cloud's statistics depend only on its own points and nodes: the same cloud alone or
    between others, at any position, gives the same bits."""
    M, k = 9, 3
    pts, off, node = _clouds([40, 75, 3], M, seed=7)
    idx, _ = ragged_emu.assign(pts, off, node, k)
    _, _, _, cm = ragged_emu.group(pts, off, idx, M, k)
    alone = pts[40:115]
    idx1, _ = ragged_emu.assign(alone, np.array([0, 75]), node[1:2], k)
    _, _, _, cm1 = ragged_emu.group(alone, np.array([0, 75]), idx1, M, k)
    assert np.array_equal(idx1, idx[3 * 40:3 * 115])
    assert np.array_equal(cm1[0], cm[1])


def test_cabi_has_the_ragged_entries(lib_built):
    import ctypes
    h = ctypes.CDLL(lib_built)
    for n in NEW_ENTRIES:
        assert hasattr(h, n) and n in _C._SIGNATURES, n
    assert not any(n in _C.ACT_ENTRIES or n in _C.F16_ENTRIES for n in NEW_ENTRIES)


def test_cabi_ragged_argument_checks(lib_built):
    lib = _C.lib()
    n = None
    assert lib.sonet_som_assign_ragged_f32(n, 10, n, 1, n, 257, 3, n, n, n, n) == -1
    assert "M=257" in _C.last_error()
    assert lib.sonet_som_assign_ragged_f32(n, 10, n, 1, n, 64, 5, n, n, n, n) == -1
    assert "k=5" in _C.last_error()
    assert lib.sonet_som_assign_ragged_f32(n, 10, n, 1, n, 64, 3, n, n, n, n) == -1
    assert "null" in _C.last_error()
    assert lib.sonet_som_group_decenter_ragged_f32(n, 1 << 24, n, 1, 64, 1, 0, n, n, n, n, n, n) == -1
    assert "24 bits" in _C.last_error()
    assert lib.sonet_som_decenter_ragged_f32(n, 10, n, 1, 64, 3, 2, n, n, n, n) == -1
    assert lib.sonet_index_max_ragged_f32(n, 384, 10, n, n, 1, 10, 64, 3, n, n, n) == -1
    assert "stride" in _C.last_error()
    assert lib.sonet_index_max_ragged_f32(n, 384, 30, n, n, 0, 10, 64, 3, n, n, n) == 0   # no cloud
    assert lib.sonet_pointresnet_tc_pool_ragged_forward(n, 6, 256, n, n, n, n, 2, 64, 0, 0, n, n,
                                                        n) == -1
    assert "activation code 0" in _C.last_error()
    assert lib.sonet_pointresnet_tc_pool_ragged_forward(n, 6, 256, n, n, n, n, 2, 300, 1, 0, n, n,
                                                        n) == -1
