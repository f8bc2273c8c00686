"""SHREC'16 retrieval ranking on the H100: the sm_90a kernels (csrc/retrieval.cu) against the files
the reference's shrec16/test.py wrote (tests/golden/retrieval.npz) and bit for bit against the host
entry, given vs argmax labels, out-of-range labels, determinism, CUDA-graph replay, no host sync,
and RetrievalBank."""
import numpy as np
import pytest
import torch

from _retrieval_check import canonical, check_case, expected_files
from helpers import golden

pytestmark = pytest.mark.gpu

G = golden("retrieval")
DEV = "cuda:0"


def as_bits(t):
    t = t.cpu()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def assert_same(a, b):
    for x, y in zip(a, b):
        assert torch.equal(as_bits(x), as_bits(y))


def make_case(Q, D, kind, seed):
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(Q, D, generator=g)
    L = max(D, 2)
    if kind == "single":
        lab = torch.zeros(Q, dtype=torch.int64)
    else:
        z = torch.from_numpy(np.random.RandomState(seed).zipf(1.3, size=Q) - 1).long()
        lab = z % L
        if kind == "empty":                     # labels only in the upper half: empty classes
            lab = lab % max(1, L // 2) + L // 2
    if kind == "nan":
        f[::97, D // 2] = float("nan")
        f[1::89, 0] = float("inf")
    dup = torch.arange(0, Q, 13)
    f[dup] = f[dup // 2]                        # duplicate rows: distance-0 ties
    if D <= 3:
        f = torch.round(f * 8) / 8              # many exact distance ties
    return f, lab, L


@pytest.mark.parametrize("tag", ["quant", "float"])
def test_kernel_matches_reference_files(tag):
    from sonet_b200 import ops
    f = torch.from_numpy(G[tag + "_score"]).to(DEV)
    idx, dist, count, label = ops.retrieval_rank(f, k=1000)
    torch.cuda.synchronize()
    assert np.array_equal(label.cpu().numpy(),
                          torch.max(torch.from_numpy(G[tag + "_score"]), 1)[1].numpy())
    check_case(G, tag, idx.cpu().numpy(), dist.cpu().numpy(), count.cpu().numpy())


def test_write_from_device_matches_reference_files(tmp_path):
    from sonet_b200 import retrieval
    res = retrieval.rank_same_label(torch.from_numpy(G["quant_score"]).to(DEV),
                                    torch.from_numpy(G["quant_ids"]))
    res.write(str(tmp_path))
    for name, data in expected_files(G, "quant").items():
        cut = data.count(b"\n") == 1000
        assert canonical((tmp_path / name).read_bytes(), cut) == canonical(data, cut), name


GRID = [  # (Q, D, k, labels)
    (1, 3, 1, "zipf"), (1, 1024, 4096, "single"),
    (777, 3, 1000, "zipf"), (777, 55, 1, "single"), (777, 55, 4096, "empty"),
    (777, 1024, 1000, "nan"), (777, 3, 4096, "single"),
    (10265, 55, 1000, "zipf"), (10265, 3, 4096, "single"), (10265, 1024, 1, "zipf"),
    (10265, 55, 1000, "single"), (10265, 55, 4096, "nan"), (10265, 1024, 1000, "empty"),
]


@pytest.mark.parametrize("Q,D,k,kind", GRID)
@pytest.mark.parametrize("given", [False, True])
def test_kernel_equals_host_entry(Q, D, k, kind, given):
    from sonet_b200 import ops
    f, lab, L = make_case(Q, D, kind, seed=Q + D + k)
    if given:
        args = (lab, L)
    else:
        args = (None, None)
    host = ops.retrieval_rank(f, *args, k=k)
    dev = ops.retrieval_rank(f.to(DEV), None if lab is None or not given else lab.to(DEV),
                             args[1], k=k)
    assert_same(dev, host)
    count = host[2]
    assert int(count.min()) >= 1
    if kind == "single" and given:
        assert int(count.max()) == min(Q, k)


def test_given_labels_equal_argmax_labels():
    from sonet_b200 import ops
    f, _, _ = make_case(3000, 55, "nan", seed=11)
    f = f.to(DEV)
    a = ops.retrieval_rank(f, k=500)
    b = ops.retrieval_rank(f, a[3].clone(), 55, k=500)
    assert_same(a, b)


def test_out_of_range_labels_are_flagged_then_raised():
    from sonet_b200 import ops, retrieval
    f, lab, L = make_case(600, 55, "zipf", seed=3)
    lab[[5, 77, 300]] = torch.tensor([-1, L, 1 << 40])
    dev = ops.retrieval_rank(f.to(DEV), lab.to(DEV), L, k=100)
    host = ops.retrieval_rank(f, lab, L, k=100)
    assert_same(dev, host)
    count = dev[2].cpu()
    assert count[[5, 77, 300]].tolist() == [-1, -1, -1] and int(count.min()) == -1
    assert bool((dev[0].cpu() != 5).all() & (dev[0].cpu() != 77).all())   # nobody's candidate
    res = retrieval.rank_same_label(f.to(DEV), torch.arange(600), lab.to(DEV), 100, L)
    with pytest.raises(RuntimeError, match="outside"):
        res.write("/nonexistent")


def test_repeated_calls_are_bit_identical():
    from sonet_b200 import ops
    f, lab, L = make_case(10265, 55, "zipf", seed=7)
    f = f.to(DEV)
    first = ops.retrieval_rank(f, k=1000)
    for _ in range(3):
        assert_same(ops.retrieval_rank(f, k=1000), first)


def test_cuda_graph_capture_and_replay():
    from sonet_b200 import ops
    f0, _, _ = make_case(2000, 55, "zipf", seed=1)
    f1, _, _ = make_case(2000, 55, "single", seed=2)
    static = f0.to(DEV)
    ops.retrieval_rank(static, k=1000)                      # warm up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            out = ops.retrieval_rank(static, k=1000)
    torch.cuda.current_stream().wait_stream(s)
    for f in (f1, f0):
        static.copy_(f.to(DEV))
        graph.replay()
        torch.cuda.synchronize()
        assert_same(out, ops.retrieval_rank(f, k=1000))


def test_no_host_sync():
    from sonet_b200 import ops, retrieval
    f, lab, L = make_case(5000, 55, "zipf", seed=4)
    f, lab = f.to(DEV), lab.to(DEV)
    ids = torch.arange(5000, device=DEV)
    ops.retrieval_rank(f, k=1000)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        ops.retrieval_rank(f, k=1000)
        ops.retrieval_rank(f, lab, L, k=4096)
        bank = retrieval.RetrievalBank()
        bank.update(f[:3000], ids[:3000])
        bank.update(f[3000:], ids[3000:])
        res = bank.rank()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert res.idx.shape == (5000, 1000)


def test_bank_in_batches_equals_one_call():
    from sonet_b200 import retrieval
    f, _, _ = make_case(1234, 55, "nan", seed=9)
    ids = torch.from_numpy(np.random.RandomState(0).choice(10 ** 7, 1234, replace=False))
    bank = retrieval.RetrievalBank()
    for a in range(0, 1234, 64):                             # the last batch is partial
        bank.update(f[a:a + 64].to(DEV), ids[a:a + 64])
    assert len(bank) == 1234
    got = bank.rank(max_results=1000)
    want = retrieval.rank_same_label(f.to(DEV), ids)
    assert_same((got.idx, got.dist, got.count, got.label, got.model_ids),
                (want.idx, want.dist, want.count, want.label, want.model_ids))
    assert got.files() == want.files()
