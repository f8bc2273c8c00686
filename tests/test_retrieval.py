"""SHREC'16 retrieval ranking without a GPU: the host entry (csrc/retrieval.cu) against the files the
reference's shrec16/test.py wrote (tests/golden/retrieval.npz), the native formatter against
np.savetxt, RetrievalResult.write(), argument validation and thread-count independence."""
import ctypes

import numpy as np
import pytest
import torch

from _retrieval_check import canonical, check_case, expected_files, savetxt_bytes
from helpers import golden

G = golden("retrieval")


def host_rank(tag, k=1000):
    f = torch.from_numpy(G[tag + "_score"])
    from sonet_b200 import ops
    return [t.numpy() for t in ops.retrieval_rank(f, k=k)]


@pytest.mark.parametrize("tag", ["quant", "float"])
def test_host_entry_matches_reference_files(tag):
    idx, dist, count, label = host_rank(tag)
    assert np.array_equal(label, torch.max(torch.from_numpy(G[tag + "_score"]), 1)[1].numpy())
    cut = check_case(G, tag, idx, dist, count)
    if tag == "quant":
        assert cut > 0          # the 1000-row cut fell inside a tie run at least once


def test_golden_covers_the_issue_cases():
    lab = torch.max(torch.from_numpy(G["quant_score"]), 1)[1].numpy()
    sizes = np.bincount(lab, minlength=55)
    assert sizes.max() > 1000 and (sizes == 1).any()
    ids = G["quant_ids"]
    assert 0 in ids and (ids >= 10 ** 6).any() and len(set(ids.tolist())) < len(ids)
    assert np.isnan(G["float_score"]).any()
    for tag in ("quant", "float"):
        assert len(G[tag + "_ids"]) % int(G[tag + "_batch"]) != 0     # final partial batch
    assert str(G["fmt"]) == "%06d %f" and str(G["delimiter"]) == " "


def test_write_matches_reference_files(tmp_path):
    from sonet_b200 import retrieval
    f = torch.from_numpy(G["quant_score"])
    res = retrieval.rank_same_label(f, torch.from_numpy(G["quant_ids"]))
    files = res.files()
    assert len(files) == len(set(G["quant_ids"].tolist()))
    want = expected_files(G, "quant")
    assert len(want) > 100
    for name, data in want.items():
        cut = data.count(b"\n") == 1000
        assert canonical(files[name], cut) == canonical(data, cut), name
    res.write(str(tmp_path))
    for name in want:
        assert (tmp_path / name).read_bytes() == files[name]
    assert len(list(tmp_path.iterdir())) == len(files)


def _format_one(ids, idx, dist, count):
    from sonet_b200 import ops
    text, off = ops.retrieval_format(torch.as_tensor(ids), torch.as_tensor(idx),
                                     torch.as_tensor(dist), torch.as_tensor(count))
    return [text[off[q]:off[q + 1]] for q in range(len(count))]


def test_formatter_matches_savetxt():
    rs = np.random.RandomState(3)
    ids = np.array([0, 5, -5, -123456, 1234567, 2 ** 53 + 1, 2 ** 62 + 12345, 2 ** 63 - 1,
                    -2 ** 63, 999999, 1000000, 42], dtype=np.int64)
    vals = [0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1e-9, 4.9999997e-7, 5e-7, 5.0000006e-7,
            1.5e-6, 0.5, 0.1234565, 2.5e-6, 3.4e38, -3.4e38, 1e10, 4294967295.0, 4294967296.0,
            123456.79, -1.25, 7.0, 1.0 - 2 ** -24, 0.9999995, 2 ** -26, 2 ** -27, 1e-45]
    vals += list(rs.uniform(0, 20, 40)) + list(10.0 ** rs.uniform(-8, 12, 40))
    vals = np.array(vals, dtype=np.float32)
    Q, k = len(ids), 8
    idx = rs.randint(0, Q, size=(Q, k)).astype(np.int64)
    dist = rs.choice(vals, size=(Q, k)).astype(np.float32)
    count = rs.randint(0, k + 1, size=Q).astype(np.int32)
    count[0], count[1] = k, 1
    texts = _format_one(ids, idx, dist, count)
    for q in range(Q):
        n = count[q]
        rows = np.transpose(np.vstack((ids[idx[q, :n]], dist[q, :n])))
        want = savetxt_bytes(rows) if n else b""
        assert texts[q] == want, (q, texts[q][:200], want[:200])
    # every special value once, in one file
    allv = np.resize(vals, (len(vals) + k - 1) // k * k).reshape(-1, k)
    Q2 = allv.shape[0]
    ids2 = np.resize(ids, Q2)
    idx2 = np.tile(np.arange(k) % Q2, (Q2, 1)).astype(np.int64)
    got = _format_one(ids2, idx2, allv, np.full(Q2, k, np.int32))
    for q in range(Q2):
        rows = np.transpose(np.vstack((ids2[idx2[q]], allv[q])))
        assert got[q] == savetxt_bytes(rows), q
    assert b"-nan" not in b"".join(got)


def test_formatter_rejects_bad_rows():
    from sonet_b200 import _C
    lib = _C.lib()
    ids = torch.arange(3, dtype=torch.int64)
    idx = torch.zeros(3, 2, dtype=torch.int64)
    dist = torch.zeros(3, 2)
    off = torch.zeros(4, dtype=torch.int64)
    for count, bad_idx in (([1, 3, 1], None), ([1, -1, 1], None), ([1, 1, 1], 3), ([1, 1, 1], -1)):
        ix = idx.clone()
        if bad_idx is not None:
            ix[1, 0] = bad_idx
        c = torch.tensor(count, dtype=torch.int32)
        assert lib.sonet_retrieval_format_cpu(ids.data_ptr(), ix.data_ptr(), dist.data_ptr(),
                                              c.data_ptr(), 3, 2, off.data_ptr(), None, 1) == -1
    c = torch.ones(3, dtype=torch.int32)
    args = (ids.data_ptr(), idx.data_ptr(), dist.data_ptr(), c.data_ptr(), 3, 2, off.data_ptr())
    total = lib.sonet_retrieval_format_cpu(*args, None, 1)
    assert total == 3 * len(b"000000 0.000000\n") and off.tolist() == [0, 16, 32, 48]
    buf = ctypes.create_string_buffer(total)
    assert lib.sonet_retrieval_format_cpu(*args, ctypes.addressof(buf), 2) == total
    assert buf.raw == b"000000 0.000000\n" * 3
    off[2] += 1                                          # offsets not from the size query
    assert lib.sonet_retrieval_format_cpu(*args, ctypes.addressof(buf), 1) == -1
    assert "offsets" in _C.last_error()


def test_argument_validation():
    from sonet_b200 import _C, ops, retrieval
    lib = _C.lib()
    f = torch.zeros(4, 3)
    for kw in (dict(k=0), dict(k=4097), dict(num_labels=0), dict(num_labels=4097)):
        with pytest.raises(RuntimeError):
            ops.retrieval_rank(f, **kw)
    for bad in (torch.zeros(4, 1025), torch.zeros(4, 0), torch.zeros(4, 3, dtype=torch.float64),
                torch.zeros(4), torch.zeros(3, 4).t()):
        with pytest.raises(RuntimeError):
            ops.retrieval_rank(bad)
    with pytest.raises(RuntimeError):
        ops.retrieval_rank(f, label=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(RuntimeError):
        ops.retrieval_rank(f, label=torch.zeros(4, dtype=torch.int32))
    assert lib.sonet_retrieval_scratch_bytes(1 << 20, 8, 4, 4096) == -1       # Q*k >= 2^31
    assert "2^31" in _C.last_error()
    assert lib.sonet_retrieval_scratch_bytes(524287, 8, 4, 4096) > 0
    for Q, D, L, k in ((-1, 3, 1, 1), (1, 0, 1, 1), (1, 1025, 1, 1), (1, 3, 0, 1), (1, 3, 4097, 1),
                       (1, 3, 1, 0), (1, 3, 1, 4097)):
        assert lib.sonet_retrieval_scratch_bytes(Q, D, L, k) == -1
        assert lib.sonet_retrieval_rank_f32(None, None, Q, D, L, k, None, 0, None, None, None, None,
                                            None) == -1
        assert lib.sonet_retrieval_rank_cpu_f32(None, None, Q, D, L, k, None, None, None, None,
                                                1) == -1
    assert lib.sonet_retrieval_rank_f32(None, None, 4, 3, 3, 2, None, 0, None, None, None, None,
                                        None) == -1
    assert "null" in _C.last_error()
    assert lib.sonet_retrieval_rank_cpu_f32(None, None, 4, 3, 3, 2, None, None, None, None, 0) == -1
    assert lib.sonet_retrieval_rank_f32(None, None, 0, 3, 3, 2, None, 0, None, None, None, None,
                                        None) == 0                         # empty: no-op
    # a label outside [0, L) is flagged, excluded, and raised when read
    lab = torch.tensor([0, 1, 5, -1], dtype=torch.int64)
    idx, dist, count, out = ops.retrieval_rank(torch.arange(12.0).view(4, 3), lab, 3, k=4)
    assert count.tolist() == [1, 1, -1, -1] and out is lab
    assert idx[2].tolist() == [-1] * 4 and bool(torch.isnan(dist[3]).all())
    res = retrieval.rank_same_label(torch.arange(12.0).view(4, 3), torch.arange(4), lab, 4, 3)
    with pytest.raises(RuntimeError, match="outside"):
        res.files()
    with pytest.raises(RuntimeError):
        retrieval.RetrievalBank().rank()


def test_thread_count_does_not_change_results():
    from sonet_b200 import ops
    rs = np.random.RandomState(5)
    Q, D = 2500, 55
    f = torch.from_numpy(rs.normal(size=(Q, D)).astype(np.float32))
    lab = torch.from_numpy((rs.zipf(1.5, size=Q) - 1) % 7).long()
    lab[:1500] = 0
    f[3, 4] = float("nan")
    one = ops.retrieval_rank(f, lab, 7, k=1000, threads=1)
    many = ops.retrieval_rank(f, lab, 7, k=1000, threads=8)
    for a, b in zip(one, many):
        assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                           b.view(torch.int32) if b.dtype == torch.float32 else b)
    argmax = ops.retrieval_rank(f, None, None, k=300, threads=3)
    given = ops.retrieval_rank(f, argmax[3].clone(), D, k=300, threads=5)
    for a, b in zip(argmax[:3], given[:3]):
        assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                           b.view(torch.int32) if b.dtype == torch.float32 else b)
