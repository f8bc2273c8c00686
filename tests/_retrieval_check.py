"""Comparison rules of the retrieval ranking against the files the reference's shrec16/test.py wrote
(tests/golden/retrieval.npz), shared by the host-entry and the kernel tests.

quant (exact distances): distances bit-equal; ids equal except inside runs of equal distance, which
are compared as sets. A run cut by the 1000-row limit must hold the lowest positions of its tie run.
float (unquantised): distances within 4 ulp; ids equal except among golden neighbours within 4 ulp
of each other (chained), compared as sets."""
import io

import numpy as np
import torch

ULP = 4


def bits(x):
    x = np.asarray(x, dtype=np.float32).copy()
    x[np.isnan(x)] = np.float32("nan")
    return np.abs(x).view(np.int32).astype(np.int64) * np.sign(np.where(np.signbit(x), -1, 1))


def runs(gd, exact):
    """[a, b) runs of the golden distances that may appear in any order."""
    out, a = [], 0
    b = bits(gd)
    for i in range(1, len(gd) + 1):
        if i == len(gd) or not ((b[i] == b[i - 1]) if exact else abs(b[i] - b[i - 1]) <= ULP):
            out.append((a, i))
            a = i
    return out


def pred_labels(score):
    return torch.max(torch.from_numpy(score), 1)[1].numpy()


def fp64_dist(score, q, members):
    d = (score[q][None, :] - score[members]).astype(np.float64)
    return np.sqrt((d * d).sum(1)).astype(np.float32)


def check_case(G, tag, idx, dist, count):
    """idx/dist/count: numpy results of ranking G[tag+'_score'] with the argmax labels, k=1000."""
    exact = tag == "quant"
    score, ids = G[tag + "_score"], G[tag + "_ids"]
    lab = pred_labels(score)
    off = G[tag + "_file_off"]
    rows_all = G[tag + "_rows"]
    cut_runs = 0
    for f, q in enumerate(G[tag + "_file_q"]):
        rows = rows_all[off[f]:off[f + 1]]
        n = len(rows)
        assert count[q] == n, (tag, q, count[q], n)
        gd = rows[:, 1].astype(np.float32)
        assert np.array_equal(gd.astype(np.float64), rows[:, 1], equal_nan=True)
        od, oi = dist[q, :n], idx[q, :n]
        if exact:
            assert np.array_equal(bits(od), bits(gd)), (tag, q)
        else:
            assert np.all(np.abs(bits(od) - bits(gd)) <= ULP), (tag, q)
        gi = rows[:, 0]
        members = np.nonzero(lab == lab[q])[0]
        for a, b in runs(gd, exact):
            if b == n and len(members) > n and exact:      # the run straddling the cut
                d = fp64_dist(score, q, members)
                ties = members[bits(d) == bits(gd[a:a + 1])[0]]
                assert np.array_equal(oi[a:b], ties[:b - a]), (tag, q)
                assert set(gi[a:b]) <= set(ids[ties].astype(np.float64))
                cut_runs += 1
            else:
                assert sorted(ids[oi[a:b]].astype(np.float64)) == sorted(gi[a:b]), (tag, q, a, b)
        assert np.all(idx[q, n:] == -1) and np.all(np.isnan(dist[q, n:]))
    return cut_runs


def savetxt_bytes(rows, fmt="%06d %f"):
    b = io.BytesIO()
    np.savetxt(b, rows, fmt=fmt, delimiter=" ")
    return b.getvalue()


def canonical(text, cut=False):
    """Lines sorted within runs of equal printed distance. With cut (the file stops at the row
    limit inside a larger group), the ids of the last run are masked: which members of a tie run
    straddling the cut the reference kept depends on its unstable sort; check_case holds ours to
    the lowest positions."""
    lines = text.split(b"\n")
    assert lines[-1] == b""
    lines = lines[:-1]
    out, a = [], 0
    for i in range(1, len(lines) + 1):
        if i == len(lines) or lines[i].split(b" ")[1] != lines[i - 1].split(b" ")[1]:
            run = lines[a:i]
            if cut and i == len(lines):
                run = [b"* " + r.split(b" ")[1] for r in run]
            out += sorted(run)
            a = i
    return b"\n".join(out) + b"\n"


def expected_files(G, tag):
    """{name: bytes} of the reference's files whose last writer is stored in the golden."""
    ids = G[tag + "_ids"]
    last = {}
    for q, mid in enumerate(ids.tolist()):
        last["%06d" % mid] = q
    off, rows = G[tag + "_file_off"], G[tag + "_rows"]
    fmt = str(G["fmt"])
    out = {}
    for f, q in enumerate(G[tag + "_file_q"].tolist()):
        name = str(G[tag + "_file_name"][f])
        if last[name] == q:
            out[name] = savetxt_bytes(rows[off[f]:off[f + 1]], fmt)
    return out
