"""numpy restatement of the SHREC'16 retrieval ranking's contract (the comment at the top of
csrc/retrieval.cu), written from the contract alone: no radix select, no tiles, no work list. It
and the case builders below need neither a GPU nor the package, so they are proven against the host
entry on a CPU machine (test_retrieval_envelope_host.py) and then hold the kernel to the same bits
(test_gpu_retrieval_envelope.py).

  label  the given one, or torch.max's CPU argmax of the row. A label outside [0, L) gives a row of
         -1 / NaN with count -1, and the item is nobody's candidate.
  d      the difference in fp32; each difference squared in fp64 (exact); the squares summed one
         after the other in index order; sqrt in fp64; one rounding to fp32; sign cleared; every
         NaN made the canonical 0x7fc00000.
  order  keys (bits(d) << 32) | p ascending; each query keeps min(n, k) of them, the remaining
         slots hold -1 / NaN.

exact_dist_bits() is a second, value-level reference: the correctly rounded fp32 value of the exact
distance of the fp32 difference vector, computed in integers."""
import math

import numpy as np
import torch

NAN_KEY = 0x7fc00000
CHUNK = 1 << 22          # distance elements per vectorised block


def labels(feature, label, L):
    """-> (label_out [Q] int64, grp [Q] int64: the label where it lies in [0, L), else -1)."""
    if label is None:
        lab = torch.max(torch.from_numpy(np.ascontiguousarray(feature, np.float32)), 1)[1].numpy()
    else:
        lab = np.asarray(label, np.int64)
    return lab, np.where((lab >= 0) & (lab < L), lab, -1)


def dist_keys(fq, F):
    """uint32 distance keys [m, n] of the query rows fq [m, D] to the rows F [n, D] (float32).
    The squares are added one dimension at a time: a sequential sum (np.sum would sum pairwise)."""
    fq = np.asarray(fq, np.float32)
    F = np.asarray(F, np.float32)
    acc = np.zeros((fq.shape[0], F.shape[0]), np.float64)
    with np.errstate(all="ignore"):
        for x in range(F.shape[1]):
            d = (fq[:, x, None] - F[None, :, x]).astype(np.float64)   # the fp32 difference
            acc += d * d                                 # an exact square, one rounding
        f = np.sqrt(acc).astype(np.float32)
    u = f.view(np.uint32) & np.uint32(0x7fffffff)
    u[u > 0x7f800000] = NAN_KEY
    return u


def rank(feature, label, L, k, queries=None):
    """The contract's result for the rows `queries` (default: every row):
    dict(idx [m,k] int64, bits [m,k] uint32 (the dist bits), count [m] int32, label [Q] int64)."""
    feature = np.ascontiguousarray(feature, np.float32)
    Q = feature.shape[0]
    lab, grp = labels(feature, label, L)
    queries = np.arange(Q) if queries is None else np.asarray(queries, np.int64)
    m = len(queries)
    idx = np.full((m, k), -1, np.int64)
    bits = np.full((m, k), NAN_KEY, np.uint32)
    count = np.full(m, -1, np.int32)
    order = np.argsort(grp, kind="stable")
    sg = grp[order]
    qg = grp[queries]
    for g in np.unique(qg[qg >= 0]):
        mem = order[np.searchsorted(sg, g, "left"):np.searchsorted(sg, g, "right")]   # ascending p
        n, c = len(mem), min(len(mem), k)
        rows = np.flatnonzero(qg == g)
        step = max(1, CHUNK // n)
        for a in range(0, len(rows), step):
            r = rows[a:a + step]
            d = dist_keys(feature[queries[r]], feature[mem]).astype(np.uint64)
            keys = (d << np.uint64(32)) | mem.astype(np.uint64)[None, :]
            if c < n:
                keys = np.partition(keys, c - 1, axis=1)[:, :c]
            keys = np.sort(keys, axis=1)
            idx[r, :c] = (keys & np.uint64(0xffffffff)).astype(np.int64)
            bits[r, :c] = (keys >> np.uint64(32)).astype(np.uint32)
            count[r] = c
    return dict(idx=idx, bits=bits, count=count, label=lab)


def exact_dist_bits(fq, fp):
    """Bits of the correctly rounded (half to even) fp32 value of the exact Euclidean norm of the
    fp32 difference vector fq - fp, or None when a difference is not finite. Every finite fp32 is
    an integer multiple of 2^-149, so in units of 2^-149 the squared norm S is an exact integer and
    the fp32 neighbours of sqrt(S) are integers too."""
    with np.errstate(all="ignore"):
        d = np.abs((np.asarray(fq, np.float32) - np.asarray(fp, np.float32)).astype(np.float64))
    if not np.all(np.isfinite(d)):
        return None
    S = sum(int(v * 2.0 ** 149) ** 2 for v in d.tolist())
    r = math.isqrt(S)
    s = 1 << max(0, r.bit_length() - 24)         # fp32 spacing at r (1 below the normal range)
    lo = r // s * s
    four_mid2 = (2 * lo + s) ** 2                # (2 * midpoint)^2, compared with 4 S
    if 4 * S > four_mid2 or (4 * S == four_mid2 and (lo // s) & 1):
        lo += s
    with np.errstate(over="ignore"):
        f = np.float32(np.float64(lo) * 2.0 ** -149)     # lo has <= 24 significant bits: exact
    return int(np.array(f).view(np.uint32))


def exit_shift(keys, k):
    """Where a top-down, 8-bit-digit selection of the k smallest of the uint32 distance keys is
    decided: the shift of the highest byte in which the k-th and (k+1)-th smallest keys differ, or
    'tie' when they are equal (the cut falls inside a run of ties). None when len(keys) <= k."""
    s = np.sort(np.asarray(keys, np.uint64))
    if len(s) <= k:
        return None
    x = int(s[k - 1]) ^ int(s[k])
    return "tie" if x == 0 else 8 * ((x.bit_length() - 1) // 8)


# ---- case builders: (feature [Q,D] f32, label [Q] int64 or None, L, k) --------------------------

def _f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def dim_case(D, seed, Q=600):
    """Random rows over four labels at dimension D, a few duplicated rows (distance-0 ties), values
    spread over six decades so the fp64 sums carry bits fp32 cannot."""
    rs = np.random.RandomState(seed)
    f = (rs.standard_normal((Q, D)) * 10.0 ** rs.uniform(-3, 3, (Q, 1))).astype(np.float32)
    dup = rs.choice(Q, Q // 10, replace=False)
    f[dup] = f[rs.choice(Q, len(dup))]
    lab = rs.randint(0, 4, Q).astype(np.int64)
    return f, lab, 4, 50


def tile_case(n, k, seed, D=5):
    """One group of n members (label 1) among 300 noise items (labels 0 and 2), all interleaved.
    Features are quantised to halves, so distances tie often and cuts fall inside tie runs."""
    rs = np.random.RandomState(seed)
    Q = n + 300
    f = (np.round(rs.standard_normal((Q, D)) * 2) / 2).astype(np.float32)
    lab = np.where(rs.permutation(Q) < n, 1, rs.choice([0, 2], Q)).astype(np.int64)
    return f, lab, 3, k


EXIT_V = 0x3fa5c3e1      # no carry when 1 is added to any of its bytes


def exit_case(kind, seed, k=200, extra=150):
    """D = 1, one label. Item `origin` sits at 0, so its distances are exactly |f_p|, and they are
    laid out so that its k-th and (k+1)-th smallest keys first differ in byte `kind` (24, 16, 8, 0),
    or are equal ('tie': a run of 40 ties at the k-th value with 5 slots left for it). The keys
    below and above share as many leading bytes with the k-th as the exit allows, so every earlier
    digit is a real narrowing. Returns (feature, label, L, k, origin)."""
    rs = np.random.RandomState(seed)
    v = EXIT_V
    ties = np.zeros(0, np.int64)
    if kind == "tie":
        below = v - rs.randint(1, 1 << 12, k - 1 - 5)
        ties = np.full(40, v)
        above = v + rs.randint(1, 1 << 12, extra)
        keys = np.concatenate([below, above])
    else:
        s = int(kind)
        w = v + (1 << s)
        span = 1 << min(s + 8, 22)
        below = v - rs.randint(1, span, k - 2)
        above = w + rs.randint(0, span, extra)
        keys = np.concatenate([below, [v, w], above])
    x = _f32(keys.astype(np.uint32)) * rs.choice(np.float32([-1, 1]), len(keys))
    feat = np.concatenate([[0.0], x]).astype(np.float32)
    perm = rs.permutation(len(feat))
    feat = feat[perm]
    origin = int(np.flatnonzero(perm == 0)[0])
    # the tie run sits at positions 120..159: 8 ties in the last lanes of one 32-candidate chunk
    # (more than the 5 slots left, so the cut falls inside a warp's ballot) and across a tile edge
    feat = np.insert(feat, 120, _f32(ties.astype(np.uint32)))[:, None]
    origin += len(ties) if origin >= 120 else 0
    return feat, np.zeros(len(feat), np.int64), 1, k, origin


def special_case(kind, seed, Q=700):
    """Groups built from one kind of row (label 1, ~300 members) among ordinary rows (label 0);
    k = 100 cuts every row of the group, k = 250 for the overflow kinds keeps their inf distances
    in view while still cutting:
      zero      identical rows: every distance 0, every cut inside the tie run
      nan       a NaN in every member: every distance NaN
      inf_diff  members at +-3e38: fp32 differences overflow to inf
      inf_round members with d up to ~2.8e38 per dim, D = 2: the fp64 sum is finite, its sqrt
                rounds past FLT_MAX (or just below it)
      tiny      +-0 and subnormal features: subnormal differences and distances"""
    rs = np.random.RandomState(seed)
    D = 2 if kind == "inf_round" else 7
    f = rs.standard_normal((Q, D)).astype(np.float32)
    lab = (rs.uniform(size=Q) < 0.43).astype(np.int64)
    g = np.flatnonzero(lab == 1)
    if kind == "zero":
        f[g] = f[g[0]]
    elif kind == "nan":
        f[g, rs.randint(0, D, len(g))] = np.nan
    elif kind == "inf_diff":
        f[g] = np.float32(3e38) * rs.choice(np.float32([-1, 1]), (len(g), D))
    elif kind == "inf_round":
        f[g] = rs.choice(np.float32([-1.4e38, 0, 1.2e38, 1.4e38, 1.7e38, 2.0e38, 2.4e38]),
                         (len(g), D)) * rs.choice(np.float32([-1, 1]), (len(g), D))
    elif kind == "tiny":
        f[g] = _f32(rs.randint(0, 1 << 20, (len(g), D)).astype(np.uint32))
        f[g] *= rs.choice(np.float32([-1, 1]), (len(g), D))
        f[g[::5]] = rs.choice(np.float32([0.0, -0.0]), (len(g[::5]), D))
    else:
        raise ValueError(kind)
    return f, lab, 2, 250 if kind.startswith("inf") else 100


def group_labels(Q, pattern, L, seed):
    """Labels for the group kernel cases; every 17th item gets an invalid label (-1, L, 2^40)."""
    rs = np.random.RandomState(seed)
    if pattern == "one":
        lab = np.full(Q, L - 1, np.int64)                   # every lower label is an empty group
    elif pattern == "own":
        lab = np.arange(Q, dtype=np.int64) % L              # every item its own label (Q <= L)
    elif pattern == "even":
        lab = 2 * rs.randint(0, max(1, L // 2), Q).astype(np.int64)   # empty groups in between
    elif pattern == "zipf":
        lab = (rs.zipf(1.3, Q) - 1).astype(np.int64) % L
    else:
        raise ValueError(pattern)
    bad = np.arange(3, Q, 17)
    lab[bad] = np.array([-1, L, 1 << 40], np.int64)[np.arange(len(bad)) % 3]
    return lab


def group_case(Q, pattern, L, seed, D=3, k=64):
    rs = np.random.RandomState(seed)
    f = (np.round(rs.standard_normal((Q, D)) * 4) / 4).astype(np.float32)
    return f, group_labels(Q, pattern, L, seed), L, k


def argmax_case(D, seed, Q=32 * 12):
    """Rows whose argmax is decided by the tie and NaN rules across every lane residue mod 32:
      rows 0..31      one maximum at column r + 32 j (each lane residue r)
      rows 32..63     the maximum tied at two columns of different lanes (and the same lane)
      rows 64..95     NaN in several lanes (the first one wins), with +inf elsewhere
      rows 96..127    -0.0 and +0.0 as the tied maximum of a negative row
      the rest        random rows quantised to 1/2 (frequent ties)."""
    rs = np.random.RandomState(seed)
    f = (np.round(rs.standard_normal((Q, D)) * 2) / 2).astype(np.float32)
    for r in range(32):
        if r >= D:
            break
        cols = np.arange(r, D, 32)
        c = cols[rs.randint(len(cols))]
        f[r] = -1.0
        f[r, c] = 5.0
        a, b = np.sort(rs.choice(D, 2, replace=False)) if D >= 2 else (0, 0)
        if r % 4 == 0 and r + 32 < D:
            a, b = r, r + 32                                  # same lane
        f[32 + r] = -2.0
        f[32 + r, [a, b]] = 3.0
        nans = np.sort(rs.choice(D, min(D, 3), replace=False))
        f[64 + r, nans] = np.nan
        f[64 + r, rs.randint(D)] = np.inf
        f[96 + r] = -3.0
        z = rs.choice(D, min(D, 2), replace=False)
        f[96 + r, z[0]] = -0.0
        f[96 + r, z[-1]] = 0.0
    return f, None, D, 20


# ---- the grid shared by the host and the kernel tests ------------------------------------------
DIMS = (1, 2, 63, 64, 65, 127, 128, 129, 1023, 1024)          # around the 64-dim chunk
TILE_N = (1, 7, 8, 9, 127, 128, 129, 255, 256, 257, 5000)     # around the 8-query, 128-row tiles
EXITS = (24, 16, 8, 0, "tie")
SPECIALS = ("zero", "nan", "inf_diff", "inf_round", "tiny")
GROUP_Q = (1, 31, 32, 33, 1023, 1024, 1025, 32 * 1024 + 1)    # around the 32 warp segments
GROUP_PATTERNS = (("one", 1), ("one", 4096), ("own", 4096), ("even", 4095), ("zipf", 2),
                  ("zipf", 4096))
ARGMAX_D = (1, 31, 33, 100, 1024)


def tile_grid():
    """(n, k): k at n - 1, n, n + 1 and at 1, 2, 4095, 4096, so min(n, k) sits at 2^m - 1, 2^m and
    2^m + 1 around the bitonic sort's padding (127..129, 255..257, 4095, 4096)."""
    return [(n, k) for n in TILE_N for k in sorted({n - 1, n, n + 1, 1, 2, 4095, 4096})
            if 1 <= k <= 4096]


def pick_queries(feature, label, L, budget, seed):
    """Every query when the restatement's cost (sum of group size x D over the queries) fits in
    `budget`, else a seeded random subset that fits, with the first and last items always in."""
    Q, D = feature.shape
    _, grp = labels(feature, label, L)
    sizes = np.bincount(grp[grp >= 0], minlength=L)
    cost = np.where(grp >= 0, sizes[np.maximum(grp, 0)], 0).astype(np.float64) * D
    if cost.sum() <= budget:
        return np.arange(Q)
    m = max(16, int(budget / max(cost.mean(), 1.0)))
    rs = np.random.RandomState(seed)
    return np.unique(np.concatenate([[0, Q - 1], rs.choice(Q, min(m, Q), replace=False)]))


def work_items(grp, L, tile=8):
    """Length of the rank kernel's work list: one item per 8-query tile of every group."""
    sizes = np.bincount(grp[grp >= 0], minlength=L)
    return int(((sizes + tile - 1) // tile).sum())


def assert_equal_rank(got, want, queries, what):
    """got = (idx, dist, count, label) of the kernel or the host entry (numpy); want = rank()."""
    idx, dist, count, lab = (np.asarray(t) for t in got)
    assert np.array_equal(lab, want["label"]), "%s: label" % what
    assert np.array_equal(count[queries], want["count"]), "%s: count" % what
    bad = np.flatnonzero((idx[queries] != want["idx"]).any(1))
    assert len(bad) == 0, "%s: idx of query %d" % (what, queries[bad[0]])
    db = dist[queries].view(np.uint32)
    bad = np.flatnonzero((db != want["bits"]).any(1))
    assert len(bad) == 0, "%s: dist bits of query %d" % (what, queries[bad[0]])


def ulp_check(feature, idx, dist, count, pairs, seed):
    """max over `pairs` sampled (query, slot) entries of |bits(d) - bits(exact)|, the ulp distance
    of the result to the correctly rounded exact distance (finite differences only), and the
    number of entries checked."""
    rs = np.random.RandomState(seed)
    qs = np.flatnonzero(count > 0)
    worst, seen = 0, 0
    for q in rs.choice(qs, min(pairs, len(qs)), replace=True) if len(qs) else []:
        i = rs.randint(count[q])
        p = int(idx[q, i])
        e = exact_dist_bits(feature[q], feature[p])
        if e is None:
            continue
        worst = max(worst, abs(int(np.asarray(dist[q, i], np.float32).view(np.uint32)) - e))
        seen += 1
    return worst, seen
