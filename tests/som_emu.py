"""A plain numpy restatement of batch-SOM training as csrc/som_train.cu documents it, with EXACT
sums: the high-precision reference the SOM envelope tests hold the kernel to.

Per iteration, vectorised over clouds, points and nodes:
  1. d[n, m] = (dx*dx + dy*dy) + dz*dz in float32, dx = x - node, every operation rounded (numpy
     never fuses); the assignment is np.argmin, i.e. the FIRST minimal node.
  2. count and coordinate sums per node are exact, rounded once to float32;
     mean = sum / (float32(count) + 1e-5f) in float32.
  3. term[m, j] = ((mean[m] - node[j]) * occupied[m]) * W[m, j] * lr, each product rounded to
     float32; delta[j] = the exact sum over m, rounded once; node[j] += delta[j] in float32.

Exact sums: a float64 sum (np.bincount / np.sum) is within n * 2^-52 * sum|t| of the exact one, so
it rounds to the same float32 unless it lies that close to a float32 rounding boundary. Those
few sums are recomputed with math.fsum (and, when fsum's float64 lands exactly on a boundary,
the side is decided by the exact sign of sum - boundary).

The kernel accumulates the point sums in fp64 in a fixed order and rounds once: that is the
float32 of the exact sum unless its own fp64 error straddles a boundary (about 1e-8 per sum at
these sizes). The node-update sums are carried exactly (fp64 TwoSum) and rounded once: a plain
fp64 sum there was one ulp off whenever a few comparable terms met exactly on a float32 midpoint
and a tiny neighbourhood-tail term, lost in fp64, decided the side. Bit equality with this
emulation is therefore the expected result."""
import math

import numpy as np

F32 = np.float32
EPS_DEN = F32(1e-5)


def distances(x, node):
    """x [B,3,N], node [B,3,M] float32 -> d [B,N,M] float32, the kernel's rounding order."""
    dx = x[:, 0, :, None] - node[:, 0, None, :]
    dy = x[:, 1, :, None] - node[:, 1, None, :]
    dz = x[:, 2, :, None] - node[:, 2, None, :]
    return (dx * dx + dy * dy) + dz * dz


def f32_exact_sum(terms):
    """float32 nearest to the exact sum of `terms` (Python floats), ties to even."""
    s = math.fsum(terms)
    f = F32(s)
    for nb in (np.nextafter(f, F32(-np.inf)), np.nextafter(f, F32(np.inf))):
        mid = (float(f) + float(nb)) / 2.0          # exact: adjacent float32 values
        if s == mid:                                 # fsum's own rounding may have landed here
            r = math.fsum(list(terms) + [-mid])
            if r != 0.0:
                f = max(f, nb) if r > 0 else min(f, nb)
            break
    return f


def round_sums(s64, abs64, n, exact_terms):
    """float32 of exact sums, given their float64 approximations s64, the float64 sums of
    absolute values abs64 and the term counts n (arrays of one shape). exact_terms(index) returns
    the terms of one sum as a list; it is called only where s64 could round differently from the
    exact sum. Returns (float32 array, number of sums recomputed exactly)."""
    f = s64.astype(F32)
    err = np.asarray(n, dtype=np.float64) * 2.0 ** -52 * abs64
    f64 = f.astype(np.float64)
    lo = (f64 + np.nextafter(f, F32(-np.inf)).astype(np.float64)) / 2.0
    hi = (f64 + np.nextafter(f, F32(np.inf)).astype(np.float64)) / 2.0
    risky = (np.abs(s64 - lo) <= err) | (np.abs(s64 - hi) <= err)
    risky &= abs64 > 0
    idx = np.argwhere(risky)
    for i in idx:
        f[tuple(i)] = f32_exact_sum(exact_terms(tuple(i)))
    return f, len(idx)


class Margin:
    """Smallest best-vs-second distance gap met by any assignment: (gap, iteration, cloud, point)."""

    def __init__(self):
        self.gap, self.where = np.inf, None

    def update(self, d, t):
        if d.shape[2] < 2:
            return
        two = np.partition(d, 1, axis=2)[:, :, :2].astype(np.float64)
        g = two[:, :, 1] - two[:, :, 0]
        b, n = np.unravel_index(np.argmin(g), g.shape)
        if g[b, n] < self.gap:
            self.gap, self.where = float(g[b, n]), (t, int(b), int(n))

    def __repr__(self):
        return "min margin %.3g at (iteration, cloud, point) %s" % (self.gap, self.where)


def assign(x, node, margin=None, t=0):
    d = distances(x, node)
    if margin is not None:
        margin.update(d, t)
    return np.argmin(d, axis=2)


def step(x, node, W, lr, margin=None, t=0):
    """One batch-SOM iteration. x [B,3,N], node [B,3,M] float32; W [M,M] (W[m, j]); lr float.
    -> (node [B,3,M] float32, assignment [B,N] int64)."""
    B, _, N = x.shape
    M = node.shape[2]
    idx = assign(x, node, margin, t)
    flat = (idx + M * np.arange(B)[:, None]).ravel()
    cnt = np.bincount(flat, minlength=B * M).reshape(B, M)
    sums = np.empty((B, 3, M), dtype=F32)
    for c in range(3):
        xc = x[:, c, :].astype(np.float64)
        s64 = np.bincount(flat, weights=xc.ravel(), minlength=B * M).reshape(B, M)
        a64 = np.bincount(flat, weights=np.abs(xc).ravel(), minlength=B * M).reshape(B, M)
        sums[:, c], _ = round_sums(s64, a64, cnt,
                                   lambda i, c=c: x[i[0], c, idx[i[0]] == i[1]].tolist())
    mean = sums / (cnt.astype(F32) + EPS_DEN)[:, None, :]
    occ = (cnt > 0).astype(F32)
    diff = (mean[:, :, :, None] - node[:, :, None, :]) * occ[:, None, :, None]   # [B,3,m,j]
    terms = (diff * W.astype(F32)[None, None]) * F32(lr)
    t64 = terms.astype(np.float64)
    delta, _ = round_sums(t64.sum(axis=2), np.abs(t64).sum(axis=2), M,
                          lambda i: terms[i[0], i[1], :, i[2]].tolist())
    return node + delta, idx


def train(x, node0, Ws, lrs, margin=None):
    """T = len(lrs) iterations from node0 ([3,M] shared or [B,3,M]). Ws [T,M,M].
    -> (node [B,3,M] float32, last assignment [B,N] int64). With T = 0 the nodes pass through and
    the assignment is the one against node0."""
    x = np.asarray(x, dtype=F32)
    node = np.asarray(node0, dtype=F32)
    if node.ndim == 2:
        node = np.broadcast_to(node, (x.shape[0],) + node.shape)
    node = np.ascontiguousarray(node)
    idx = None
    for t in range(len(lrs)):
        node, idx = step(x, node, np.asarray(Ws[t]), float(lrs[t]), margin, t)
    if idx is None:
        idx = assign(x, node, margin, 0)
    return node, idx


def first_divergence(x, node0, Ws, lrs, other_nodes):
    """Where an iterated run first assigns a point differently from a run whose node trajectory
    is `other_nodes` (a list of [B,3,M] arrays, node after each iteration): the emulation's
    distances are evaluated against both node sets. -> (iteration, cloud, point, gap) or None,
    gap = the emulation's best-vs-second distance gap of that point."""
    x = np.asarray(x, dtype=F32)
    node = np.ascontiguousarray(np.broadcast_to(np.asarray(node0, dtype=F32),
                                                (x.shape[0], 3, np.asarray(node0).shape[-1])))
    prev_other = node
    for t in range(len(lrs)):
        a = assign(x, node)
        o = assign(x, np.asarray(prev_other, dtype=F32))
        bad = np.argwhere(a != o)
        if len(bad):
            b, n = bad[0]
            d = np.sort(distances(x[b:b + 1], node[b:b + 1])[0, n])
            return t, int(b), int(n), float(d[1] - d[0]) if len(d) > 1 else np.inf
        node, _ = step(x, node, np.asarray(Ws[t]), float(lrs[t]))
        prev_other = other_nodes[t]
    return None
