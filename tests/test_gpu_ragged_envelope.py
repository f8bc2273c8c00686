"""-m gpu: the ragged encoder's kernels (csrc/som_ragged.cu, index_max_ragged in csrc/index_max.cu,
the RAGGED pool epilogue of csrc/pointmlp_tc.cu) across their envelope, against the numpy
restatements of tests/ragged_emu.py bit for bit:

A. the assignment at every node count and k, with clouds whose edges fall inside and between the
   kernel's 256-thread blocks, adversarial and non-finite inputs, and the fp64 nearest nodes;
B. the (cloud, node) sort, cluster means and decentring from synthetic ids, with k*P at the sort's
   warp-range edges, a cloud of 2^24 - 1 points (the 24-bit point field at its limit), and every
   cluster mean against the fp64 mean within the bound of its summation order;
C. the fused RAGGED pool against the unfused index_max_ragged and its restatement, at the tile
   edges of the total row count and across thousands of tiny clouds; index_max_ragged alone;
D. forward_ragged / score_clouds in mixed batches against each cloud's dense forward;
E. malformed offsets at the C-ABI, with canary regions around every buffer.
"""
import itertools

import numpy as np
import pytest
import torch

import ragged_emu
from helpers import assert_close
from sonet_b200 import _C, ops
from test_gpu_pool_envelope import fused_net
from test_gpu_ragged_encoder import _clouds, _cls

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24                     # unit roundoff of float32
CANARY = 0x5A5A5A5A                # 1.5e16 as a float: reading it changes any result here
PATTERN = 0x13579BDF               # untouched output elements keep it
GUARD = 4096                       # elements on each side of every buffer (E and the group entry)


def _i32(a):
    return np.ascontiguousarray(a).view(np.int32)


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32).numpy()


class Guarded:
    """n 4-byte elements inside one allocation with GUARD canary elements on each side. Inputs take
    their values; outputs start at PATTERN."""

    def __init__(self, n, values=None, dtype=torch.float32):
        self.n, self.dtype = n, dtype
        self.base = torch.full((n + 2 * GUARD,), CANARY, dtype=torch.int32, device=DEV)
        if values is None:
            self.base[GUARD:GUARD + n] = PATTERN
        else:
            v = torch.as_tensor(values).reshape(-1)
            self.base[GUARD:GUARD + n] = v.to(DEV).view(torch.int32) if v.element_size() == 4 \
                else v.to(torch.int32).to(DEV)
        self.ptr = self.base.data_ptr() + 4 * GUARD

    def body(self):
        return self.base[GUARD:GUARD + self.n].cpu().numpy().view(
            np.float32 if self.dtype == torch.float32 else np.int32)

    def untouched(self):
        return self.base[GUARD:GUARD + self.n].cpu().numpy() == PATTERN

    def intact(self):
        b = self.base.cpu().numpy()
        return bool((b[:GUARD] == CANARY).all() and (b[GUARD + self.n:] == CANARY).all())


def _off64(offsets):
    """offsets as a guarded int64 device array (two int32 elements per offset)."""
    o = np.asarray(offsets, dtype=np.int64)
    g = Guarded(2 * len(o), torch.from_numpy(o.view(np.int32).copy()), dtype=torch.int32)
    return g


def _group_call(pts_np, offsets, ids_np, M, k, with_sn):
    """sonet_som_group_decenter_ragged_f32 on guarded buffers -> dict of host arrays; asserts the
    guards of every buffer are intact."""
    T = pts_np.shape[0]
    B = len(offsets) - 1
    CA = 6 if with_sn else 3
    pts = Guarded(6 * T, torch.from_numpy(np.ascontiguousarray(pts_np)))
    off = _off64(offsets)
    ids = Guarded(k * T, torch.from_numpy(np.ascontiguousarray(ids_np, dtype=np.int32)), torch.int32)
    cm, xs = Guarded(B * 3 * M), Guarded(CA * k * T)
    ns, p0 = Guarded(k * T, dtype=torch.int32), Guarded(B, dtype=torch.int32)
    _C.check(_C.lib().sonet_som_group_decenter_ragged_f32(
        pts.ptr, T, off.ptr, B, M, k, int(with_sn), ids.ptr, cm.ptr, xs.ptr, ns.ptr, p0.ptr, None),
        "som_group_decenter_ragged")
    torch.cuda.synchronize()
    for name, g in (("points", pts), ("offsets", off), ("min_idx", ids), ("cluster_mean", cm),
                    ("x_sorted", xs), ("node_sorted", ns), ("pos0", p0)):
        assert g.intact(), "%s: canary overwritten" % name
    return dict(cm=cm.body().reshape(B, 3, M), xs=xs.body().reshape(CA, k * T), ns=ns.body(),
                p0=p0.body(), xs_untouched=xs.untouched().reshape(CA, k * T),
                ns_untouched=ns.untouched(), p0_untouched=p0.untouched())


def _sorted_rows(pts, offsets, order, k):
    """The point row of every stacked column, in sorted order."""
    T = pts.shape[0]
    lo, hi = ragged_emu.ragged_ranges(offsets, T)
    pt_of = np.full(k * T, -1, np.int64)
    for b in range(len(lo)):
        P = hi[b] - lo[b]
        pt_of[k * lo[b]:k * hi[b]] = lo[b] + np.tile(np.arange(P), k)
    return pt_of[order]


def _check_group_against_emu(pts, offsets, ids, M, k, with_sn, got, clouds=None):
    """The group entry's outputs against group_fast, cloud by cloud (all clouds unless given)."""
    T = pts.shape[0]
    order, ns, p0, cm = ragged_emu.group_fast(pts, offsets, ids, M, k)
    lo, hi = ragged_emu.ragged_ranges(offsets, T)
    clouds = range(len(lo)) if clouds is None else clouds
    for b in clouds:
        c = slice(k * lo[b], k * hi[b])
        assert np.array_equal(got["ns"][c], ns[c]), "node_sorted, cloud %d" % b
        assert np.array_equal(_i32(got["cm"][b]), _i32(cm[b])), "cluster_mean, cloud %d" % b
        if hi[b] > lo[b]:
            assert got["p0"][b] == p0[b], "pos0, cloud %d" % b
        else:
            assert got["p0_untouched"][b], "pos0 of empty cloud %d written" % b
        src = _sorted_rows(pts, offsets, order[c], k)
        want = pts[src, :3].T - cm[b][:, ns[c] - b * M]
        assert np.array_equal(_i32(got["xs"][:3, c]), _i32(want)), "x_sorted xyz, cloud %d" % b
        if with_sn:
            assert np.array_equal(_i32(got["xs"][3:, c]), _i32(pts[src, 3:].T)), "x_sorted sn %d" % b
    return order, cm


def _mean_bound_check(pts, offsets, ids, M, k, cm, what):
    """Every cluster mean against the fp64 mean of the same copies. The stated order sums a node's
    copies in 32 lane chains of at most L = ceil(count/32) terms, then 5 butterfly levels: the sum
    is within gamma_(L+5) * sum|x| of the exact one (recursive summation, Higham (4.4)); den =
    fl(count + 1e-5) and the quotient add one rounding each, so |mean - S/(count + 1e-5)| <=
    gamma_(L+7) * sum|x| / (count + 1e-5). Returns the largest error relative to that bound."""
    T = pts.shape[0]
    lo, hi = ragged_emu.ragged_ranges(offsets, T)
    worst = 0.0
    for b in range(len(lo)):
        P = int(hi[b] - lo[b])
        if P == 0:
            continue
        nd = np.clip(ids[k * lo[b]:k * hi[b]].astype(np.int64), 0, M - 1)
        rows = np.tile(np.arange(P), k)
        cnt = np.bincount(nd, minlength=M).astype(np.float64)
        L = np.ceil(cnt / 32)
        gam = (L + 7) * U / (1 - (L + 7) * U)
        den = cnt + 1e-5
        for c in range(3):
            x = pts[lo[b]:hi[b], c].astype(np.float64)[rows]
            S = np.bincount(nd, weights=x, minlength=M)
            A = np.bincount(nd, weights=np.abs(x), minlength=M)
            err = np.abs(cm[b, c].astype(np.float64) - S / den)
            bound = gam * A / den
            assert np.all(err <= bound), "%s: cloud %d coordinate %d: error %.3e > bound %.3e" % (
                what, b, c, err.max(), bound[np.argmax(err - bound)])
            worst = max(worst, float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), 0))))
    return worst


# ---- A. the assignment -----------------------------------------------------------------------------------
MK = [(M, k) for M in (1, 2, 3, 9, 64, 65, 121, 255, 256) for k in (1, 2, 3, 4) if k <= M]


def _assign_batch(M, k, seed):
    """Ragged clouds with 1-point clouds, clouds of fewer than k points and of 255/256/257 points,
    so that the 256-thread blocks' edges fall inside and between clouds; points on nodes and
    duplicated nodes for exact ties."""
    sizes = [1, 255, max(k - 1, 1), 256, 1, 257, 3, 700]
    rs = np.random.RandomState(seed)
    T = sum(sizes)
    pts = rs.uniform(-1, 1, size=(T, 6)).astype(np.float32)
    node = rs.uniform(-1, 1, size=(len(sizes), 3, M)).astype(np.float32)
    if M >= 4:
        node[:, :, 1] = node[:, :, 3]                           # a duplicated node: exact ties
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    for b in range(len(sizes)):                                 # some points exactly on nodes
        r = np.arange(off[b], off[b + 1])[::5]
        pts[r, :3] = node[b][:, rs.randint(0, M, len(r))].T
    return pts, off, node


def _fp64_nearest_check(pts, off, node, idx, k):
    """The chosen k nodes are the fp64 k nearest: each chosen node's fp64 distance is at most the
    k-th smallest fp64 distance plus the fp32 distance's error, 2 * gamma_5 * d (dx = fl(p - n)
    and three products and sums, each one rounding; two such distances compared). Returns the
    largest excess over the k-th distance as a fraction of that bar (0 when every choice is the
    fp64 one)."""
    g5 = 5 * U / (1 - 5 * U)
    worst = 0.0
    for b in range(len(off) - 1):
        lo, hi = off[b], off[b + 1]
        d = ((pts[lo:hi, None, :3].astype(np.float64) - node[b].T[None].astype(np.float64)) ** 2).sum(2)
        kth = np.sort(d, axis=1)[:, k - 1]
        blk = idx[k * lo:k * hi].reshape(k, hi - lo).T                 # [P, k]
        chosen = np.take_along_axis(d, blk.astype(np.int64), axis=1)
        bar = 2 * g5 * chosen.max(1) + 1e-38
        assert np.all(chosen.max(1) <= kth + bar), b
        worst = max(worst, float(((chosen.max(1) - kth) / bar).max()))
    return worst


FP64_MARGIN = []     # the measured excess of every assignment test, reported at the last one


@pytest.mark.parametrize("M,k", MK, ids=["M%d-k%d" % c for c in MK])
def test_assign_bits_and_fp64_nearest(M, k):
    pts, off, node = _assign_batch(M, k, seed=M * 5 + k)
    idx, count, row_max = ops.som_assign_ragged(torch.from_numpy(pts).to(DEV),
                                                torch.from_numpy(off).to(DEV),
                                                torch.from_numpy(node).to(DEV), k)
    e_idx, e_count = ragged_emu.assign(pts, off, node, k)
    assert np.array_equal(idx.cpu().numpy(), e_idx)
    assert np.array_equal(count.cpu().numpy(), e_count)
    assert np.array_equal(row_max.cpu().numpy(), (e_count > 0).astype(np.int32))
    FP64_MARGIN.append(_fp64_nearest_check(pts, off, node, e_idx, k))
    if (M, k) == MK[-1]:
        print("\n[fp64 nearest] largest excess over the k-th fp64 distance: %.3g of the bar"
              % max(FP64_MARGIN))


@pytest.mark.parametrize("M,k", [(9, 3), (64, 4), (256, 2), (2, 2)])
def test_assign_adversarial_inputs(M, k):
    """NaN and +-inf points, coordinates whose squares overflow (every distance +inf: the fill
    rule), exact ties, and nodes with non-finite coordinates."""
    pts, off, node = _assign_batch(M, k, seed=M + 100 * k)
    bad = np.arange(0, len(pts), 37)
    pts[bad[0::5], 0] = np.nan
    pts[bad[1::5], 1] = np.inf
    pts[bad[2::5], 2] = -np.inf
    pts[bad[3::5], :3] = 3e19                                  # squares overflow
    pts[bad[4::5], 0] = 2e19
    node[1::2, 0, M - 1] = np.nan
    node[2::3, 1, 0] = np.inf
    node[3, 2, M // 2] = -np.inf
    node[4, :, :] = node[4, :, :1]                              # every node the same: all ties
    idx, count, row_max = ops.som_assign_ragged(torch.from_numpy(pts).to(DEV),
                                                torch.from_numpy(off).to(DEV),
                                                torch.from_numpy(node).to(DEV), k)
    e_idx, e_count = ragged_emu.assign(pts, off, node, k)
    assert np.array_equal(idx.cpu().numpy(), e_idx)
    assert np.array_equal(count.cpu().numpy(), e_count)
    assert np.array_equal(row_max.cpu().numpy(), (e_count > 0).astype(np.int32))


# ---- B. group, sort and decentre -------------------------------------------------------------------------
KP_EDGES = (1, 31, 32, 33, 1023, 1024, 1025, 32 * 1024 - 1, 32 * 1024 + 1, 64 * 1024 - 1, 64 * 1024 + 1)
GROUP_MS = (1, 2, 3, 65, 129, 256)
GROUP_DISTS = ("uniform", "one_node", "two_nodes", "clamped")
# every (k, M) meets every id distribution; with_sn alternates so that each distribution meets both
GROUP_CASES = [(k, M, (k + i) % 2 == 1, d)
               for k, M in itertools.product((1, 2, 3, 4), GROUP_MS) if k <= M
               for i, d in enumerate(GROUP_DISTS)]


def _edge_sizes(k):
    """Cloud sizes whose k*P lands on each edge (or on both sides of it when k does not divide it):
    warp ranges of R = roundup32(ceil(kP/32)) rows, one row batch, 1024 rows, 32*1024 and 64*1024."""
    s = set()
    for t in KP_EDGES:
        s.update({max(t // k, 1), -(-t // k)})
    return sorted(s)


def _ids(dist, n, M, rs):
    if dist == "uniform":
        return rs.randint(0, M, n).astype(np.int32)
    if dist == "one_node":                                     # every node empty but one
        return np.full(n, M - 1, np.int32)
    if dist == "two_nodes":                                    # the lowest and highest id: every id bit
        return np.where(rs.rand(n) < 0.5, 0, M - 1).astype(np.int32)
    ids = rs.randint(0, M, n).astype(np.int32)                 # clamped: -1, M and 2^31-1 mixed in
    pick = rs.rand(n)
    ids[pick < 0.1] = -1
    ids[(pick >= 0.1) & (pick < 0.2)] = M
    ids[(pick >= 0.2) & (pick < 0.25)] = 2 ** 31 - 1
    return ids


@pytest.mark.parametrize("k,M,with_sn,dist", GROUP_CASES,
                         ids=["k%d-M%d-sn%d-%s" % (k, M, sn, d) for k, M, sn, d in GROUP_CASES])
def test_group_sort_and_means_at_warp_range_edges(k, M, with_sn, dist):
    sizes = _edge_sizes(k)
    rs = np.random.RandomState(k * 1000 + M)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    T = int(off[-1])
    pts = rs.uniform(-1, 1, size=(T, 6)).astype(np.float32)
    pts[:, :3] += rs.uniform(-4, 4, size=(1, 3)).astype(np.float32)
    ids = _ids(dist, k * T, M, rs)
    got = _group_call(pts, off, ids, M, k, with_sn)
    _, cm = _check_group_against_emu(pts, off, ids, M, k, with_sn, got)
    _mean_bound_check(pts, off, ids, M, k, cm, "k%d M%d %s" % (k, M, dist))
    # the decentred copies in stacked order (the unfused route's input), ids clamped the same way
    x_aug = ops.som_decenter_ragged(torch.from_numpy(pts).to(DEV), torch.from_numpy(off).to(DEV),
                                    torch.from_numpy(ids).to(DEV),
                                    torch.from_numpy(got["cm"]).to(DEV), k, with_sn)
    want, writes = ragged_emu.decenter(pts, off, ids, got["cm"], k, with_sn)
    assert np.all(writes == 1)
    assert np.array_equal(_bits(x_aug[0]), _i32(want))


def test_largest_cloud_keeps_every_point_index():
    """One cloud of 2^24 - 1 points (the entry's limit on T) at k = 1: the point field of a sorted
    copy (n | node << 24) at its widest. Centred at 100 with unit extent, so that every cluster
    mean also shows the error of the stated summation order at lane chains of ~8000 terms; the
    error is reported next to torch's float32 mean of the same copies."""
    P, M, k = (1 << 24) - 1, 65, 1
    rs = np.random.RandomState(24)
    pts = np.empty((P, 6), np.float32)
    pts[:, :3] = 100 + rs.uniform(-0.5, 0.5, size=(P, 3)).astype(np.float32)
    pts[:, 3:] = rs.uniform(-1, 1, size=(P, 3)).astype(np.float32)
    ids = rs.randint(0, M, P).astype(np.int32)
    off = np.array([0, P], np.int64)
    got = _group_call(pts, off, ids, M, k, True)
    _, cm = _check_group_against_emu(pts, off, ids, M, k, True, got)
    rel = _mean_bound_check(pts, off, ids, M, k, cm, "2^24-1 points")
    # measured errors against the fp64 mean, and torch's float32 mean on the GPU for scale
    x = torch.from_numpy(pts[:, :3]).to(DEV)
    nd = torch.from_numpy(ids).to(DEV).long()
    cnt = np.bincount(ids, minlength=M).astype(np.float64)
    ours, theirs = 0.0, 0.0
    for c in range(3):
        S = np.bincount(ids, weights=pts[:, c].astype(np.float64), minlength=M)
        exact = S / (cnt + 1e-5)
        ours = max(ours, float(np.abs(cm[0, c].astype(np.float64) - exact).max()))
        tm = torch.stack([x[nd == m, c].mean() for m in range(M)]).cpu().double().numpy()
        theirs = max(theirs, float(np.abs(tm - S / cnt).max()))
    print("\n[largest cloud] max |cluster_mean - fp64 mean| = %.3e (%.3f of the bound); torch float32 "
          "mean: %.3e" % (ours, rel, theirs))


# ---- C. both pools -----------------------------------------------------------------------------------------
MODES = [("relu", False), ("relu", True), ("elu", False), ("elu", True)]


def _tiny_sizes(total, rs, hi=5):
    s = []
    while sum(s) < total:
        s.append(int(min(rs.randint(1, hi + 1), total - sum(s))))
    return s


def _pool_case(name):
    """-> (sizes, M, k, sentinel, nonfinite)."""
    rs = np.random.RandomState(sum(map(ord, name)))
    if name.startswith("rows"):                                # k*T at the 64/128-row tile edges
        return _tiny_sizes(int(name[4:]), rs, 3), 9, 1, False, False
    return {"tiny4000": (_tiny_sizes(12000, rs), 9, 3, False, False),
            "m1": ([1, 3, 2, 200, 1, 64], 1, 1, False, False),
            "m256": ([300, 1, 2, 700, 5], 256, 4, False, False),
            "sentinel": (_tiny_sizes(600, rs) + [400], 64, 3, True, False),
            "nonfinite": ([3, 500, 2, 1, 900], 9, 2, False, True)}[name]


POOL_CASES = ["rows%d" % n for n in (1, 63, 64, 65, 127, 128, 129, 255, 256, 257)] + \
    ["tiny4000", "m1", "m256", "sentinel", "nonfinite"]


@pytest.mark.parametrize("mode", MODES, ids=["%s-%s" % (a, "fp16" if f else "split") for a, f in MODES])
@pytest.mark.parametrize("case", POOL_CASES)
def test_fused_pool_matches_index_max_ragged(case, mode):
    """Tiny clouds back to back put the same local node of neighbouring clouds into one warp's 16
    rows; most of their nodes are empty, so every cloud's copy-0 fallback (pos0[cloud]) is read."""
    act, f16 = mode
    sizes, M, k, sentinel, nonfinite = _pool_case(case)
    pts, off, node, _ = _clouds(sizes, M, 0, seed=len(sizes) + M)
    if nonfinite:
        pts[4, 0] = float("nan")
        pts[600, 1] = float("inf")
        pts[601, 2] = -float("inf")
        pts[1400, :3] = float("nan")
    blob, fpar = fused_net(3, sentinel=sentinel)
    idx, _, _ = ops.som_assign_ragged(pts, off, node, k)
    xs, ns, p0s, cm = ops.som_group_decenter_ragged(pts, off, idx, M, k, True)
    keys, p0 = ops.pointresnet_tc_pool_ragged(xs, blob, fpar, ns, p0s, M, f16=f16, act=act)
    fused = ops.pool_finalize(keys, p0)
    x_aug = ops.som_decenter_ragged(pts, off, idx, cm, k, True)
    fpo = ops.pointresnet_tc(x_aug, blob, fpar, f16=f16, act=act)
    out_idx, val = ops.index_max_ragged(fpo[0], idx, off, M, k)
    w_idx, w_val = ragged_emu.index_max_ragged(fpo[0].cpu().numpy(), idx.cpu().numpy(),
                                               off.cpu().numpy(), M, k)
    assert np.array_equal(out_idx.cpu().numpy(), w_idx)
    assert np.array_equal(_bits(val), _i32(w_val))
    assert np.array_equal(_bits(fused), _i32(w_val))
    h_idx = idx.cpu().numpy()
    cnt = np.stack([np.bincount(h_idx[k * a:k * b], minlength=M)
                    for a, b in zip(off.tolist()[:-1], off.tolist()[1:])])
    if case == "tiny4000" or case.startswith("rows"):     # most clouds read their copy-0 fallback
        assert (cnt == 0).any(1).mean() > 0.5
    if sentinel:
        assert (w_idx == 0).sum() > 0


def _imr_data(C, kT, seed):
    rs = np.random.RandomState(seed)
    d = rs.randint(-3, 4, size=(C, kT)).astype(np.float32)      # exact ties across copies
    d[:, ::7] = -0.0
    d[:, 1::9] = 0.0
    d[:, 2::13] = np.nan
    d[:, 3::17] = np.inf
    d[:, 4::19] = -np.inf
    d[1::3] = -1000.0 - rs.randint(0, 2, size=(1, kT)).astype(np.float32)   # at the sentinel
    return d


@pytest.mark.parametrize("C", [1, 15, 16, 17, 384])
def test_index_max_ragged_alone(C):
    """Channel counts around IMR_G = 16, signed zeros, ties, NaN, +-inf, the -1000 sentinel, an
    empty cloud, and ids M .. M+3 (clamped to M-1). Ids stay within [0, M+3] at M = 9, so that a
    kernel without the clamp still indexes inside its [16 x 256] shared arrays; the restatement's
    reading of negative ids is checked on the host."""
    M, k = 9, 2
    sizes = [1, 4, 0, 37, 2, 300, 1]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    T = int(off[-1])
    data = _imr_data(C, k * T, seed=C)
    rs = np.random.RandomState(C)
    index = rs.randint(0, M, size=k * T).astype(np.int32)
    index[::11] = M + rs.randint(0, 4, size=len(index[::11]))
    out_idx, val = ops.index_max_ragged(torch.from_numpy(data).to(DEV), torch.from_numpy(index).to(DEV),
                                        torch.from_numpy(off).to(DEV), M, k)
    w_idx, w_val = ragged_emu.index_max_ragged(data, index, off, M, k)
    assert np.array_equal(out_idx.cpu().numpy(), w_idx)
    assert np.array_equal(_bits(val), _i32(w_val))


def test_index_max_ragged_ids_past_m():
    """Ids M .. M+3 at M = 9 read as M-1."""
    M, k, C = 9, 1, 33
    sizes = [5, 40, 1]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    data = _imr_data(C, k * 46, seed=3)
    index = np.random.RandomState(4).randint(0, M + 4, size=46).astype(np.int32)
    out_idx, val = ops.index_max_ragged(torch.from_numpy(data).to(DEV), torch.from_numpy(index).to(DEV),
                                        torch.from_numpy(off).to(DEV), M, k)
    w_idx, w_val = ragged_emu.index_max_ragged(data, index, off, M, k)
    assert np.array_equal(out_idx.cpu().numpy(), w_idx)
    assert np.array_equal(_bits(val), _i32(w_val))


# ---- D. model level ----------------------------------------------------------------------------------------
MODEL_CASES = [  # tc, M, k, som_k, surface_normal
    ("1", 9, 1, 9, True), ("fp16", 121, 2, 0, False), ("0", 256, 4, 9, True),
    ("1", 256, 2, 0, False), ("fp16", 9, 4, 9, True), ("0", 121, 1, 0, False)]


@pytest.mark.parametrize("tc,M,k,som_k,sn", MODEL_CASES,
                         ids=["tc%s-M%d-k%d-somk%d-sn%d" % c for c in MODEL_CASES])
def test_mixed_tiny_clouds_match_each_cloud_alone(monkeypatch, tc, M, k, som_k, sn):
    sizes = [1, 2, 3, 1, 5, 4, 1, 300, 2, 1, 1500]
    m = _cls(monkeypatch, tc, B=1, N=256, k=k, node_num=M, som_k=som_k, surface_normal=sn)
    enc = m.encoder
    pts, off, node, knn = _clouds(sizes, M, som_k, seed=M + k)
    feat, nodes = enc.forward_ragged(pts, off, node, knn, return_nodes=True)
    score = m.score_clouds(pts, off, node, knn)
    o = off.tolist()
    for b in range(len(sizes)):
        c = pts[o[b]:o[b + 1]]
        with torch.no_grad():
            f1 = enc(c[:, :3].t().contiguous().unsqueeze(0), c[:, 3:].t().contiguous().unsqueeze(0),
                     node[b:b + 1], knn[b:b + 1])
            s1 = m.classifier(f1)
        if tc == "0":       # the dense fp32 route sums cluster means in som_stats_kernel's order
            assert_close(nodes["som_node"][b], enc.som_node[0], "cluster_mean %d" % b)
            assert_close(nodes["first_pn_out_masked_max"][b], enc.first_pn_out_masked_max[0], "max %d" % b)
        else:
            assert torch.equal(nodes["som_node"][b], enc.som_node[0]), b
            assert torch.equal(nodes["first_pn_out_masked_max"][b], enc.first_pn_out_masked_max[0]), b
        tol = 4e-3 if tc == "fp16" else 1e-4
        assert_close(feat[b], f1[0], "feature %d" % b, tol)
        assert_close(score[b], s1[0], "score %d" % b, tol)
    # chunk_points at, one below and one above every cloud boundary change no bit
    for j in range(1, len(sizes)):
        for chunk in (o[j] - 1, o[j], o[j] + 1):
            if chunk < 1:
                continue
            f, n = enc.forward_ragged(pts, off, node, knn, chunk_points=chunk, return_nodes=True)
            assert torch.equal(f, feat), chunk
            assert torch.equal(n["first_pn_out_masked_max"], nodes["first_pn_out_masked_max"]), chunk
            assert torch.equal(n["som_node"], nodes["som_node"]), chunk
    assert torch.equal(m.score_clouds(pts, off, node, knn, chunk_points=o[len(sizes) // 2]), score)


# ---- E. malformed offsets at the C-ABI ---------------------------------------------------------------------
T_E = 60
BAD_OFFSETS = {
    "negative": [-7, 10, 25, 40, 60],
    "past_T": [0, 10, 25, T_E + 20, T_E + 37],
    "gap": [3, 10, 10, 40, 52],              # rows 0..2 and 52..59 in no cloud, cloud 1 empty
    "decreasing": [0, 20, 12, 30, 25, 60],   # cloud 1 empty, cloud 2 [12, 30) overlaps cloud 0
    "b_large": [0, 30, 60, 60, 60, 60, 90],  # more clouds than non-empty ones
    # cloud 7 [10, 60) overlaps cloud 0 [0, 30): its flat ids 63..71 in shared columns, read back
    # as point indices of cloud 0, would name rows past T unless clamped to cloud 0's own
    "overlap_far": [0, 30, 30, 30, 30, 30, 30, 10, 60],
}


def _overlapping(lo, hi):
    """Clouds whose clamped row range overlaps another non-empty cloud's."""
    bad = set()
    for a in range(len(lo)):
        for b in range(a + 1, len(lo)):
            if lo[a] < hi[a] and lo[b] < hi[b] and lo[a] < hi[b] and lo[b] < hi[a]:
                bad.update((a, b))
    return bad


@pytest.mark.parametrize("k", [1, 4])
@pytest.mark.parametrize("case", list(BAD_OFFSETS))
def test_malformed_offsets_stay_in_range(case, k):
    """Every entry with offsets that are negative, decreasing, past T or leave rows in no cloud:
    every canary is intact, every untouched element keeps its pattern, and every output with a
    defined value equals the restatement under the clamped offsets. Columns that two clouds (or two
    rows) claim, possible only when offsets decrease, have no defined value."""
    offsets = BAD_OFFSETS[case]
    B, M, T, C = len(offsets) - 1, 9, T_E, 17
    rs = np.random.RandomState(len(case) + k)
    pts_np = rs.uniform(-1, 1, size=(T, 6)).astype(np.float32)
    node_np = rs.uniform(-1, 1, size=(B, 3, M)).astype(np.float32)
    lib = _C.lib()
    off = _off64(offsets)
    lo, hi = ragged_emu.ragged_ranges(offsets, T)

    # assignment
    pts = Guarded(6 * T, torch.from_numpy(pts_np))
    node = Guarded(B * 3 * M, torch.from_numpy(node_np))
    idx, cnt, rmax = Guarded(k * T, dtype=torch.int32), Guarded(B * M, dtype=torch.int32), \
        Guarded(B * M, dtype=torch.int32)
    _C.check(lib.sonet_som_assign_ragged_f32(pts.ptr, T, off.ptr, B, node.ptr, M, k, idx.ptr, cnt.ptr,
                                             rmax.ptr, None), "som_assign_ragged")
    torch.cuda.synchronize()
    e_idx, e_count, writes = ragged_emu.assign_rows(pts_np, offsets, node_np, k)
    for name, g in (("points", pts), ("offsets", off), ("node", node), ("min_idx", idx),
                    ("count", cnt), ("row_max", rmax)):
        assert g.intact(), "assign: %s canary" % name
    assert np.array_equal(idx.untouched(), writes == 0)
    one = writes == 1
    assert np.array_equal(idx.body()[one], e_idx[one])
    assert np.array_equal(cnt.body().reshape(B, M), e_count)
    assert np.array_equal(rmax.body().reshape(B, M), (e_count > 0).astype(np.int32))

    # group, sort and decentre from synthetic ids (out-of-range ones among them)
    ids = rs.randint(-1, M + 1, size=k * T).astype(np.int32)
    got = _group_call(pts_np, offsets, ids, M, k, True)
    bad = _overlapping(lo, hi)
    ok = [b for b in range(B) if b not in bad]
    _check_group_against_emu(pts_np, offsets, ids, M, k, True, got, clouds=ok)
    claimed = np.zeros(k * T, bool)
    for b in range(B):
        claimed[k * lo[b]:k * hi[b]] = True
    assert got["ns_untouched"][~claimed].all() and got["xs_untouched"][:, ~claimed].all()
    # columns of overlapping clouds: unspecified, but made of the clouds' own rows and nodes only:
    # flat ids of a claiming cloud, |x - mean| within twice the largest coordinate, real normals
    for b in bad:
        c = slice(k * lo[b], k * hi[b])
        owners = [a for a in bad if lo[a] < hi[b] and lo[b] < hi[a]]
        assert np.isin(got["ns"][c] // M, owners).all(), "node_sorted of overlapping cloud %d" % b
        assert np.all(np.abs(got["xs"][:3, c]) <= 2 * np.abs(pts_np[:, :3]).max()), b
        assert np.isin(got["xs"][3:, c], pts_np[:, 3:]).all(), b

    # decentring in stacked order
    cm_np = rs.uniform(-1, 1, size=(B, 3, M)).astype(np.float32)
    cmg = Guarded(B * 3 * M, torch.from_numpy(cm_np))
    xa, dids = Guarded(6 * k * T), Guarded(k * T, torch.from_numpy(ids), torch.int32)
    _C.check(lib.sonet_som_decenter_ragged_f32(pts.ptr, T, off.ptr, B, M, k, 1, dids.ptr, cmg.ptr,
                                               xa.ptr, None), "som_decenter_ragged")
    torch.cuda.synchronize()
    assert xa.intact() and cmg.intact() and pts.intact()
    want, dw = ragged_emu.decenter(pts_np, offsets, ids, cm_np, k, True)
    body = xa.body().reshape(6, k * T)
    assert (xa.untouched().reshape(6, k * T)[:, dw == 0]).all()
    assert np.array_equal(_i32(body[:, dw == 1]), _i32(want[:, dw == 1]))

    # index_max_ragged (reads only: every cloud has a defined result); ids in [0, M+3] only, as in
    # test_index_max_ragged_alone
    ids = rs.randint(0, M + 4, size=k * T).astype(np.int32)
    data_np = _imr_data(C, k * T, seed=k)
    data = Guarded(C * k * T, torch.from_numpy(data_np))
    ig = Guarded(k * T, torch.from_numpy(ids), torch.int32)
    oi, ov = Guarded(B * C * M, dtype=torch.int32), Guarded(B * C * M)
    _C.check(lib.sonet_index_max_ragged_f32(data.ptr, C, k * T, ig.ptr, off.ptr, B, T, M, k, oi.ptr,
                                            ov.ptr, None), "index_max_ragged")
    torch.cuda.synchronize()
    assert data.intact() and ig.intact() and oi.intact() and ov.intact()
    w_idx, w_val = ragged_emu.index_max_ragged(data_np, ids, offsets, M, k)
    assert np.array_equal(oi.body().reshape(B, C, M), w_idx)
    assert np.array_equal(_i32(ov.body().reshape(B, C, M)), _i32(w_val))
