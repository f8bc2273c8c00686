"""numpy restatement of the ragged encoder's assignment, (cloud, node) sort and cluster statistics
(csrc/som_ragged.cu, networks.Encoder.forward_ragged): the definitions the kernels must meet bit for
bit, runnable without a GPU."""
import numpy as np

from test_seg_full_envelope_host import topk_ref


def assign(points, offsets, node, k):
    """points [T,6] f32, offsets [B+1], node [B,3,M] f32 -> (min_idx [k*T] i32 cloud-local, stacked
    column k*offsets[b] + s*P_b + n; count [B,M] i32). Each point's k nodes are topk_ref's."""
    B, _, M = node.shape
    T = points.shape[0]
    idx = np.empty(k * T, dtype=np.int32)
    count = np.zeros((B, M), dtype=np.int32)
    for b in range(B):
        lo, hi = int(offsets[b]), int(offsets[b + 1])
        top = topk_ref(points[lo:hi, :3].astype(np.float32), node[b], k)   # [P, k]
        idx[k * lo:k * hi] = top.T.reshape(-1)
        np.add.at(count[b], top.reshape(-1), 1)
    return idx, count


def group(points, offsets, idx, M, k):
    """-> (order [k*T] stacked columns in sorted order (cloud, node, ascending stacked column),
    node_sorted [k*T] flat ids b*M+m, pos0 [B], cluster_mean [B,3,M] f32 in the stated order:
    lane l sums copies l, l+32, ... of a node in sequence, then the xor butterfly 16, 8, 4, 2, 1,
    then / (count + 1e-5))."""
    B = len(offsets) - 1
    order = np.empty_like(idx, dtype=np.int64)
    node_sorted = np.empty_like(idx)
    pos0 = np.empty(B, dtype=np.int32)
    cm = np.zeros((B, 3, M), dtype=np.float32)
    for b in range(B):
        lo, hi = int(offsets[b]), int(offsets[b + 1])
        P = hi - lo
        cols = idx[k * lo:k * hi]
        perm = np.argsort(cols, kind="stable")
        order[k * lo:k * hi] = k * lo + perm
        node_sorted[k * lo:k * hi] = b * M + cols[perm]
        pos0[b] = k * lo + int(np.flatnonzero(perm == 0)[0])
        xyz = points[lo:hi, :3].astype(np.float32)
        for m in range(M):
            rows = perm[cols[perm] == m] % P                        # point of each copy, ascending
            for c in range(3):
                v = xyz[rows, c]
                lanes = np.zeros(32, dtype=np.float32)
                for lane in range(32):
                    s = np.float32(0)
                    for x in v[lane::32]:
                        s = np.float32(s + x)
                    lanes[lane] = s
                for o in (16, 8, 4, 2, 1):
                    lanes = (lanes + lanes[np.arange(32) ^ o]).astype(np.float32)
                den = np.float32(np.float32(len(rows)) + np.float32(1e-5))
                cm[b, c, m] = np.float32(lanes[0] / den)
    return order, node_sorted, pos0, cm


# ---- offsets as the kernels clamp them (common.cuh: ragged_offset, ragged_range, ragged_find) -----
def clamped_offsets(offsets, T):
    """Every offset clamped into [0, T] (int64)."""
    return np.clip(np.asarray(offsets, dtype=np.int64), 0, T)


def ragged_ranges(offsets, T):
    """(lo [B], hi [B]) of every cloud: lo = clamp(offsets[b]), hi = clamp(offsets[b+1]) but never
    below lo, so a decreasing pair is an empty cloud. Clouds may overlap when offsets decrease."""
    c = clamped_offsets(offsets, T)
    return c[:-1], np.maximum(c[:-1], c[1:])


def ragged_find(offsets, T, g):
    """The cloud ragged_find gives each row of g (int64 array): its binary search over the clamped
    offsets, step for step, so that any offsets array (not only a sorted one) picks the same cloud.
    -> (b, inside) where inside is lo_b <= g < hi_b; a row outside its cloud belongs to none."""
    c = clamped_offsets(offsets, T)
    B = len(c) - 1
    g = np.asarray(g, dtype=np.int64)
    a = np.zeros(g.shape, np.int64)
    z = np.full(g.shape, B - 1, np.int64)
    while True:
        act = a < z
        if not act.any():
            break
        mid = (a + z + 1) >> 1
        le = c[np.minimum(mid, B - 1)] <= g
        a = np.where(act & le, mid, a)
        z = np.where(act & ~le, mid - 1, z)
    lo, hi = ragged_ranges(offsets, T)
    return a, (lo[a] <= g) & (g < hi[a])


def assign_rows(points, offsets, node, k):
    """sonet_som_assign_ragged_f32 for any offsets array: row g is assigned only inside its cloud
    b = ragged_find(g) and writes stacked column k*lo_b + s*P_b + (g - lo_b). -> (min_idx [k*T] i32,
    count [B,M] i32, writes [k*T] the number of rows that write each column: 0 leaves it untouched,
    more than one races, so only columns written once have a defined value)."""
    B, _, M = node.shape
    T = points.shape[0]
    lo, hi = ragged_ranges(offsets, T)
    b, inside = ragged_find(offsets, T, np.arange(T))
    idx = np.zeros(k * T, np.int32)
    writes = np.zeros(k * T, np.int64)
    count = np.zeros((B, M), np.int32)
    for bb in np.unique(b[inside]):
        g = np.flatnonzero(inside & (b == bb))
        top = topk_ref(points[g, :3].astype(np.float32), node[bb], k)      # [rows, k]
        P = hi[bb] - lo[bb]
        for s in range(k):
            cols = k * lo[bb] + s * P + (g - lo[bb])
            idx[cols] = top[:, s]
            np.add.at(writes, cols, 1)
        np.add.at(count[bb], top.reshape(-1), 1)
    return idx, count, writes


# ---- the group kernel, vectorised -----------------------------------------------------------------
def group_fast(points, offsets, idx, M, k):
    """group() for any offsets array and any ids, vectorised so that a cloud of 2^24 - 1 points
    restates in seconds. Ids are clamped into [0, M-1] and offsets as ragged_range, as the kernel
    reads them. Same outputs as group() (bit for bit where both apply); a cloud with no copies
    leaves its pos0 at -1 (the kernel does not write it) and its means 0 (0 / 1e-5). Each node's
    copies are padded to [L, 32] with +0 (lane l's copies l, l+32, ... in column l), then the L
    rows are summed in order with float32 vector adds: adding +0 to a sum that starts at +0 changes
    no bit, so this is the loop version's sequence."""
    T = points.shape[0]
    B = len(offsets) - 1
    lo, hi = ragged_ranges(offsets, T)
    ids = np.clip(np.asarray(idx).astype(np.int64), 0, M - 1)
    order = np.empty(len(ids), dtype=np.int64)
    node_sorted = np.empty(len(ids), dtype=np.int32)
    pos0 = np.full(B, -1, dtype=np.int32)
    cm = np.zeros((B, 3, M), dtype=np.float32)
    for b in range(B):
        P = int(hi[b] - lo[b])
        base = k * int(lo[b])
        cols = ids[base:base + k * P]
        perm = np.argsort(cols, kind="stable")
        order[base:base + k * P] = base + perm
        node_sorted[base:base + k * P] = b * M + cols[perm]
        if P:
            pos0[b] = base + int(np.flatnonzero(perm == 0)[0])
        nd = cols[perm]
        cnt = np.bincount(nd, minlength=M)
        start = np.concatenate([[0], np.cumsum(cnt)[:-1]])
        rank = np.arange(k * P) - start[nd]                      # position among the node's copies
        L = max(int(-(-cnt.max() // 32)) if P else 0, 1)
        den = (cnt.astype(np.float32) + np.float32(1e-5)).astype(np.float32)
        xyz = points[int(lo[b]):int(hi[b]), :3].astype(np.float32)
        for c in range(3):
            pad = np.zeros((L, M, 32), np.float32)
            pad[rank // 32, nd, rank % 32] = xyz[perm % P, c] if P else 0
            lanes = np.zeros((M, 32), np.float32)
            for step in range(L):
                lanes += pad[step]
            for o in (16, 8, 4, 2, 1):
                lanes = lanes + lanes[:, np.arange(32) ^ o]
            cm[b, c] = lanes[:, 0] / den
    return order, node_sorted, pos0, cm


def decenter(points, offsets, idx, cm, k, with_sn):
    """sonet_som_decenter_ragged_f32: the decentred copies in stacked order -> (x_aug [3(+3), k*T]
    f32, writes [k*T] the number of rows that write each column, as assign_rows). Row g of cloud b = ragged_find(g) (inside its cloud only) writes its
    copies at columns k*lo_b + s*P_b + (g - lo_b): xyz - cluster_mean[b, :, id] with the id clamped
    into [0, M-1], and the normal as it is."""
    B, _, M = cm.shape
    T = points.shape[0]
    lo, hi = ragged_ranges(offsets, T)
    b, inside = ragged_find(offsets, T, np.arange(T))
    g = np.flatnonzero(inside)
    b = b[g]
    P = hi[b] - lo[b]
    xa = np.zeros((6 if with_sn else 3, k * T), np.float32)
    writes = np.zeros(k * T, np.int64)
    for s in range(k):
        cols = k * lo[b] + s * P + (g - lo[b])
        ids = np.clip(np.asarray(idx)[cols].astype(np.int64), 0, M - 1)
        with np.errstate(all="ignore"):
            xa[:3, cols] = points[g, :3].T - cm[b, :, ids].T
        if with_sn:
            xa[3:, cols] = points[g, 3:].T
        np.add.at(writes, cols, 1)
    return xa, writes


# ---- index_max_ragged ---------------------------------------------------------------------------
SENTINEL = np.float32(-1000.0)


def index_max_ragged(data, index, offsets, M, k):
    """sonet_index_max_ragged_f32 per cloud: data [C, >= k*T] f32, index [k*T] cloud-local ids read
    as min(uint32(id), M-1), clamped offsets. For every (cloud, channel, node): the first
    cloud-local column whose value is the maximum, among values > float32(-1000) (strict; NaN never
    qualifies; +0 and -0 compare equal, so the first of them wins), else column 0. The value is the
    data at that column; a cloud with no copies gives (0, 0). -> (idx [B,C,M] i32, val [B,C,M] f32)."""
    data = np.asarray(data, dtype=np.float32)
    C = data.shape[0]
    B = len(offsets) - 1
    T = len(index) // k
    lo, hi = ragged_ranges(offsets, T)
    ids = np.minimum(np.asarray(index).astype(np.int32).view(np.uint32), np.uint32(M - 1)).astype(np.int64)
    out_i = np.zeros((B, C, M), np.int32)
    out_v = np.zeros((B, C, M), np.float32)
    for b in range(B):
        c0, c1 = k * int(lo[b]), k * int(hi[b])
        if c1 == c0:
            continue
        v = data[:, c0:c1]
        m = ids[c0:c1]
        with np.errstate(invalid="ignore"):
            ok = v > SENTINEL                                        # NaN: False
        w = np.where(ok, v + np.float32(0), -np.inf).astype(np.float32)   # -0 + 0 = +0
        best = np.full((C, M), -np.inf, np.float32)
        np.maximum.at(best.T, m, w.T)                               # per node, per channel
        hit = ok & (w == best[:, m])
        first = np.full((C, M), np.iinfo(np.int32).max, np.int64)
        j = np.broadcast_to(np.arange(c1 - c0), v.shape)
        np.minimum.at(first.T, m, np.where(hit, j, np.iinfo(np.int32).max).T)
        arg = np.where(first == np.iinfo(np.int32).max, 0, first)
        out_i[b] = arg
        out_v[b] = v[np.arange(C)[:, None], arg]
    return out_i, out_v
