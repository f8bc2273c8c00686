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
