"""Numpy restatement of the Chamfer kernels' contract (csrc/chamfer.cu), dense and ragged, without
importing the package:

  nn_scan     the brute-force nearest neighbour of every point of one cloud in another: fp32
              ((dx*dx + dy*dy) + dz*dz), every op rounded on its own; the scan starts from (+inf,
              index 0) and moves only on a strictly smaller distance, so ties go to the lowest index
              and a point with no finite neighbour keeps index 0 (its distance is then the one to the
              other cloud's point 0);
  elem        sqrt(d + 1e-8) per point;
  cloud_mean  chamfer_cloud_kernel's fixed order: 1024 thread-strided partial sums, the xor tree
              16..1 inside each warp, the same tree over the 32 warp sums, then / P;
  final_loss  chamfer_final_kernel's order: 256 thread-strided partial sums, a halving tree
              128..1, then / B, and forward + backward;
  chamfer_ragged  all of it per cloud of a ragged ground-truth set, the gt-side arrays stacked."""
import numpy as np

F32 = np.float32
EPS = F32(1e-8)


def dist2(p, g):
    """p [3] or [3,n], g [3,m] -> fp32 squared distances [m] or [n,m], rounded op by op."""
    with np.errstate(all="ignore"):
        p = np.asarray(p, F32).reshape(3, -1)
        g = np.asarray(g, F32)
        d = p[:, :, None] - g[:, None, :]
        return ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]).astype(F32)


def nn_scan(q, db, chunk=2048):
    """Nearest point of db [3,m] for every point of q [3,n] -> (idx [n] int64, d [n] f32)."""
    n = q.shape[1]
    idx = np.empty(n, np.int64)
    d = np.empty(n, F32)
    for s in range(0, n, chunk):
        D = dist2(q[:, s:s + chunk], db)                          # [c, m]
        key = np.where(np.isnan(D), np.inf, D)
        i = key.argmin(1)                                          # first minimum; all +inf -> 0
        i[np.isinf(key[np.arange(len(i)), i])] = 0
        idx[s:s + chunk] = i
        d[s:s + chunk] = D[np.arange(len(i)), i]
    return idx, d


def elem(d):
    with np.errstate(all="ignore"):
        return np.sqrt(np.asarray(d, F32) + EPS).astype(F32)


def _xor_tree(v):
    """Lane 0's value after v += shfl_xor(v, o) for o = 16..1, over the last axis (32 lanes)."""
    o = v.shape[-1] // 2
    while o:
        v = (v[..., :o] + v[..., o:2 * o]).astype(F32)
        o //= 2
    return v[..., 0]


def cloud_mean(e):
    """chamfer_cloud_kernel's mean of the per-point terms e [P] (P >= 1)."""
    e = np.asarray(e, F32)
    P = e.shape[0]
    rows = -(-P // 1024)
    pad = np.zeros(rows * 1024, F32)
    pad[:P] = e
    s = np.zeros(1024, F32)
    with np.errstate(all="ignore"):
        for r in range(rows):                                      # thread t adds t, t+1024, ...
            s = (s + pad[r * 1024:(r + 1) * 1024]).astype(F32)
        # padding adds +0.0: s + 0 == s for every s, -0 included (no term is -0)
        t = _xor_tree(s.reshape(32, 32))                           # per warp
        return F32(_xor_tree(t) / F32(P))


def _block_sum_256(s):
    s = np.asarray(s, F32).copy()
    w = 128
    while w:
        s[:w] = (s[:w] + s[w:2 * w]).astype(F32)
        w //= 2
    return s[0]


def final_loss(fwd_arr, bwd_arr):
    """chamfer_final_kernel: loss [3] of the per-cloud means."""
    out = []
    with np.errstate(all="ignore"):
        for a in (fwd_arr, bwd_arr):
            a = np.asarray(a, F32)
            B = a.shape[0]
            s = np.zeros(256, F32)
            for i in range(0, B, 256):
                c = a[i:i + 256]
                s[:len(c)] = (s[:len(c)] + c).astype(F32)
            out.append(F32(_block_sum_256(s) / F32(B)))
        return np.array([out[0], out[1], F32(out[0] + out[1])], F32)


def chamfer_cloud(pred, gt):
    """One cloud: pred [3,Mp], gt [3,N] -> dict of idx_fwd, idx_bwd, elem_fwd, elem_bwd, fwd, bwd."""
    i_f, d_f = nn_scan(pred, gt)
    i_b, d_b = nn_scan(gt, pred)
    e_f, e_b = elem(d_f), elem(d_b)
    return dict(idx_fwd=i_f, idx_bwd=i_b, elem_fwd=e_f, elem_bwd=e_b, fwd=cloud_mean(e_f),
                bwd=cloud_mean(e_b))


def chamfer_ragged(pred, points, offsets):
    """pred [B,3,Mp], points [T,>=3], offsets [B+1] -> the C-ABI's outputs as numpy arrays."""
    pred = np.asarray(pred, F32)
    points = np.asarray(points, F32)
    B = pred.shape[0]
    r = [chamfer_cloud(pred[b], points[offsets[b]:offsets[b + 1], :3].T) for b in range(B)]
    out = dict(idx_fwd=np.stack([c["idx_fwd"] for c in r]),
               idx_bwd=np.concatenate([c["idx_bwd"] for c in r]),
               elem_fwd=np.stack([c["elem_fwd"] for c in r]),
               elem_bwd=np.concatenate([c["elem_bwd"] for c in r]),
               fwd_arr=np.array([c["fwd"] for c in r], F32),
               bwd_arr=np.array([c["bwd"] for c in r], F32))
    out["loss"] = final_loss(out["fwd_arr"], out["bwd_arr"])
    return out
