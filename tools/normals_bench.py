"""normals_bench.py — exact per-cloud k-NN and PCA normal estimation on one GPU.

    python tools/normals_bench.py [--reps 10] [--ref-clouds 64] [--quick]

Workloads (random clouds in the unit cube, seeded):
  - 1,024 clouds of 10,000 points (meshes.sample_surface's default), at k = 16 and k = 32;
  - 2,048 ragged clouds of 2,000 to 3,000 points (ShapeNetPart's sizes), k = 16;
  - 8 clouds of 100,000 points (scan-sized), k = 16.
For each: the k-NN time (sonet_point_knn_f32), the normal time (sonet_point_normals_f32, centroid
orientation) and the orientation time (sonet_point_normals_orient_f32, minimum spanning tree with
the centroid anchor) apart, CUDA events around single warm calls, median of --reps; candidate pairs per
second (sum P_i^2 pairs); the k-NN's share of the FP32 bound, counting 8 flops per pair
(3 sub, 3 mul, 2 add: 8 * sum P_i^2 flops) against the H100 SXM data-sheet 67 TFLOP/s; and a speed
reference, torch.cdist + topk on the same clouds (query blocks of 4096 rows), timed on the first
--ref-clouds clouds and scaled to the workload by its pair count. For the orientation: the Borůvka
rounds that actually ran (read from the scratch's round flags), k-NN entries (T*K directed edges)
per second, and a CPU reference, scipy's minimum_spanning_tree + breadth_first_order and a
vectorised parity pass over the tree on the first --mst-clouds clouds, scaled by entry count. The
card's name, power limit and maximum SM clock are read in the same run. Prints one JSON line last.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import breadth_first_order, minimum_spanning_tree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

from sonet_b200 import ops  # noqa: E402

FP32_FLOPS = 67e12          # H100 SXM data sheet, dense FP32, 700 W
FLOPS_PER_PAIR = 8


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        out["power_limit"], out["max_sm_clock"] = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    except Exception as e:    # the numbers are still measured; the card's limits are then unknown
        out["power_limit"] = out["max_sm_clock"] = "unknown (%s)" % type(e).__name__
    return out


def median_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def torch_reference_ms(data, counts, k, n_clouds):
    """torch.cdist + topk over the first n_clouds clouds, ms (one pass after a warm-up)."""
    starts = np.concatenate([[0], np.cumsum(counts)])

    def run():
        for s in range(n_clouds):
            c = data[starts[s]:starts[s + 1], :3]
            for q0 in range(0, len(c), 4096):
                torch.cdist(c[q0:q0 + 4096], c).topk(k, dim=1, largest=False)
    return median_ms(run, 1)


def scipy_orient_ms(data, idx, counts, n_clouds):
    """scipy's MST of each of the first n_clouds k-NN graphs (weights 2 - |n_u . n_v|: 1 - |dot|
    offset past scipy's dropped zeros), a breadth-first order from point 0 and the signs by
    pointer doubling over the tree, ms (one pass after a warm-up)."""
    h = data[:, 3:6].cpu().numpy().astype(np.float64)
    nb = idx.cpu().numpy()
    starts = np.concatenate([[0], np.cumsum(counts)])

    def run():
        for s in range(n_clouds):
            P, r0 = int(counts[s]), int(starts[s])
            n, J = h[r0:r0 + P], nb[r0:r0 + P]
            u = np.repeat(np.arange(P), J.shape[1])
            v = J.reshape(-1).astype(np.int64)
            ok = (v >= 0) & (v != u)
            dot = (n[u[ok]] * n[v[ok]]).sum(1)
            tree = minimum_spanning_tree(coo_matrix((2.0 - np.abs(dot), (u[ok], v[ok])), shape=(P, P)).tocsr())
            order, pred = breadth_first_order(tree, 0, directed=False)
            anc = np.where(pred < 0, np.arange(P), pred)
            par = ((n * n[anc]).sum(1) < 0).astype(np.int8)
            while (anc != anc[anc]).any():
                par ^= par[anc]
                anc = anc[anc]
            n[order] *= np.where(par[order] == 1, -1.0, 1.0)[:, None]
    return median_ms(run, 1)


def workload(name, counts, k, reps, ref_clouds, rs, mst_clouds):
    counts = np.asarray(counts, np.int64)
    T = int(counts.sum())
    data = torch.from_numpy(rs.uniform(-1, 1, size=(T, 6)).astype(np.float32)).cuda()
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)])).cuda()
    idx, _ = ops.point_knn(data, off, k)
    t_knn = median_ms(lambda: ops.point_knn(data, off, k), reps)
    out = data[:, 3:6]
    t_nrm = median_ms(lambda: ops.estimate_normals(data, off, idx, ops.NORMALS_AWAY_FROM_CENTROID,
                                                   out=out), reps)
    maxp = int(counts.max())
    nbytes = int(ops._C.lib().sonet_point_normals_orient_scratch_bytes(T, len(counts)))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=data.device)
    t_ori = median_ms(lambda: ops.orient_normals(data, off, idx, out, ops.NORMALS_AWAY_FROM_CENTROID,
                                                 max_points=maxp, scratch=scratch), reps)
    flags = scratch[:4 * ops.POINT_ORIENT_MAX_ROUNDS].view(torch.int32).cpu().numpy()
    sched = ops.orient_rounds(maxp)
    rounds = min(sched, int(flags[:sched].sum()) + 1)
    n_mst = min(mst_clouds, len(counts))
    t_mst = scipy_orient_ms(data, idx, counts, n_mst) * T / float(counts[:n_mst].sum())
    pairs = float((counts.astype(np.float64) ** 2).sum())
    n_ref = min(ref_clouds, len(counts))
    ref_pairs = float((counts[:n_ref].astype(np.float64) ** 2).sum())
    t_ref = torch_reference_ms(data, counts, k, n_ref) * pairs / ref_pairs
    r = dict(workload=name, clouds=len(counts), points=T, k=k, knn_ms=round(t_knn, 3),
             normals_ms=round(t_nrm, 3), orient_ms=round(t_ori, 3), orient_rounds_run=rounds,
             orient_rounds_scheduled=sched, orient_entries_per_s=T * k / (t_ori / 1e3),
             scipy_mst_orient_ms_scaled=round(t_mst, 1), scipy_mst_clouds=n_mst,
             orient_speedup_vs_scipy=t_mst / t_ori, pairs_per_s=pairs / (t_knn / 1e3),
             knn_share_of_fp32_bound_8flops_per_pair=FLOPS_PER_PAIR * pairs / (t_knn / 1e3) / FP32_FLOPS,
             torch_cdist_topk_ms_scaled=round(t_ref, 1), torch_ref_clouds=n_ref,
             knn_speedup_vs_torch=t_ref / t_knn)
    print(json.dumps(r))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ref-clouds", type=int, default=64)
    ap.add_argument("--mst-clouds", type=int, default=4)
    ap.add_argument("--quick", action="store_true", help="small sizes, to check the script runs")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "normals_bench.py measures on a GPU"
    rs = np.random.RandomState(0)
    scale = 16 if a.quick else 1
    info = card()
    print(json.dumps(info))
    ref = (a.ref_clouds, rs, a.mst_clouds)
    res = [workload("modelnet_10k", [10000] * (1024 // scale), 16, a.reps, *ref),
           workload("modelnet_10k", [10000] * (1024 // scale), 32, a.reps, *ref),
           workload("shapenet_ragged", rs.randint(2000, 3001, size=2048 // scale), 16, a.reps, *ref),
           workload("scan_100k", [100000] * (8 if not a.quick else 1), 16, a.reps, *ref)]
    print(json.dumps(dict(card=info, results=res)))


if __name__ == "__main__":
    main()
