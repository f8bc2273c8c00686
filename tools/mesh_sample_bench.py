"""mesh_sample_bench.py — throughput of building a dataset from meshes on one GPU.

    python tools/mesh_sample_bench.py [--meshes 32] [--N 10000] [--reps 10] [--cpu-meshes 4]

Synthetic triangle meshes sized like SHREC'16 and ModelNet (face counts log-uniform from a few
hundred to about 10^6), N surface points each. Reports
  - meshes/s of the sampling alone (sonet_mesh_sample_f32) and of sampling plus the 8x8 SOM of 4096
    chosen points (meshes.som_nodes), CUDA events around whole batches;
  - the sampling's estimated HBM traffic as a share of the H100's 3.35 TB/s: one pass over faces
    (12 B read, 8 B CDF written) and vertices (24 B), then per sample three vertex reads (72 B),
    the face's indices (12 B) and the 24-byte row; the ~log2 F CDF probes per sample are counted
    apart, as L2 traffic;
  - the same work as a numpy per-mesh restatement of sampler.m plus the notebook's per-shape SOM
    (oracle/oracle.py's restatement of util/som.py, on the CPU), on --cpu-meshes meshes;
  - the host parse time per file (read_off / read_obj) of a 10^5-face mesh.
Prints one JSON line last.
"""
import argparse
import json
import math
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

from sonet_b200 import meshes, ops  # noqa: E402

HBM_BPS = 3.35e12


def synth_meshes(rs, B, lo=300, hi=1_000_000):
    out = []
    for F in np.exp(rs.uniform(math.log(lo), math.log(hi), B)).astype(np.int64):
        V = max(3, int(F) // 2)
        out.append((rs.uniform(-1, 1, size=(V, 3)), rs.randint(0, V, size=(int(F), 3))))
    return out


def gpu_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


def numpy_sampler(v, f, N, rs):
    """sampler.m in numpy (uniform on the triangle), one mesh."""
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    n = np.cross(b - a, c - a)
    ln = np.sqrt((n * n).sum(1))
    cdf = np.cumsum(0.5 * ln)
    idx = np.minimum(np.searchsorted(cdf, rs.random_sample(N) * cdf[-1], side="right"), len(f) - 1)
    u, w = rs.random_sample(N), rs.random_sample(N)
    s = u + w > 1
    u[s], w[s] = 1 - u[s], 1 - w[s]
    p = a[idx] + u[:, None] * (b - a)[idx] + w[:, None] * (c - a)[idx]
    return np.concatenate([p, n[idx] / ln[idx, None]], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--meshes", type=int, default=32)
    ap.add_argument("--N", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cpu-meshes", type=int, default=4)
    args = ap.parse_args()
    rs = np.random.RandomState(0)
    ms = synth_meshes(rs, args.meshes)
    B, N = len(ms), args.N
    F = np.array([len(f) for _, f in ms])
    V = np.array([len(v) for v, _ in ms])
    m = meshes.Meshes(ms, device="cuda")
    res = dict(meshes=B, N=N, faces_total=int(F.sum()), faces_min=int(F.min()), faces_max=int(F.max()),
               device=torch.cuda.get_device_name(0))

    def sample():
        return ops.mesh_sample(m.verts, m.v_off, m.faces, m.f_off, m.mesh_ids, N, seed=1)[0]

    def sample_som():
        pts = sample()
        return meshes.som_nodes(pts.view(B, N, 6), 8, 8, 4096, seed=1)

    t_s = gpu_time(sample, args.reps)
    t_ss = gpu_time(sample_som, max(2, args.reps // 2))
    hbm = F.sum() * (12 + 8) + V.sum() * 24 + B * N * (72 + 12 + 24)
    l2 = B * N * 16 * float(np.mean(np.log2(np.maximum(F, 2))))
    res.update(sample_s=t_s, sample_meshes_per_s=B / t_s, sample_som_s=t_ss,
               sample_som_meshes_per_s=B / t_ss, hbm_bytes=int(hbm), hbm_share=hbm / t_s / HBM_BPS,
               probe_l2_bytes=int(l2))

    # the numpy per-mesh restatement plus the notebook's SOM, on the CPU
    from oracle import oracle
    from sonet_b200 import som as som_mod
    init = som_mod.BatchSOM(8, 8, 3, 0, 1).node_init_value
    k = min(args.cpu_meshes, B)
    order = np.argsort(F)[np.linspace(0, B - 1, k).astype(int)]    # a spread of sizes
    crs = np.random.RandomState(1)
    t0 = time.perf_counter()
    for i in order:
        v, f = ms[i]
        numpy_sampler(v, f, N, crs)
    t_np = (time.perf_counter() - t0) / k
    t0 = time.perf_counter()
    for i in order:
        v, f = ms[i]
        pc = numpy_sampler(v, f, N, crs)[:, :3]
        x = torch.from_numpy(pc[crs.choice(N, 4096, replace=False)].T.astype(np.float32))[None]
        oracle.som_optimize(x, init, 8, 8)
    t_np_som = (time.perf_counter() - t0) / k
    # the cpu meshes' mean size differs from the batch's: scale by faces
    fscale = F.mean() / F[order].mean()
    res.update(cpu_sample_meshes_per_s=1 / t_np, cpu_sample_som_meshes_per_s=1 / t_np_som,
               cpu_meshes=k, cpu_mean_faces=float(F[order].mean()), cpu_face_scale=float(fscale))

    # host parse time per file
    v, f = synth_meshes(np.random.RandomState(2), 1, 100_000, 100_001)[0]
    with tempfile.TemporaryDirectory() as tmp:
        off, obj = os.path.join(tmp, "m.off"), os.path.join(tmp, "m.obj")
        with open(off, "w") as fh:
            fh.write("OFF\n%d %d 0\n" % (len(v), len(f)))
            np.savetxt(fh, v, fmt="%.6f")
            np.savetxt(fh, np.concatenate([np.full((len(f), 1), 3), f], 1), fmt="%d")
        with open(obj, "w") as fh:
            np.savetxt(fh, v, fmt="v %.6f %.6f %.6f")
            np.savetxt(fh, f + 1, fmt="f %d %d %d")
        for name, fn, path in (("off", meshes.read_off, off), ("obj", meshes.read_obj, obj)):
            t0 = time.perf_counter()
            fn(path)
            res["parse_%s_s_per_100k_faces" % name] = time.perf_counter() - t0
    for key, val in res.items():
        print("%-32s %s" % (key, ("%.4g" % val) if isinstance(val, float) else val))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
