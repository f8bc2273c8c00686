"""Datasets from meshes: the two offline steps in front of SO-Net's loaders, batched on the device.

1. Surface sampling (the reference's data/sampler_matlab/sampler.m): a face is chosen with
   probability proportional to its area, a point uniformly on it, and the point carries the face's
   unit normal; sample_surface runs it for a whole batch of meshes (csrc/mesh_sample.cu).
2. Per-shape SOM nodes (data/build_som/save_som.ipynb): choice(P, 4096, replace=False), then an
   8x8 SOM's optimize(); som_nodes runs it for the batch with sample_points and BatchSOM.

build_dataset chains both into an augmentation.DeviceDataset, save_npz writes the notebook's
model_<name>.npz files (pc, sn, som_node). Mesh files are parsed on the host (read_obj, read_off).

Deviations from the reference, all deliberate:
  - sampler.m:35 computes a + u*b + v*c, which is not a point of the triangle; the point here is
    (a + u*(b-a)) + v*(c-a), uniform on the triangle, as the reference README describes.
  - read_obj.m keeps the first three indices of every face; polygons are triangulated here as a fan
    (v0, vk, vk+1), so an n-gon's whole area is sampled.
  - MATLAB's random streams are not reproduced: the draws come from numpy (draw_host, in
    sampler.m's order) or from the kernel's Philox generator.
"""
import os

import numpy as np
import torch

from . import ops
from .augmentation import DeviceDataset
from .som import BatchSOM

_MAX_COUNT = 2 ** 31 - 1      # faces and vertices per mesh


# ---- host parsers ---------------------------------------------------------------------------------
def _fan(poly):
    """Triangles (v0, vk, vk+1) of one polygon's vertex list."""
    return [(poly[0], poly[k], poly[k + 1]) for k in range(1, len(poly) - 1)]


def _faces_array(tris, V, path):
    f = np.asarray(tris, dtype=np.int64).reshape(-1, 3)
    if f.size and (f.min() < 0 or f.max() >= V):
        bad = int(np.flatnonzero((f < 0).any(1) | (f >= V).any(1))[0])
        raise ValueError("%s: face %d refers to a vertex outside [0, %d)" % (path, bad, V))
    return f.astype(np.int32)


def read_obj(path):
    """(verts [V,3] f64, faces [F,3] i32) of a Wavefront OBJ file. Only `v` and `f` lines are read;
    face tokens may be `i`, `i/j`, `i/j/k` or `i//k` (the vertex index is the first field), 1-based
    or negative (relative to the vertices defined so far). Polygons are fan-triangulated. An index
    outside the vertices raises ValueError."""
    verts, tris = [], []
    with open(path, "r", newline=None) as fh:
        for lineno, line in enumerate(fh, 1):
            tok = line.split("#", 1)[0].split()
            if not tok:
                continue
            if tok[0] == "v":
                if len(tok) < 4:
                    raise ValueError("%s:%d: vertex with fewer than 3 coordinates" % (path, lineno))
                verts.append((float(tok[1]), float(tok[2]), float(tok[3])))
            elif tok[0] == "f":
                poly = []
                for t in tok[1:]:
                    i = int(t.split("/", 1)[0])
                    if i == 0:
                        raise ValueError("%s:%d: vertex index 0 (OBJ indices start at 1)" % (path, lineno))
                    poly.append(i - 1 if i > 0 else len(verts) + i)
                if len(poly) < 3:
                    raise ValueError("%s:%d: face with fewer than 3 vertices" % (path, lineno))
                tris.extend(_fan(poly))
    V = len(verts)
    return np.asarray(verts, dtype=np.float64).reshape(V, 3), _faces_array(tris, V, path)


def read_off(path):
    """(verts [V,3] f64, faces [F,3] i32) of an OFF file (ModelNet's format). Accepts `#` comments,
    the counts on the header line itself, also when merged into it as ModelNet writes them
    (`OFF1234 5678 0`), and face lines `n i0 .. i(n-1)` (fan-triangulated; values after the n
    indices, such as colours, are ignored). An index outside the vertices raises ValueError."""
    with open(path, "r", newline=None) as fh:
        lines = [ln.split("#", 1)[0].split() for ln in fh]
    lines = [t for t in lines if t]
    if not lines or not lines[0][0].startswith("OFF"):
        raise ValueError("%s: not an OFF file (no OFF header)" % path)
    head = lines[0]
    rest = [head[0][3:]] if len(head[0]) > 3 else []
    counts = rest + head[1:]
    body = 1
    if not counts:
        counts, body = lines[1], 2
    if len(counts) < 2:
        raise ValueError("%s: the OFF header needs vertex and face counts" % path)
    nv, nf = int(counts[0]), int(counts[1])
    if len(lines) < body + nv + nf:
        raise ValueError("%s: %d vertices and %d faces declared, %d lines present"
                         % (path, nv, nf, len(lines) - body))
    vl = lines[body:body + nv]
    verts = np.array([[float(x) for x in t[:3]] for t in vl], dtype=np.float64).reshape(nv, 3)
    tris = []
    for t in lines[body + nv:body + nv + nf]:
        n = int(t[0])
        if n < 3 or len(t) < n + 1:
            raise ValueError("%s: face line %r needs at least 3 indices" % (path, " ".join(t)))
        poly = [int(x) for x in t[1:n + 1]]
        tris.extend([tuple(poly)] if n == 3 else _fan(poly))
    return verts, _faces_array(tris, nv, path)


# ---- the device batch -----------------------------------------------------------------------------
class Meshes:
    """A batch of B meshes uploaded once as ragged device arrays: verts [sum V, 3] f64, faces
    [sum F, 3] i32 (mesh-local indices), v_off / f_off [B+1] i64 and mesh_ids [B] i64 (default
    0..B-1), the key of the in-kernel draws: give each mesh of a dataset its own id and the points
    do not depend on how the dataset is cut into batches."""

    def __init__(self, meshes, mesh_ids=None, device="cuda"):
        B = len(meshes)
        vs, fs = [], []
        for i, (v, f) in enumerate(meshes):
            v = np.asarray(v, dtype=np.float64)
            f = np.asarray(f)
            if v.ndim != 2 or v.shape[1] != 3 or f.ndim != 2 or f.shape[1] != 3:
                raise ValueError("Meshes: mesh %d has verts %s and faces %s, expected [V,3] and [F,3]"
                                 % (i, v.shape, f.shape))
            if len(v) > _MAX_COUNT or len(f) > _MAX_COUNT:
                raise ValueError("Meshes: mesh %d has more than 2^31-1 vertices or faces" % i)
            vs.append(v)
            fs.append(f.astype(np.int32))
        self.v_counts = np.array([len(v) for v in vs], dtype=np.int64)
        self.f_counts = np.array([len(f) for f in fs], dtype=np.int64)
        ids = np.arange(B, dtype=np.int64) if mesh_ids is None else \
            np.asarray(mesh_ids, dtype=np.int64).reshape(-1)
        if len(ids) != B:
            raise ValueError("Meshes: %d mesh ids for %d meshes" % (len(ids), B))
        self.device = torch.device(device)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)  # noqa: E731
        self.verts = up(np.concatenate(vs) if B else np.zeros((0, 3)))
        self.faces = up(np.concatenate(fs) if B else np.zeros((0, 3), np.int32))
        self.v_off = up(np.concatenate([[0], np.cumsum(self.v_counts)]).astype(np.int64))
        self.f_off = up(np.concatenate([[0], np.cumsum(self.f_counts)]).astype(np.int64))
        self.mesh_ids = up(ids)

    def __len__(self):
        return len(self.f_counts)


def draw_host(rng, B, N):
    """The (r, u, v) draws [B*N, 3] f64 of B meshes from the numpy generator `rng`, in sampler.m's
    order per mesh: N face uniforms, then N u, then N v; mesh b's rows are b*N .. b*N+N-1."""
    out = np.empty((B, N, 3), dtype=np.float64)
    for b in range(B):
        for k in range(3):
            out[b, :, k] = rng.random_sample(N)
    return out.reshape(B * N, 3)


def sample_surface(meshes, N=10000, seed=0, draws=None, want_faces=False, want_area=False):
    """N area-weighted surface points with their face normals per mesh: [B*N, 6] f32 on the meshes'
    device, xyz | normal, mesh b owning rows b*N .. b*N+N-1 (DeviceDataset's ragged layout).
    draws: [B*N, 3] (r, u, v) (e.g. draw_host's; numpy or tensor) or None for the kernel's draws
    keyed by (seed, mesh id, sample). With want_faces / want_area returns (points, faces [B*N] i32
    or None, areas [B] f64 or None). Raises ValueError naming the first mesh whose total area is 0
    or not finite (it has nothing to sample)."""
    dev = meshes.device
    if draws is not None:
        draws = torch.as_tensor(draws, dtype=torch.float64).to(dev).contiguous()
    out, face, area = ops.mesh_sample(meshes.verts, meshes.v_off, meshes.faces, meshes.f_off,
                                      meshes.mesh_ids, N, draws=draws, seed=seed,
                                      want_faces=want_faces, want_area=True)
    a = area.cpu().numpy()
    bad = ~(np.isfinite(a) & (a > 0))
    if bad.any():
        b = int(np.flatnonzero(bad)[0])
        raise ValueError("sample_surface: mesh %d (id %d) has total area %r: nothing to sample"
                         % (b, int(meshes.mesh_ids[b]), float(a[b])))
    if not (want_faces or want_area):
        return out
    return out, face, (area if want_area else None)


def som_nodes(points, rows=8, cols=8, n=4096, seed=0, rng=None):
    """The notebook's per-shape SOM (save_som.ipynb) for a batch: points [B, P, >=3] on the device
    (e.g. sample_surface's output viewed [B, N, 6]); n of each cloud's P points are chosen without
    replacement (in the kernel, keyed by `seed` and the batch position, or, with a numpy `rng`, by
    rng.choice(P, n, replace=False) per cloud as the notebook does), then BatchSOM(rows, cols)
    .optimize. -> [B, rows*cols, 3] f32."""
    if points.dim() != 3 or points.shape[2] < 3 or not points.is_cuda:
        raise RuntimeError("som_nodes: points must be a CUDA tensor [B, P, >=3]")
    B, P = points.shape[0], points.shape[1]
    if n > P:
        raise ValueError("som_nodes: cannot take a larger sample (%d) than population (%d) when "
                         "'replace=False'" % (n, P))
    dev = points.device
    data = torch.zeros((B * P, 6), dtype=torch.float32, device=dev)
    data[:, :3] = points.reshape(B * P, -1)[:, :3]
    offsets = torch.arange(B + 1, dtype=torch.int64, device=dev) * P
    ids = torch.arange(B, dtype=torch.int64, device=dev)
    indices = None
    if rng is not None:
        sel = np.stack([rng.choice(P, n, replace=False) for _ in range(B)]).astype(np.int32)
        indices = torch.from_numpy(sel).to(dev)
    elif P > ops.SAMPLE_MAX_P:
        raise ValueError("som_nodes: in-kernel choice supports P <= %d (got %d); pass rng"
                         % (ops.SAMPLE_MAX_P, P))
    pc, _, _ = ops.sample_points(data, offsets, ids, n, ops.SAMPLE_SUBSET, P, indices=indices,
                                 seed=seed)
    som = BatchSOM(rows, cols, 3, dev.index if dev.index is not None else 0, B)
    som.optimize(pc)
    return som.node.transpose(1, 2).contiguous()


def build_dataset(meshes, labels, N=10000, rows=8, cols=None, n=4096, seed=0, draws=None, rng=None):
    """Meshes -> an augmentation.DeviceDataset: N surface points per mesh (sample_surface) and its
    rows x cols SOM nodes (som_nodes, from n of those points), with the class ids `labels`."""
    B = len(meshes)
    if len(labels) != B:
        raise ValueError("build_dataset: %d labels for %d meshes" % (len(labels), B))
    pts = sample_surface(meshes, N, seed=seed, draws=draws)
    nodes = som_nodes(pts.view(B, N, 6), rows, rows if cols is None else cols, n, seed=seed, rng=rng)
    offsets = torch.arange(B + 1, dtype=torch.int64, device=pts.device) * N
    lab = torch.as_tensor(np.asarray(labels, dtype=np.int64))
    return DeviceDataset.from_device(pts, offsets, lab, nodes.transpose(1, 2).contiguous())


def save_npz(folder, names, points, som_nodes):
    """The notebook's files: folder/model_<name>.npz with pc [N,3], sn [N,3] and som_node [M,3]
    (the keys data/modelnet_shrec_loader.py reads) per shape. points [B, N, 6] and som_nodes
    [B, M, 3], numpy or tensors."""
    pts = points.detach().cpu().numpy() if torch.is_tensor(points) else np.asarray(points)
    nodes = som_nodes.detach().cpu().numpy() if torch.is_tensor(som_nodes) else np.asarray(som_nodes)
    if pts.ndim != 3 or pts.shape[2] != 6 or nodes.ndim != 3 or nodes.shape[2] != 3 \
            or len(names) != len(pts) or len(nodes) != len(pts):
        raise ValueError("save_npz: expected names [B], points [B,N,6], som_nodes [B,M,3]")
    os.makedirs(folder, exist_ok=True)
    paths = []
    for name, p, s in zip(names, pts, nodes):
        path = os.path.join(folder, "model_%s.npz" % name)
        np.savez(path, pc=p[:, 0:3], sn=p[:, 3:6], som_node=s)
        paths.append(path)
    return paths
