"""Tensor-level wrappers over the C-ABI: validate, allocate outputs, pass the current stream.

Every function here launches hand-written sm_90a kernels from libsonet_b200.so on the tensors'
device and the current torch stream. Inputs must be CUDA, contiguous, of the stated dtype — the
same checks the reference plugin does with CHECK_INPUT (models/index_max_ext/index_max.cpp:119-121),
raised as RuntimeError. Nothing here falls back to PyTorch or the CPU.
"""
import ctypes
import os

import torch

from . import _C

LAUNCHES = 0          # C-ABI compute calls issued
KERNEL_LAUNCHES = 0   # CUDA kernels launched by those calls (bench.py's gpu_launches)
_KERNELS_PER_CALL = {"sonet_som_assign": 2, "sonet_chamfer_f32": 3}
PROFILE = None        # when a list: every call appends (name, start_event, end_event)


def _chk(t, name, dtype=None, optional=False):
    if t is None:
        if optional:
            return
        raise RuntimeError("%s must not be None" % name)
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor/variable" % name)
    if not t.is_contiguous():
        raise RuntimeError("%s must be contiguous" % name)
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError("%s must have dtype %s (got %s)" % (name, dtype, t.dtype))


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


# activation codes of the C-ABI (SONET_ACT_*, include/sonet_b200.h)
ACT_NONE = _C.CONSTANTS["SONET_ACT_NONE"]
ACT_RELU = _C.CONSTANTS["SONET_ACT_RELU"]
ACT_ELU = _C.CONSTANTS["SONET_ACT_ELU"]
_ACT_NAMES = {None: ACT_NONE, "relu": ACT_RELU, "elu": ACT_ELU}


def act_code(act):
    """An activation as its C-ABI code: a layer's activation name (None, 'relu', 'elu'), a bool
    (False / True = none / ReLU, the old flag) or a code, which the library validates."""
    if isinstance(act, bool):
        return int(act)
    if act is None or isinstance(act, str):
        if act not in _ACT_NAMES:
            raise RuntimeError("activation %r has no kernel (None, 'relu' or 'elu')" % (act,))
        return _ACT_NAMES[act]
    return int(act)


def _entry(name, f16):
    """The C-ABI entry of an eval wgmma launch: `name`, or with f16 its one-product `_f16` twin
    (same arguments; include/sonet_b200.h)."""
    return name + "_f16" if f16 else name


def _call(name, *args, kernels=None):
    global LAUNCHES, KERNEL_LAUNCHES
    LAUNCHES += 1
    KERNEL_LAUNCHES += _KERNELS_PER_CALL.get(name, 1) if kernels is None else kernels
    if PROFILE is None:
        _C.check(getattr(_C.lib(), name)(*args), name)
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _C.check(getattr(_C.lib(), name)(*args), name)
    e1.record()
    PROFILE.append((name, e0, e1, args))


def index_max(data, index, K, with_values=False):
    """data [B,C,N] f32, index [B,N] i32 -> max_idx [B,C,K] i32 (and values [B,C,K] f32)."""
    _chk(data, "data", torch.float32)
    _chk(index, "index", torch.int32)
    if data.dim() != 3 or index.dim() != 2 or index.shape[0] != data.shape[0] \
            or index.shape[1] != data.shape[2]:
        raise RuntimeError("index_max: expected data [B,C,N] and index [B,N], got %s and %s"
                           % (tuple(data.shape), tuple(index.shape)))
    B, C, N = data.shape
    with torch.cuda.device(data.device):
        out_idx = torch.empty((B, C, K), dtype=torch.int32, device=data.device)
        out_val = torch.empty((B, C, K), dtype=torch.float32, device=data.device) \
            if with_values else None
        _call("sonet_index_max_f32", _C.ptr(data), _C.ptr(index), B, C, N, int(K),
              _C.ptr(out_idx), _C.ptr(out_val), _stream(data))
    return (out_idx, out_val) if with_values else out_idx


def som_assign(x, node, k, want_i64=False, want_stats=True):
    """x [B,3,N], node [B,3,M] -> dict(min_idx_i32 [B,kN], min_idx_i64?, count, row_max [B,M] i32,
    cluster_mean [B,3,M])."""
    _chk(x, "x", torch.float32)
    _chk(node, "node", torch.float32)
    if x.dim() != 3 or x.shape[1] != 3 or node.dim() != 3 or node.shape[1] != 3 \
            or node.shape[0] != x.shape[0]:
        raise RuntimeError("som_assign: expected x [B,3,N], node [B,3,M], got %s and %s"
                           % (tuple(x.shape), tuple(node.shape)))
    B, _, N = x.shape
    M = node.shape[2]
    dev = x.device
    with torch.cuda.device(dev):
        idx32 = torch.empty((B, k * N), dtype=torch.int32, device=dev)
        idx64 = torch.empty((B, k * N), dtype=torch.int64, device=dev) if want_i64 else None
        count = cmean = None
        row_max = torch.empty((B, M), dtype=torch.int32, device=dev)   # always (cheap flags)
        if want_stats:
            count = torch.empty((B, M), dtype=torch.int32, device=dev)
            cmean = torch.empty((B, 3, M), dtype=torch.float32, device=dev)
        _call("sonet_som_assign", _C.ptr(x), _C.ptr(node), B, N, M, int(k), _C.ptr(idx32),
              _C.ptr(idx64), _C.ptr(count), _C.ptr(row_max), _C.ptr(cmean), _stream(x),
              kernels=2 if want_stats else 1)
    return dict(min_idx_i32=idx32, min_idx_i64=idx64, count=count, row_max=row_max,
                cluster_mean=cmean)


def som_mask(min_idx_i32, M):
    """min_idx [B,kN] i32 -> one-hot mask [B,kN,M] i32."""
    _chk(min_idx_i32, "min_idx", torch.int32)
    B, kN = min_idx_i32.shape
    with torch.cuda.device(min_idx_i32.device):
        mask = torch.empty((B, kN, M), dtype=torch.int32, device=min_idx_i32.device)
        _call("sonet_som_mask", _C.ptr(min_idx_i32), B, kN, int(M), _C.ptr(mask),
              _stream(min_idx_i32))
    return mask


def som_train(x, node_init, weights, lr, want_idx=False):
    """T batch-SOM iterations in one launch (util/som.py:295-366). x [B,3,N]; node_init [3,M]
    (shared) or [B,3,M]; weights [T,M,M]; lr [T] -> node [B,3,M] (and the last assignment
    [B,N] i32: the one computed in iteration T, against the nodes before its update; with T = 0
    the assignment against node_init, and the nodes pass through unchanged)."""
    _chk(x, "x", torch.float32)
    _chk(node_init, "node_init", torch.float32)
    _chk(weights, "weights", torch.float32)
    _chk(lr, "lr", torch.float32)
    B, C, N = x.shape
    M = node_init.shape[-1]
    T = weights.shape[0]
    batched = node_init.dim() == 3
    if C != 3 or node_init.shape[-2] != 3 or (batched and node_init.shape[0] != B) \
            or tuple(weights.shape[1:]) != (M, M) or lr.numel() != T:
        raise RuntimeError("som_train: expected x [B,3,N], node_init [3,M]|[B,3,M], weights [T,M,M], "
                           "lr [T]; got %s %s %s %s" % (tuple(x.shape), tuple(node_init.shape),
                                                        tuple(weights.shape), tuple(lr.shape)))
    with torch.cuda.device(x.device):
        out = torch.empty((B, 3, M), dtype=torch.float32, device=x.device)
        idx = torch.empty((B, N), dtype=torch.int32, device=x.device) if want_idx else None
        _call("sonet_som_train", _C.ptr(x), _C.ptr(node_init), int(batched), _C.ptr(weights),
              _C.ptr(lr), T, B, N, M, _C.ptr(out), _C.ptr(idx), _stream(x))
    return (out, idx) if want_idx else out


def augment(pc, sn, som, rot1=None, rot2=None, scale=None, shift=None, jitter_pc=(0.0, 1.0),
            jitter_sn=(0.0, 1.0), jitter_som=(0.0, 1.0), noise_pc=None, noise_sn=None,
            noise_som=None, seed=0):
    """One-launch batch augmentation (csrc/augment.cu). pc, sn [B,3,N], som [B,3,M] f32 (sn / som
    may be None); rot1/rot2 [B,3,3], scale [B], shift [B,3], noise_* [B,P,3]: float64 device
    tensors or None. jitter_* = (sigma, clip). -> (pc', sn', som')."""
    _chk(pc, "pc", torch.float32)
    _chk(sn, "sn", torch.float32, optional=True)
    _chk(som, "som", torch.float32, optional=True)
    for t, n in ((rot1, "rot1"), (rot2, "rot2"), (scale, "scale"), (shift, "shift"),
                 (noise_pc, "noise_pc"), (noise_sn, "noise_sn"), (noise_som, "noise_som")):
        _chk(t, n, torch.float64, optional=True)
    B, _, N = pc.shape
    M = 0 if som is None else som.shape[2]
    for t, shp, n in ((rot1, (B, 3, 3), "rot1"), (rot2, (B, 3, 3), "rot2"), (scale, (B,), "scale"),
                      (shift, (B, 3), "shift"), (noise_pc, (B, N, 3), "noise_pc"),
                      (noise_sn, (B, N, 3), "noise_sn"), (noise_som, (B, M, 3), "noise_som")):
        if t is not None and tuple(t.shape) != shp:
            raise RuntimeError("augment: %s must have shape %s, got %s" % (n, shp, tuple(t.shape)))
    with torch.cuda.device(pc.device):
        po = torch.empty_like(pc)
        so = torch.empty_like(sn) if sn is not None else None
        mo = torch.empty_like(som) if som is not None else None
        _call("sonet_augment_f32", _C.ptr(pc), _C.ptr(sn), _C.ptr(som), B, N, M, _C.ptr(rot1),
              _C.ptr(rot2), _C.ptr(scale), _C.ptr(shift), float(jitter_pc[0]), float(jitter_pc[1]),
              float(jitter_sn[0]), float(jitter_sn[1]), float(jitter_som[0]), float(jitter_som[1]),
              _C.ptr(noise_pc), _C.ptr(noise_sn), _C.ptr(noise_som), int(seed) & (2 ** 64 - 1),
              _C.ptr(po), _C.ptr(so), _C.ptr(mo), _stream(pc))
    return po, so, mo


# point-selection rules of the C-ABI (SONET_SAMPLE_*, include/sonet_b200.h)
SAMPLE_SUBSET = _C.CONSTANTS["SONET_SAMPLE_SUBSET"]
SAMPLE_FILL = _C.CONSTANTS["SONET_SAMPLE_FILL"]
SAMPLE_MAX_P = _C.CONSTANTS["SONET_SAMPLE_MAX_P"]      # largest cloud of the in-kernel draws


def sample_points(data, offsets, cloud_ids, N, rule, max_P, labels=None, indices=None, seed=0):
    """The loaders' random choice of N points per cloud (csrc/sample_points.cu) from a ragged
    dataset on the device: data [sum P, 6] f32, offsets [S+1] i64, cloud_ids [B] i64, labels
    [sum P] i32 or None; indices [B,N] i32 (given source positions) or None (in-kernel draws keyed
    by `seed`). -> (pc [B,3,N], sn [B,3,N], seg [B,N] i64 or None)."""
    _chk(data, "data", torch.float32)
    _chk(offsets, "offsets", torch.int64)
    _chk(cloud_ids, "cloud_ids", torch.int64)
    _chk(labels, "labels", torch.int32, optional=True)
    _chk(indices, "indices", torch.int32, optional=True)
    if data.dim() != 2 or data.shape[1] != 6 or offsets.dim() != 1 or cloud_ids.dim() != 1:
        raise RuntimeError("sample_points: expected data [sum P, 6], offsets [S+1], cloud_ids [B]; "
                           "got %s %s %s" % (tuple(data.shape), tuple(offsets.shape),
                                             tuple(cloud_ids.shape)))
    B, N = cloud_ids.shape[0], int(N)
    if labels is not None and labels.shape != (data.shape[0],):
        raise RuntimeError("sample_points: labels must have shape (%d,)" % data.shape[0])
    if indices is not None and tuple(indices.shape) != (B, N):
        raise RuntimeError("sample_points: indices must have shape %s" % ((B, N),))
    dev = data.device
    with torch.cuda.device(dev):
        pc = torch.empty((B, 3, N), dtype=torch.float32, device=dev)
        sn = torch.empty((B, 3, N), dtype=torch.float32, device=dev)
        seg = torch.empty((B, N), dtype=torch.int64, device=dev) if labels is not None else None
        _call("sonet_sample_points_f32", _C.ptr(data), _C.ptr(offsets), offsets.shape[0] - 1,
              _C.ptr(labels), _C.ptr(cloud_ids), B, N, int(max_P), int(rule), _C.ptr(indices),
              int(seed) & (2 ** 64 - 1), _C.ptr(pc), _C.ptr(sn), _C.ptr(seg), _stream(data))
    return pc, sn, seg


MESH_MAX_N = _C.CONSTANTS["SONET_MESH_MAX_N"]      # largest sample count per mesh


def mesh_sample(verts, v_off, faces, f_off, mesh_ids, N, draws=None, seed=0, want_faces=False,
                want_area=False):
    """Area-weighted surface sampling of B meshes (csrc/mesh_sample.cu): verts [sum V, 3] f64 with
    v_off [B+1] i64, faces [sum F, 3] i32 (mesh-local vertex indices) with f_off [B+1] i64,
    mesh_ids [B] i64 (the key of the in-kernel draws); draws [B*N, 3] f64 (r, u, v) or None.
    -> (out [B*N, 6] f32 xyz | normal, face [B*N] i32 or None, area [B] f64 or None); a mesh
    with no face of positive finite area gets NaN rows."""
    _chk(verts, "verts", torch.float64)
    _chk(v_off, "v_off", torch.int64)
    _chk(faces, "faces", torch.int32)
    _chk(f_off, "f_off", torch.int64)
    _chk(mesh_ids, "mesh_ids", torch.int64)
    _chk(draws, "draws", torch.float64, optional=True)
    B, N = mesh_ids.shape[0] if mesh_ids.dim() == 1 else -1, int(N)
    if verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3 \
            or B < 0 or tuple(v_off.shape) != (B + 1,) or tuple(f_off.shape) != (B + 1,):
        raise RuntimeError("mesh_sample: expected verts [V,3], faces [F,3], mesh_ids [B], v_off and "
                           "f_off [B+1]; got %s %s %s %s %s" % (
                               tuple(verts.shape), tuple(faces.shape), tuple(mesh_ids.shape),
                               tuple(v_off.shape), tuple(f_off.shape)))
    if draws is not None and tuple(draws.shape) != (B * N, 3):
        raise RuntimeError("mesh_sample: draws must have shape %s" % ((B * N, 3),))
    dev = mesh_ids.device
    total_F = faces.shape[0]
    with torch.cuda.device(dev):
        nbytes = int(_C.lib().sonet_mesh_sample_scratch_bytes(B, total_F))
        _C.check(0 if nbytes >= 0 else nbytes, "sonet_mesh_sample_scratch_bytes")
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        out = torch.empty((B * N, 6), dtype=torch.float32, device=dev)
        face = torch.empty((B * N,), dtype=torch.int32, device=dev) if want_faces else None
        area = torch.empty((B,), dtype=torch.float64, device=dev) if want_area else None
        _call("sonet_mesh_sample_f32", _C.ptr(verts), _C.ptr(v_off), verts.shape[0], _C.ptr(faces),
              _C.ptr(f_off), total_F, _C.ptr(mesh_ids), B, N, _C.ptr(draws),
              int(seed) & (2 ** 64 - 1), _C.ptr(scratch), nbytes, _C.ptr(out), _C.ptr(face),
              _C.ptr(area), _stream(mesh_ids), kernels=4)
    return out, face, area


POINT_KNN_MAX_K = _C.CONSTANTS["SONET_POINT_KNN_MAX_K"]
# sign rules of the estimated normals (SONET_NORMALS_*, include/sonet_b200.h)
NORMALS_CANONICAL = _C.CONSTANTS["SONET_NORMALS_CANONICAL"]
NORMALS_AWAY_FROM_CENTROID = _C.CONSTANTS["SONET_NORMALS_AWAY_FROM_CENTROID"]
NORMALS_TOWARD_VIEWPOINT = _C.CONSTANTS["SONET_NORMALS_TOWARD_VIEWPOINT"]


def _rows_arg(data, what):
    """(T, stride) of a point-major [T, stride] f32 tensor whose rows may be longer than xyz."""
    _chk(data, "data", torch.float32)
    if data.dim() != 2 or data.shape[1] < 3:
        raise RuntimeError("%s: expected data [T, >=3], got %s" % (what, tuple(data.shape)))
    return data.shape[0], data.shape[1]


def point_knn(data, offsets, K, want_dist=False):
    """Exact K nearest neighbours of every point within its own cloud (csrc/point_normals.cu):
    data [T, stride>=3] f32 (xyz in columns 0..2), offsets [S+1] i64. -> (idx [T, K] i32
    cloud-local, dist [T, K] f32 or None); ascending distance, lowest index on ties, NaN last."""
    T, stride = _rows_arg(data, "point_knn")
    _chk(offsets, "offsets", torch.int64)
    S = offsets.shape[0] - 1
    dev = data.device
    with torch.cuda.device(dev):
        idx = torch.empty((T, int(K)), dtype=torch.int32, device=dev)
        dist = torch.empty((T, int(K)), dtype=torch.float32, device=dev) if want_dist else None
        _call("sonet_point_knn_f32", _C.ptr(data), T, stride, _C.ptr(offsets), S, int(K),
              _C.ptr(idx), _C.ptr(dist), _stream(data), kernels=int(S > 0))
    return idx, dist


def estimate_normals(data, offsets, idx, orient, view=None, out=None, want_curvature=False):
    """PCA normals of every point from its neighbours idx [T, K] i32 (point_knn's) with the sign
    rule `orient` (NORMALS_*); view [S, 3] f32 for NORMALS_TOWARD_VIEWPOINT. out: [T, 3] f32 whose
    rows may be strided (e.g. data[:, 3:6]), or None for a new tensor. -> (normals, curvature [T]
    or None); a degenerate neighbourhood gives the zero vector and NaN curvature."""
    T, stride = _rows_arg(data, "estimate_normals")
    _chk(offsets, "offsets", torch.int64)
    _chk(idx, "idx", torch.int32)
    _chk(view, "view", torch.float32, optional=True)
    S = offsets.shape[0] - 1
    if idx.dim() != 2 or idx.shape[0] != T:
        raise RuntimeError("estimate_normals: idx must be [%d, K], got %s" % (T, tuple(idx.shape)))
    if view is not None and tuple(view.shape) != (S, 3):
        raise RuntimeError("estimate_normals: view must be [%d, 3], got %s" % (S, tuple(view.shape)))
    dev = data.device
    if out is not None and (not out.is_cuda or out.dtype != torch.float32 or out.dim() != 2
                            or tuple(out.shape) != (T, 3) or out.stride(1) != 1
                            or (T > 1 and out.stride(0) < 3)):
        raise RuntimeError("estimate_normals: out must be a CUDA f32 [T, 3] view with unit column "
                           "stride, got %s with strides %s" % (tuple(out.shape), out.stride()))
    with torch.cuda.device(dev):
        normals = torch.empty((T, 3), dtype=torch.float32, device=dev) if out is None else out
        curv = torch.empty((T,), dtype=torch.float32, device=dev) if want_curvature else None
        scratch, nbytes = None, 0
        if orient == NORMALS_AWAY_FROM_CENTROID:
            nbytes = int(_C.lib().sonet_point_normals_scratch_bytes(S))
            _C.check(0 if nbytes >= 0 else nbytes, "sonet_point_normals_scratch_bytes")
            scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        _call("sonet_point_normals_f32", _C.ptr(data), T, stride, _C.ptr(offsets), S, _C.ptr(idx),
              idx.shape[1], int(orient), _C.ptr(view), _C.ptr(scratch), nbytes, _C.ptr(normals),
              max(normals.stride(0), 3), _C.ptr(curv), _stream(data),
              kernels=(S > 0) * (1 + (orient == NORMALS_AWAY_FROM_CENTROID)))
    return normals, curv


POINT_ORIENT_MAX_POINTS = _C.CONSTANTS["SONET_POINT_ORIENT_MAX_POINTS"]
POINT_ORIENT_MAX_ROUNDS = _C.CONSTANTS["SONET_POINT_ORIENT_MAX_ROUNDS"]


def orient_rounds(max_points):
    """The rounds sonet_point_normals_orient_f32 schedules: ceil(log2(max_points)), 0 below 2."""
    return 0 if max_points <= 1 else int(max_points - 1).bit_length()


def orient_normals(data, offsets, idx, normals, anchor, view=None, max_points=None,
                   want_component=False, scratch=None):
    """Consistent normal signs within each cloud, propagated along the minimum spanning tree of the
    k-NN graph idx [T, K] i32 (point_knn's, cloud-local) and anchored per component by `anchor`
    (NORMALS_AWAY_FROM_CENTROID or NORMALS_TOWARD_VIEWPOINT with view [S, 3] f32). normals: a [T, 3]
    f32 CUDA view with unit column stride (e.g. data[:, 3:6]), negated in place where the tree says
    so. max_points: the largest cloud, read from the offsets on the host when None. scratch: a uint8
    CUDA tensor of at least sonet_point_normals_orient_scratch_bytes(T, S) bytes, or None for a new
    one; its first POINT_ORIENT_MAX_ROUNDS int32 then say which rounds merged components.
    -> (normals, component [T] i32 or None): the cloud-local index of each vertex's anchor, -1 off
    the graph."""
    T, stride = _rows_arg(data, "orient_normals")
    _chk(offsets, "offsets", torch.int64)
    _chk(idx, "idx", torch.int32)
    _chk(view, "view", torch.float32, optional=True)
    S = offsets.shape[0] - 1
    if idx.dim() != 2 or idx.shape[0] != T:
        raise RuntimeError("orient_normals: idx must be [%d, K], got %s" % (T, tuple(idx.shape)))
    if view is not None and tuple(view.shape) != (S, 3):
        raise RuntimeError("orient_normals: view must be [%d, 3], got %s" % (S, tuple(view.shape)))
    if (not torch.is_tensor(normals) or not normals.is_cuda or normals.dtype != torch.float32
            or normals.dim() != 2 or tuple(normals.shape) != (T, 3) or normals.stride(1) != 1
            or (T > 1 and normals.stride(0) < 3)):
        raise RuntimeError("orient_normals: normals must be a CUDA f32 [T, 3] view with unit column "
                           "stride, got %s" % (tuple(normals.shape) if torch.is_tensor(normals)
                                               else type(normals).__name__,))
    if max_points is None:
        off = offsets.cpu().clamp(0, T)
        max_points = int((off[1:] - off[:-1]).clamp(min=0).max()) if S > 0 else 0
    dev = data.device
    with torch.cuda.device(dev):
        comp = torch.empty((T,), dtype=torch.int32, device=dev) if want_component else None
        nbytes = int(_C.lib().sonet_point_normals_orient_scratch_bytes(T, S))
        _C.check(0 if nbytes >= 0 else nbytes, "sonet_point_normals_orient_scratch_bytes")
        if scratch is None:
            scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        elif not (scratch.is_cuda and scratch.dtype == torch.uint8 and scratch.numel() >= nbytes):
            raise RuntimeError("orient_normals: scratch must be a CUDA uint8 tensor of >= %d bytes"
                               % nbytes)
        launches = 1 + 5 * orient_rounds(int(max_points)) + 3 + (anchor == NORMALS_AWAY_FROM_CENTROID)
        _call("sonet_point_normals_orient_f32", _C.ptr(data), T, stride, _C.ptr(offsets), S,
              int(max_points), _C.ptr(idx), idx.shape[1], int(anchor), _C.ptr(view), _C.ptr(scratch),
              nbytes, _C.ptr(normals), max(normals.stride(0), 3), _C.ptr(comp), _stream(data),
              kernels=(S > 0) * launches)
    return normals, comp


def som_decenter(x, sn, cluster_mean, min_idx_i32, k, want_centers=False):
    """-> (x_aug [B,3(+3),kN], centers [B,3,kN] or None)."""
    _chk(x, "x", torch.float32)
    _chk(sn, "sn", torch.float32, optional=True)
    _chk(cluster_mean, "cluster_mean", torch.float32)
    _chk(min_idx_i32, "min_idx", torch.int32)
    B, _, N = x.shape
    M = cluster_mean.shape[2]
    kN = k * N
    with torch.cuda.device(x.device):
        x_aug = torch.empty((B, 6 if sn is not None else 3, kN), dtype=torch.float32,
                            device=x.device)
        centers = torch.empty((B, 3, kN), dtype=torch.float32, device=x.device) \
            if want_centers else None
        _call("sonet_som_decenter", _C.ptr(x), _C.ptr(sn), _C.ptr(cluster_mean),
              _C.ptr(min_idx_i32), B, N, M, int(k), _C.ptr(centers), _C.ptr(x_aug), _stream(x))
    return x_aug, centers


def pointwise_layer(x0, Wt, scale, shift, act, x1=None, addend=None, gidx=None, out=None):
    """x0 [B,C0,P] (+ x1 [B,C1,P]) -> [B,Cout,P]; Wt [C0+C1,Cout] transposed folded weights;
    act: activation (act_code)."""
    _chk(x0, "x0", torch.float32)
    _chk(x1, "x1", torch.float32, optional=True)
    _chk(Wt, "Wt", torch.float32)
    _chk(scale, "scale", torch.float32, optional=True)
    _chk(shift, "shift", torch.float32, optional=True)
    _chk(addend, "addend", torch.float32, optional=True)
    _chk(gidx, "gidx", torch.int32, optional=True)
    B, C0, P = x0.shape
    C1 = 0 if x1 is None else x1.shape[1]
    if Wt.shape[0] != C0 + C1:
        raise RuntimeError("pointwise_layer: Wt has %d input channels, inputs have %d"
                           % (Wt.shape[0], C0 + C1))
    Cout = Wt.shape[1]
    G = 0 if addend is None else addend.shape[2]
    with torch.cuda.device(x0.device):
        if out is None:
            out = torch.empty((B, Cout, P), dtype=torch.float32, device=x0.device)
        _call("sonet_pointwise_layer_f32", _C.ptr(x0), C0, _C.ptr(x1), C1, B, P, _C.ptr(Wt),
              _C.ptr(scale), _C.ptr(shift), Cout, act_code(act), _C.ptr(addend), _C.ptr(gidx), G,
              _C.ptr(out), _stream(x0))
    return out


def linear(x, W, scale, shift, act):
    """x [B,Cin], W [Cout,Cin] -> [B,Cout]; act: activation (act_code)."""
    _chk(x, "x", torch.float32)
    _chk(W, "W", torch.float32)
    _chk(scale, "scale", torch.float32, optional=True)
    _chk(shift, "shift", torch.float32, optional=True)
    B, Cin = x.shape
    Cout = W.shape[0]
    with torch.cuda.device(x.device):
        out = torch.empty((B, Cout), dtype=torch.float32, device=x.device)
        _call("sonet_linear_f32", _C.ptr(x), B, Cin, _C.ptr(W), _C.ptr(scale), _C.ptr(shift),
              Cout, act_code(act), _C.ptr(out), _stream(x))
    return out


def rowmax(t):
    """max over the last dim of a contiguous tensor."""
    _chk(t, "input", torch.float32)
    L = t.shape[-1]
    R = t.numel() // max(L, 1)
    with torch.cuda.device(t.device):
        out = torch.empty(t.shape[:-1], dtype=torch.float32, device=t.device)
        _call("sonet_rowmax_f32", _C.ptr(t), R, L, _C.ptr(out), _stream(t))
    return out


def knn_gather(src, idx, K=None):
    """src [B,C,M], idx [B,M,K'] i64 -> [B,C,M,K]."""
    _chk(src, "som_node", torch.float32)
    _chk(idx, "som_node_knn_I", torch.int64)
    B, C, M = src.shape
    Kstride = idx.shape[2]
    K = Kstride if K is None else K
    with torch.cuda.device(src.device):
        out = torch.empty((B, C, M, K), dtype=torch.float32, device=src.device)
        _call("sonet_knn_gather_f32", _C.ptr(src), _C.ptr(idx), B, C, M, K, Kstride, _C.ptr(out),
              _stream(src))
    return out


def knn_assemble(coord, feat, idx, K, center_type, want_x_aug=True):
    """-> (center [B,3,M], x_aug [B,3+C,M*K], or None with want_x_aug=False)."""
    _chk(coord, "coordinate", torch.float32)
    _chk(feat, "x", torch.float32)
    _chk(idx, "knn_I", torch.int64)
    B, C, M = feat.shape
    Kstride = idx.shape[2]
    ct = {"avg": 0, "center": 1}[center_type]
    with torch.cuda.device(feat.device):
        center = torch.empty((B, 3, M), dtype=torch.float32, device=feat.device)
        x_aug = torch.empty((B, 3 + C, M * K), dtype=torch.float32, device=feat.device) \
            if want_x_aug else None
        _call("sonet_knn_assemble_f32", _C.ptr(coord), _C.ptr(feat), _C.ptr(idx), B, C, M, int(K),
              Kstride, ct, _C.ptr(center), _C.ptr(x_aug), _stream(feat))
    return center, x_aug


def node_knn(coord, K):
    _chk(coord, "coordinate", torch.float32)
    B, _, M = coord.shape
    with torch.cuda.device(coord.device):
        idx = torch.empty((B, M, K), dtype=torch.int64, device=coord.device)
        _call("sonet_node_knn", _C.ptr(coord), B, M, int(K), _C.ptr(idx), _stream(coord))
    return idx


def gather_points(src, gidx):
    """src [B,C,M], gidx [B,P] i32 -> [B,C,P]."""
    _chk(src, "src", torch.float32)
    _chk(gidx, "gidx", torch.int32)
    B, C, M = src.shape
    P = gidx.shape[1]
    with torch.cuda.device(src.device):
        out = torch.empty((B, C, P), dtype=torch.float32, device=src.device)
        _call("sonet_gather_points_f32", _C.ptr(src), _C.ptr(gidx), B, C, M, P, _C.ptr(out),
              _stream(src))
    return out


def kcopy_mean(t, k):
    """[B,C,k*N] -> [B,C,N], mean of the k stacked copies."""
    _chk(t, "input", torch.float32)
    B, C, kN = t.shape
    N = kN // k
    with torch.cuda.device(t.device):
        out = torch.empty((B, C, N), dtype=torch.float32, device=t.device)
        _call("sonet_kcopy_mean_f32", _C.ptr(t), B, C, N, int(k), _C.ptr(out), _stream(t))
    return out


# reduction codes of sonet_instance_norm_f32 (SONET_REDUCE_*, include/sonet_b200.h)
REDUCE_NONE = _C.CONSTANTS["SONET_REDUCE_NONE"]
REDUCE_KCOPY_MEAN = _C.CONSTANTS["SONET_REDUCE_KCOPY_MEAN"]
REDUCE_GROUP_MAX = _C.CONSTANTS["SONET_REDUCE_GROUP_MAX"]


def instance_norm(z, gamma, beta, eps, act, kcopy=None, group_max=None, save_stats=False, out=None):
    """Instance norm + activation of z [B,C,P] per row (b, c): act(gamma*(z-mean)*invstd + beta)
    with the row's biased statistics (nn.InstanceNorm1d/2d, affine, no running statistics).
    gamma, beta [C] or None (identity); act: activation (act_code). kcopy=k: the mean over the k
    stacked copies, out [B,C,P/k]; group_max=K: the max over consecutive groups of K, out
    [B,C,P/K]. out: the output tensor (may be z itself without a reduction). save_stats: also
    return the row statistics (mean, invstd), each [B,C]."""
    _chk(z, "z", torch.float32)
    _chk(gamma, "gamma", torch.float32, optional=True)
    _chk(beta, "beta", torch.float32, optional=True)
    if z.dim() != 3:
        raise RuntimeError("instance_norm: expected z [B,C,P], got %s" % (tuple(z.shape),))
    if kcopy is not None and group_max is not None:
        raise RuntimeError("instance_norm: kcopy and group_max exclude each other")
    B, C, P = z.shape
    reduce, k = REDUCE_NONE, 1
    if kcopy is not None:
        reduce, k = REDUCE_KCOPY_MEAN, int(kcopy)
    elif group_max is not None:
        reduce, k = REDUCE_GROUP_MAX, int(group_max)
    dev = z.device
    _chk(out, "out", torch.float32, optional=True)
    if out is not None and out.numel() != B * C * (P // max(k, 1)):
        raise RuntimeError("instance_norm: out has %d elements, expected %d"
                           % (out.numel(), B * C * (P // max(k, 1))))
    with torch.cuda.device(dev):
        if out is None:
            out = torch.empty((B, C, P // max(k, 1)), dtype=torch.float32, device=dev)
        mean = invstd = None
        if save_stats:
            mean = torch.empty((B, C), dtype=torch.float32, device=dev)
            invstd = torch.empty((B, C), dtype=torch.float32, device=dev)
        _call("sonet_instance_norm_f32", _C.ptr(z), _C.ptr(gamma), _C.ptr(beta), B, C, P, float(eps),
              act_code(act), reduce, k, _C.ptr(out), _C.ptr(mean), _C.ptr(invstd), _stream(z))
    return (out, mean, invstd) if save_stats else out


def seg_loss(score, target, size_average=True):
    """score [B,C,N] f32, target [B,N] int64 -> scalar loss tensor (mean/sum of the per-point NLL
    of log_softmax over the class axis, models/losses.py:30-43)."""
    _chk(score, "score", torch.float32)
    _chk(target, "target", torch.int64)
    B, C, N = score.shape
    if tuple(target.shape) != (B, N):
        raise RuntimeError("seg_loss: target shape %s does not match scores %s"
                           % (tuple(target.shape), tuple(score.shape)))
    lib = _C.lib()
    with torch.cuda.device(score.device):
        scratch = torch.empty(int(lib.sonet_seg_loss_scratch_bytes(B, N)), dtype=torch.uint8,
                              device=score.device)
        loss = torch.empty((), dtype=torch.float32, device=score.device)
        _call("sonet_seg_loss_f32", _C.ptr(score), _C.ptr(target), B, C, N, int(bool(size_average)),
              _C.ptr(scratch), _C.ptr(loss), _stream(score), kernels=2)
    return loss


def seg_loss_ragged(score, target, offsets):
    """seg_loss over whole shapes of any size: score [T,C] f32 point-major, target [T] int64,
    offsets [B+1] int64 on score's device (cloud b is rows offsets[b] .. offsets[b+1]) -> (loss,
    loss_array [B]): the mean NLL over every counted point of the batch (with equal sizes P,
    seg_loss's bits on the scores laid out [B,C,P]) and each cloud's own mean (NaN for a cloud with
    no counted point). Copies the offsets to the host (one synchronisation) and refuses bad offsets
    before any launch."""
    _chk(score, "score", torch.float32)
    _chk(target, "target", torch.int64)
    _chk(offsets, "offsets", torch.int64)
    if score.dim() != 2 or score.shape[1] < 1 or tuple(target.shape) != (score.shape[0],):
        raise RuntimeError("seg_loss_ragged: expected score [T,C] with C >= 1 and target [T], got "
                           "%s and %s" % (tuple(score.shape), tuple(target.shape)))
    if target.device != score.device or offsets.device != score.device:
        raise RuntimeError("seg_loss_ragged: score, target and offsets must be on one device "
                           "(got %s, %s, %s)" % (score.device, target.device, offsets.device))
    T, C = score.shape
    if offsets.dim() != 1 or offsets.numel() < 2:
        raise RuntimeError("seg_loss_ragged: offsets must be [B+1] with B >= 1 (got %s)"
                           % (tuple(offsets.shape),))
    B = offsets.numel() - 1
    off = ragged_offsets(offsets, T, B)
    lib = _C.lib()
    dev = score.device
    with torch.cuda.device(dev):
        scratch = torch.empty(int(lib.sonet_seg_loss_ragged_scratch_bytes(B, T)), dtype=torch.uint8,
                              device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        loss_array = torch.empty((B,), dtype=torch.float32, device=dev)
        _call("sonet_seg_loss_ragged_f32", _C.ptr(score), _C.ptr(target), _C.ptr(offsets),
              off.ctypes.data, B, C, T, _C.ptr(scratch), _C.ptr(loss), _C.ptr(loss_array),
              _stream(score), kernels=3)
    return loss, loss_array


# ShapeNetPart: category -> its part ids, in the reference's order (models/losses.py:74-91)
SHAPENET_PART_TABLE = ((0, 1, 2, 3), (4, 5), (6, 7), (8, 9, 10, 11), (12, 13, 14, 15), (16, 17, 18),
                       (19, 20, 21), (22, 23), (24, 25, 26, 27), (28, 29), (30, 31, 32, 33, 34, 35),
                       (36, 37), (38, 39, 40), (41, 42, 43), (44, 45, 46), (47, 48, 49))
SEG_IOU_MAX_PARTS = 256
_PART_TABLES = {}


def part_table_csr(table, C, device):
    """Validated (offsets [K+1], ids) int32 tensors of a category -> part ids table on `device`,
    uploaded once per (table, device) and cached: later calls neither copy nor allocate."""
    table = SHAPENET_PART_TABLE if table is None else tuple(tuple(int(p) for p in parts)
                                                            for parts in table)
    key = (table, C, str(device))
    hit = _PART_TABLES.get(key)
    if hit is None:
        if not table:
            raise RuntimeError("seg_iou: the part table has no category")
        for k, parts in enumerate(table):
            if not 1 <= len(parts) <= SEG_IOU_MAX_PARTS:
                raise RuntimeError("seg_iou: category %d has %d parts (1..%d allowed)"
                                   % (k, len(parts), SEG_IOU_MAX_PARTS))
            if any(not 0 <= p < C for p in parts):
                raise RuntimeError("seg_iou: category %d has a part id outside [0, C=%d)" % (k, C))
        offsets = [0]
        for parts in table:
            offsets.append(offsets[-1] + len(parts))
        ids = [p for parts in table for p in parts]
        hit = (torch.tensor(offsets, dtype=torch.int32, device=device),
               torch.tensor(ids, dtype=torch.int32, device=device), len(table))
        _PART_TABLES[key] = hit
    return hit


def _seg_iou_args(score, seg, label):
    if score.dim() != 3 or tuple(seg.shape) != (score.shape[0], score.shape[2]) \
            or tuple(label.shape) != (score.shape[0],):
        raise RuntimeError("seg_iou: expected score [B,C,N], seg [B,N], label [B], got %s, %s, %s"
                           % (tuple(score.shape), tuple(seg.shape), tuple(label.shape)))
    return score.shape


def seg_iou(score, seg, label, table=None, want_pred=False, want_correct=False):
    """Part-segmentation IoU of every cloud (models/losses.py:73-116) in one launch, no sync.
    score [B,C,N] f32, seg [B,N] int64, label [B] int64 (CUDA, contiguous); table: category ->
    part ids (default SHAPENET_PART_TABLE). Returns (iou_shape [B] f64, pred [B,N] int64 or None,
    correct [B] int32 or None). A label outside the table gives iou_shape[b] = NaN (the device
    cannot raise without a sync). The table is uploaded on its first use per device, so a call
    captured in a CUDA graph needs one call with that table before the capture."""
    _chk(score, "score", torch.float32)
    _chk(seg, "seg", torch.int64)
    _chk(label, "label", torch.int64)
    B, C, N = _seg_iou_args(score, seg, label)
    dev = score.device
    with torch.cuda.device(dev):
        offsets, ids, K = part_table_csr(table, C, dev)
        iou = torch.empty((B,), dtype=torch.float64, device=dev)
        pred = torch.empty((B, N), dtype=torch.int64, device=dev) if want_pred else None
        correct = torch.empty((B,), dtype=torch.int32, device=dev) if want_correct else None
        _call("sonet_seg_iou_f32", _C.ptr(score), _C.ptr(seg), _C.ptr(label), B, C, N,
              _C.ptr(offsets), _C.ptr(ids), K, _C.ptr(iou), _C.ptr(pred), _C.ptr(correct),
              _stream(score))
    return iou, pred, correct


def ragged_offsets(offsets, total, B=None):
    """Host copy (numpy int64) of ragged offsets [B+1], checked: 0 first, `total` last, non-decreasing;
    B, when given, is the expected number of shapes."""
    if offsets.dtype != torch.int64 or offsets.dim() != 1 or offsets.numel() < 1:
        raise RuntimeError("offsets must be a 1-D int64 tensor [B+1] (got %s %s)"
                           % (offsets.dtype, tuple(offsets.shape)))
    if B is not None and offsets.numel() != B + 1:
        raise RuntimeError("offsets has %d entries, the batch needs B+1 = %d"
                           % (offsets.numel(), B + 1))
    off = offsets.detach().cpu().numpy()
    if off[0] != 0 or off[-1] != total or (off[1:] < off[:-1]).any():
        raise RuntimeError("offsets must run from 0 to %d without decreasing" % total)
    return off


def seg_iou_ragged(score, seg, label, offsets, table=None, want_pred=False, want_correct=False):
    """seg_iou over every point of each shape, one launch: score [T,C] f32, seg [T] int64, label [B]
    int64, offsets [B+1] int64 (CUDA, contiguous; shape b owns points offsets[b] .. offsets[b+1]).
    Returns (iou_shape [B] f64, pred [T] int64 or None, correct [B] int32 or None). The offsets are
    checked by the caller (ragged_offsets); the device marks a shape with bad offsets NaN."""
    _chk(score, "score", torch.float32)
    _chk(seg, "seg", torch.int64)
    _chk(label, "label", torch.int64)
    _chk(offsets, "offsets", torch.int64)
    if score.dim() != 2 or tuple(seg.shape) != (score.shape[0],) or label.dim() != 1 \
            or tuple(offsets.shape) != (label.shape[0] + 1,):
        raise RuntimeError("seg_iou_ragged: expected score [T,C], seg [T], label [B], offsets [B+1], "
                           "got %s, %s, %s, %s" % (tuple(score.shape), tuple(seg.shape),
                                                   tuple(label.shape), tuple(offsets.shape)))
    T, C = score.shape
    B = label.shape[0]
    dev = score.device
    with torch.cuda.device(dev):
        poff, ids, K = part_table_csr(table, C, dev)
        iou = torch.empty((B,), dtype=torch.float64, device=dev)
        pred = torch.empty((T,), dtype=torch.int64, device=dev) if want_pred else None
        correct = torch.empty((B,), dtype=torch.int32, device=dev) if want_correct else None
        _call("sonet_seg_iou_ragged_f32", _C.ptr(score), _C.ptr(seg), _C.ptr(label), _C.ptr(offsets),
              B, C, T, _C.ptr(poff), _C.ptr(ids), K, _C.ptr(iou), _C.ptr(pred), _C.ptr(correct),
              _stream(score))
    return iou, pred, correct


def seg_points_assign(points, offsets, node, cluster_mean, k, with_sn, row0, rows, rows_pad):
    """Rows [row0, row0+rows) of the ragged set points [T,6] (offsets [B+1] int64, checked by the
    caller) -> (gidx [1,k*rows_pad] int32 flat cloud*M+node ids, x_aug [1,3(+3),k*rows_pad],
    pt [1,9(+3),k*rows_pad]), copy-major, padded with zero rows (csrc/seg_points.cu)."""
    _chk(points, "points", torch.float32)
    _chk(offsets, "offsets", torch.int64)
    _chk(node, "node", torch.float32)
    _chk(cluster_mean, "cluster_mean", torch.float32)
    if points.dim() != 2 or points.shape[1] != 6 or node.dim() != 3 or node.shape[1] != 3 \
            or tuple(cluster_mean.shape) != tuple(node.shape) \
            or tuple(offsets.shape) != (node.shape[0] + 1,):
        raise RuntimeError("seg_points_assign: expected points [T,6], offsets [B+1], node and "
                           "cluster_mean [B,3,M], got %s, %s, %s, %s"
                           % (tuple(points.shape), tuple(offsets.shape), tuple(node.shape),
                              tuple(cluster_mean.shape)))
    B, _, M = node.shape
    cols = k * rows_pad
    dev = points.device
    with torch.cuda.device(dev):
        gidx = torch.empty((1, cols), dtype=torch.int32, device=dev)
        x_aug = torch.empty((1, 6 if with_sn else 3, cols), dtype=torch.float32, device=dev)
        pt = torch.empty((1, 12 if with_sn else 9, cols), dtype=torch.float32, device=dev)
        _call("sonet_seg_points_assign_f32", _C.ptr(points), points.shape[0], _C.ptr(offsets), B,
              _C.ptr(node), _C.ptr(cluster_mean), M, int(k), int(bool(with_sn)), int(row0), int(rows),
              int(rows_pad), _C.ptr(gidx), _C.ptr(x_aug), _C.ptr(pt), _stream(points))
    return gidx, x_aug, pt


def _ragged_args(points, offsets, what):
    _chk(points, "points", torch.float32)
    _chk(offsets, "offsets", torch.int64)
    if points.dim() != 2 or points.shape[1] != 6 or offsets.dim() != 1 or offsets.numel() < 2:
        raise RuntimeError("%s: expected points [T,6] and offsets [B+1], got %s and %s"
                           % (what, tuple(points.shape), tuple(offsets.shape)))
    return points.shape[0], offsets.numel() - 1


def som_assign_ragged(points, offsets, node, k):
    """Ragged clouds (points [T,6], offsets [B+1] checked by the caller) against their loader nodes
    node [B,3,M] -> (min_idx [k*T] i32 cloud-local node of every stacked copy, count [B,M] i32,
    row_max [B,M] i32) (csrc/som_ragged.cu)."""
    T, B = _ragged_args(points, offsets, "som_assign_ragged")
    _chk(node, "node", torch.float32)
    if node.dim() != 3 or node.shape[0] != B or node.shape[1] != 3:
        raise RuntimeError("som_assign_ragged: node must be [%d,3,M] (got %s)" % (B, tuple(node.shape)))
    M = node.shape[2]
    dev = points.device
    with torch.cuda.device(dev):
        idx = torch.empty((k * T,), dtype=torch.int32, device=dev)
        count = torch.empty((B, M), dtype=torch.int32, device=dev)
        row_max = torch.empty((B, M), dtype=torch.int32, device=dev)
        _call("sonet_som_assign_ragged_f32", _C.ptr(points), T, _C.ptr(offsets), B, _C.ptr(node),
              int(M), int(k), _C.ptr(idx), _C.ptr(count), _C.ptr(row_max), _stream(points),
              kernels=1 if T else 0)
    return idx, count, row_max


def som_group_decenter_ragged(points, offsets, min_idx, M, k, with_sn):
    """Cluster statistics + stable (cloud, node) sort + decentring of ragged clouds, one launch ->
    (x_sorted [3(+3),k*T], node_sorted [k*T] i32 flat ids b*M+m, pos0 [B] i32, cluster_mean [B,3,M])."""
    T, B = _ragged_args(points, offsets, "som_group_decenter_ragged")
    _chk(min_idx, "min_idx", torch.int32)
    dev = points.device
    with torch.cuda.device(dev):
        xs = torch.empty((6 if with_sn else 3, k * T), dtype=torch.float32, device=dev)
        ns = torch.empty((k * T,), dtype=torch.int32, device=dev)
        p0 = torch.empty((B,), dtype=torch.int32, device=dev)
        cmean = torch.empty((B, 3, M), dtype=torch.float32, device=dev)
        _call("sonet_som_group_decenter_ragged_f32", _C.ptr(points), T, _C.ptr(offsets), B, int(M),
              int(k), int(bool(with_sn)), _C.ptr(min_idx), _C.ptr(cmean), _C.ptr(xs), _C.ptr(ns),
              _C.ptr(p0), _stream(points))
    return xs, ns, p0, cmean


def som_decenter_ragged(points, offsets, min_idx, cluster_mean, k, with_sn):
    """The decentred stacked copies of ragged clouds in stacked order -> x_aug [1,3(+3),k*T]."""
    T, B = _ragged_args(points, offsets, "som_decenter_ragged")
    _chk(min_idx, "min_idx", torch.int32)
    _chk(cluster_mean, "cluster_mean", torch.float32)
    M = cluster_mean.shape[2]
    dev = points.device
    with torch.cuda.device(dev):
        x_aug = torch.empty((1, 6 if with_sn else 3, k * T), dtype=torch.float32, device=dev)
        _call("sonet_som_decenter_ragged_f32", _C.ptr(points), T, _C.ptr(offsets), B, int(M), int(k),
              int(bool(with_sn)), _C.ptr(min_idx), _C.ptr(cluster_mean), _C.ptr(x_aug),
              _stream(points))
    return x_aug


def pointresnet_tc_pool_ragged(x_sorted, blob, fparams, node_sorted, pos0, M, owner=None, f16=False,
                               act=ACT_RELU):
    """pointresnet_tc_pool(finalize=False) over the sorted copies of a ragged batch, x_sorted
    [Cin,P] with flat node ids node_sorted [P] (som_group_decenter_ragged's) -> (keys [B,384,M] i32,
    p0 [B,384]) for pool_finalize / knn_assemble_pool."""
    act = act_code(act)
    _chk(x_sorted, "x_sorted", torch.float32)
    _chk(blob, "blob", torch.uint8)
    _chk(fparams, "fparams", torch.float32)
    _chk(node_sorted, "node_sorted", torch.int32)
    _chk(pos0, "pos0", torch.int32)
    Cin, P = x_sorted.shape
    B = pos0.shape[0]
    dev = x_sorted.device
    with torch.cuda.device(dev):
        keys = (owner or _DEFAULT_POOL_KEYS).acquire(dev, B, M, _stream(x_sorted))
        p0 = torch.empty((B, 384), dtype=torch.float32, device=dev)
        _call("sonet_pointresnet_tc_pool_ragged_forward", _C.ptr(x_sorted), Cin, P, _C.ptr(blob),
              _C.ptr(fparams), _C.ptr(node_sorted), _C.ptr(pos0), B, int(M), act, int(bool(f16)),
              _C.ptr(keys), _C.ptr(p0), _stream(x_sorted))
    return keys, p0


def index_max_ragged(data, index, offsets, M, k):
    """index_max per cloud of a ragged batch: data [C,k*T] f32 in stacked column order, index [k*T]
    i32 cloud-local node ids, offsets [B+1] -> (out_idx [B,C,M] i32 cloud-local stacked column,
    out_val [B,C,M] f32)."""
    _chk(data, "data", torch.float32)
    _chk(index, "index", torch.int32)
    _chk(offsets, "offsets", torch.int64)
    if data.dim() != 2 or index.dim() != 1 or index.shape[0] != data.shape[1] \
            or index.shape[0] % k != 0 or offsets.dim() != 1 or offsets.numel() < 2:
        raise RuntimeError("index_max_ragged: expected data [C,k*T], index [k*T], offsets [B+1], got "
                           "%s, %s, %s" % (tuple(data.shape), tuple(index.shape), tuple(offsets.shape)))
    C, cols = data.shape
    B = offsets.numel() - 1
    dev = data.device
    with torch.cuda.device(dev):
        out_idx = torch.empty((B, C, M), dtype=torch.int32, device=dev)
        out_val = torch.empty((B, C, M), dtype=torch.float32, device=dev)
        _call("sonet_index_max_ragged_f32", _C.ptr(data), C, cols, _C.ptr(index), _C.ptr(offsets), B,
              cols // k, int(M), int(k), _C.ptr(out_idx), _C.ptr(out_val), _stream(data))
    return out_idx, out_val



def index_max_ragged_backward(grad_out, idx, col_offsets, L):
    """The backward of index_max_ragged's gather: grad_out, idx [B,C,M] (index_max_ragged's out_idx),
    col_offsets [B+1] int64 (cloud b's columns, k*offsets; checked by the caller) -> grad [C,L] f32,
    zero but for grad[c, col_offsets[b] + idx[b,c,m]] += grad_out[b,c,m] in ascending m."""
    _chk(grad_out, "grad_out", torch.float32)
    _chk(idx, "idx", torch.int32)
    _chk(col_offsets, "col_offsets", torch.int64)
    if grad_out.dim() != 3 or tuple(idx.shape) != tuple(grad_out.shape) or col_offsets.dim() != 1 \
            or col_offsets.numel() != grad_out.shape[0] + 1:
        raise RuntimeError("index_max_ragged_backward: expected grad_out and idx [B,C,M], col_offsets "
                           "[B+1], got %s, %s, %s" % (tuple(grad_out.shape), tuple(idx.shape),
                                                      tuple(col_offsets.shape)))
    B, C, M = grad_out.shape
    dev = grad_out.device
    with torch.cuda.device(dev):
        grad = torch.empty((C, int(L)), dtype=torch.float32, device=dev)
        _call("sonet_index_max_ragged_backward_f32", _C.ptr(grad_out), _C.ptr(idx), _C.ptr(col_offsets),
              B, C, M, int(L), _C.ptr(grad), _stream(grad_out), kernels=2)
    return grad


def _bn_ragged_args(x, col_offsets, what):
    _chk(x, "x", torch.float32)
    _chk(col_offsets, "col_offsets", torch.int64)
    if x.dim() == 3 and x.shape[0] == 1:
        x = x[0]
    if x.dim() != 2 or col_offsets.dim() != 1 or col_offsets.numel() < 2:
        raise RuntimeError("%s: expected x [1,C,L] or [C,L] and col_offsets [B+1], got %s and %s"
                           % (what, tuple(x.shape), tuple(col_offsets.shape)))
    return x, col_offsets.numel() - 1


def bn_cloud_partials_ragged(x, col_offsets, act=ACT_NONE, dy=None, mean=None, invstd=None,
                             gamma=None, beta=None):
    """The per-(cloud, channel) BatchNorm records of a ragged batch (csrc/train.cu): x [1,C,L] (or
    [C,L]) with cloud b's columns col_offsets[b] .. col_offsets[b+1] (checked by the caller). Without
    dy: the forward records [B,C,SONET_BN_REC_FWD]; with dy (and mean, invstd): the backward ones
    [B,C,SONET_BN_REC_BWD] of act."""
    x, B = _bn_ragged_args(x, col_offsets, "bn_cloud_partials_ragged")
    bwd = dy is not None
    if bwd:
        dy = dy.reshape(x.shape)
        for t, n in ((dy, "dy"), (mean, "mean"), (invstd, "invstd")):
            _chk(t, n, torch.float32)
    C, L = x.shape
    dev = x.device
    with torch.cuda.device(dev):
        rec = torch.empty((B, C, _C.CONSTANTS["SONET_BN_REC_BWD" if bwd else "SONET_BN_REC_FWD"]),
                          dtype=torch.float64, device=dev)
        _call("sonet_bn_cloud_partials_ragged_f32", _C.ptr(x), _C.ptr(dy), _C.ptr(mean), _C.ptr(invstd),
              _C.ptr(gamma), _C.ptr(beta), C, L, _C.ptr(col_offsets), B, act_code(act), int(bwd),
              _C.ptr(rec), _stream(x), kernels=3)
    return rec


def bn_ragged_forward(rec, col_offsets, x, gamma, beta, eps, act):
    """The forward records rec [B,C,3] folded with each cloud's own count, then act(BN(x)) over x
    [1,C,L] -> (y [1,C,L], mean [C], var [C] (biased), invstd [C])."""
    x2, B = _bn_ragged_args(x, col_offsets, "bn_ragged_forward")
    _chk(rec, "rec", torch.float64)
    C, L = x2.shape
    dev = x2.device
    with torch.cuda.device(dev):
        y = torch.empty((1, C, L), dtype=torch.float32, device=dev)
        mean, var, invstd = (torch.empty(C, dtype=torch.float32, device=dev) for _ in range(3))
        _call("sonet_bn_ragged_forward_f32", _C.ptr(rec), _C.ptr(col_offsets), B, _C.ptr(x2),
              _C.ptr(gamma), _C.ptr(beta), C, L, float(eps), act_code(act), _C.ptr(y), _C.ptr(mean),
              _C.ptr(var), _C.ptr(invstd), _stream(x2), kernels=2)
    return y, mean, var, invstd


def bn_ragged_backward(rec, col_offsets, dy, x, mean, invstd, gamma, beta, act):
    """The backward records rec [B,C,2] folded in ascending cloud order, then dx over x [1,C,L] ->
    (dx [1,C,L], dgamma [C], dbeta [C])."""
    x2, B = _bn_ragged_args(x, col_offsets, "bn_ragged_backward")
    _chk(rec, "rec", torch.float64)
    _chk(dy, "dy", torch.float32)
    C, L = x2.shape
    dev = x2.device
    with torch.cuda.device(dev):
        dx = torch.empty((1, C, L), dtype=torch.float32, device=dev)
        dgamma = torch.empty(C, dtype=torch.float32, device=dev)
        dbeta = torch.empty(C, dtype=torch.float32, device=dev)
        _call("sonet_bn_ragged_backward_f32", _C.ptr(rec), _C.ptr(col_offsets), B, _C.ptr(dy),
              _C.ptr(x2), _C.ptr(mean), _C.ptr(invstd), _C.ptr(gamma), _C.ptr(beta), C, L,
              act_code(act), _C.ptr(dx), _C.ptr(dgamma), _C.ptr(dbeta), _stream(x2), kernels=2)
    return dx, dgamma, dbeta


def augment_ragged(points, offsets, som, rot1=None, rot2=None, scale=None, shift=None,
                   jitter_pc=(0.0, 1.0), jitter_sn=(0.0, 1.0), jitter_som=(0.0, 1.0), seed=0):
    """augment over whole clouds (csrc/augment.cu): points [T,6] f32 rows xyz | normal, offsets [B+1]
    int64 (checked by the caller), som [B,3,M] f32 or None; rot1/rot2 [B,3,3], scale [B], shift
    [B,3] float64 device tensors or None; the jitter drawn in the kernel from `seed`, cloud b's row
    n as augment's point n of cloud b. -> (points' [T,6], som' or None)."""
    T, B = _ragged_args(points, offsets, "augment_ragged")
    _chk(som, "som", torch.float32, optional=True)
    for t, n in ((rot1, "rot1"), (rot2, "rot2"), (scale, "scale"), (shift, "shift")):
        _chk(t, n, torch.float64, optional=True)
    M = 0 if som is None else som.shape[2]
    if som is not None and (som.dim() != 3 or som.shape[0] != B or som.shape[1] != 3):
        raise RuntimeError("augment_ragged: som must be [%d,3,M] (got %s)" % (B, tuple(som.shape)))
    for t, shp, n in ((rot1, (B, 3, 3), "rot1"), (rot2, (B, 3, 3), "rot2"), (scale, (B,), "scale"),
                      (shift, (B, 3), "shift")):
        if t is not None and tuple(t.shape) != shp:
            raise RuntimeError("augment_ragged: %s must have shape %s, got %s" % (n, shp, tuple(t.shape)))
    with torch.cuda.device(points.device):
        po = torch.empty_like(points)
        mo = torch.empty_like(som) if som is not None else None
        _call("sonet_augment_ragged_f32", _C.ptr(points), T, 6, _C.ptr(offsets), B, _C.ptr(som), M,
              _C.ptr(rot1), _C.ptr(rot2), _C.ptr(scale), _C.ptr(shift), float(jitter_pc[0]),
              float(jitter_pc[1]), float(jitter_sn[0]), float(jitter_sn[1]), float(jitter_som[0]),
              float(jitter_som[1]), int(seed) & (2 ** 64 - 1), _C.ptr(po), _C.ptr(mo), _stream(points))
    return po, mo

RETRIEVAL_MAX_D = 1024
RETRIEVAL_MAX_K = 4096
RETRIEVAL_MAX_L = 4096


def retrieval_rank(feature, label=None, num_labels=None, k=1000, threads=None):
    """Same-label retrieval ranking (shrec16/test.py:64-99) of every item, no sync.

    feature [Q,D] f32; label [Q] int64 on the same device, or None for the row argmax (lowest
    index on ties, the first NaN wins); num_labels L (default D): labels live in [0, L). For each
    query q, the items p with the same label (q included) sorted by the fp32 distance
    ||f_q - f_p||_2 (fp32 differences summed in fp64), ties by ascending p, NaN last, at most k.
    Returns (idx [Q,k] int64, dist [Q,k] f32, count [Q] int32, label [Q] int64) on the features'
    device: slots past count[q] hold -1 / NaN, and count[q] = -1 flags a label outside [0, L).
    CUDA tensors run the sm_90a kernels; CPU tensors run the host entry (bit-identical), over
    `threads` threads (default torch.get_num_threads())."""
    if not isinstance(feature, torch.Tensor) or feature.dtype != torch.float32 or feature.dim() != 2:
        raise RuntimeError("retrieval_rank: feature must be a [Q,D] float32 tensor")
    if not feature.is_contiguous():
        raise RuntimeError("feature must be contiguous")
    Q, D = feature.shape
    L = D if num_labels is None else int(num_labels)
    k = int(k)
    if not 1 <= D <= RETRIEVAL_MAX_D:
        raise RuntimeError("retrieval_rank: D=%d outside [1, %d]" % (D, RETRIEVAL_MAX_D))
    if not 1 <= k <= RETRIEVAL_MAX_K:
        raise RuntimeError("retrieval_rank: k=%d outside [1, %d]" % (k, RETRIEVAL_MAX_K))
    if not 1 <= L <= RETRIEVAL_MAX_L:
        raise RuntimeError("retrieval_rank: num_labels=%d outside [1, %d]" % (L, RETRIEVAL_MAX_L))
    if Q * k >= 1 << 31:
        raise RuntimeError("retrieval_rank: Q*k=%d must be < 2^31" % (Q * k))
    if label is not None:
        if label.dtype != torch.int64 or tuple(label.shape) != (Q,) or label.device != feature.device:
            raise RuntimeError("retrieval_rank: label must be int64 [Q=%d] on %s" % (Q, feature.device))
        if not label.is_contiguous():
            raise RuntimeError("label must be contiguous")
    dev = feature.device
    idx = torch.empty((Q, k), dtype=torch.int64, device=dev)
    dist = torch.empty((Q, k), dtype=torch.float32, device=dev)
    count = torch.empty((Q,), dtype=torch.int32, device=dev)
    label_out = torch.empty((Q,), dtype=torch.int64, device=dev) if label is None else label
    out_ptr = _C.ptr(label_out) if label is None else None
    if not feature.is_cuda:
        nt = torch.get_num_threads() if threads is None else int(threads)
        _C.check(_C.lib().sonet_retrieval_rank_cpu_f32(
            feature.data_ptr(), _C.ptr(label), Q, D, L, k, idx.data_ptr(), dist.data_ptr(),
            count.data_ptr(), out_ptr, nt), "sonet_retrieval_rank_cpu_f32")
        return idx, dist, count, label_out
    with torch.cuda.device(dev):
        nbytes = int(_C.lib().sonet_retrieval_scratch_bytes(Q, D, L, k))
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        _call("sonet_retrieval_rank_f32", _C.ptr(feature), _C.ptr(label), Q, D, L, k, _C.ptr(scratch),
              nbytes, _C.ptr(idx), _C.ptr(dist), _C.ptr(count), out_ptr, _stream(feature), kernels=4)
    return idx, dist, count, label_out


def retrieval_format(ids, idx, dist, count, threads=None):
    """Host bytes of np.savetxt(f, rows, fmt='%06d %f') per query, for the rows
    (ids[idx[q,i]], dist[q,i]), i < count[q], of a retrieval_rank result (CPU tensors).
    Returns (text bytes, offsets [Q+1] int64): query q's file is text[offsets[q]:offsets[q+1]]."""
    Q, k = idx.shape
    for t, name, dt in ((ids, "ids", torch.int64), (idx, "idx", torch.int64),
                        (dist, "dist", torch.float32), (count, "count", torch.int32)):
        if t.is_cuda or t.dtype != dt or not t.is_contiguous():
            raise RuntimeError("retrieval_format: %s must be a contiguous CPU %s tensor" % (name, dt))
    if tuple(ids.shape) != (Q,) or tuple(dist.shape) != (Q, k) or tuple(count.shape) != (Q,):
        raise RuntimeError("retrieval_format: expected ids [Q], idx/dist [Q,k], count [Q]")
    nt = torch.get_num_threads() if threads is None else int(threads)
    lib = _C.lib()
    offsets = torch.empty((Q + 1,), dtype=torch.int64)
    args = (ids.data_ptr(), idx.data_ptr(), dist.data_ptr(), count.data_ptr(), Q, k,
            offsets.data_ptr())
    total = lib.sonet_retrieval_format_cpu(*args, None, nt)
    if total < 0:
        raise RuntimeError("retrieval_format failed: %s" % _C.last_error())
    if total == 0:
        return b"", offsets
    buf = bytearray(total)
    cbuf = (ctypes.c_char * total).from_buffer(buf)
    if lib.sonet_retrieval_format_cpu(*args, ctypes.addressof(cbuf), nt) != total:
        raise RuntimeError("retrieval_format failed: %s" % _C.last_error())
    del cbuf
    return bytes(buf), offsets


def chamfer(pred, gt, want_idx=False):
    """pred [B,3,Mp], gt [B,3,N] -> dict(loss [3], fwd_arr [B], bwd_arr [B], elem_fwd, elem_bwd,
    idx_fwd?, idx_bwd?)."""
    _chk(pred, "predict_pc", torch.float32)
    _chk(gt, "gt_pc", torch.float32)
    B, _, Mp = pred.shape
    N = gt.shape[2]
    dev = pred.device
    with torch.cuda.device(dev):
        idx_f = torch.empty((B, Mp), dtype=torch.int32, device=dev) if want_idx else None
        idx_b = torch.empty((B, N), dtype=torch.int32, device=dev) if want_idx else None
        ef = torch.empty((B, Mp), dtype=torch.float32, device=dev)
        eb = torch.empty((B, N), dtype=torch.float32, device=dev)
        fa = torch.empty((B,), dtype=torch.float32, device=dev)
        ba = torch.empty((B,), dtype=torch.float32, device=dev)
        loss = torch.empty((3,), dtype=torch.float32, device=dev)
        _call("sonet_chamfer_f32", _C.ptr(pred), _C.ptr(gt), B, Mp, N, _C.ptr(idx_f),
              _C.ptr(idx_b), _C.ptr(ef), _C.ptr(eb), _C.ptr(fa), _C.ptr(ba), _C.ptr(loss),
              _stream(pred), kernels=4 if want_idx else 3)
    return dict(loss=loss, fwd_arr=fa, bwd_arr=ba, elem_fwd=ef, elem_bwd=eb, idx_fwd=idx_f,
                idx_bwd=idx_b)


CHAMFER_RAGGED_MAX_POINTS = (1 << 24) - 1   # P_b must be exact as the float divisor of its mean


def chamfer_ragged(pred, points, offsets, want_idx=False):
    """chamfer against whole clouds: pred [B,3,Mp] f32, points [T,>=3] f32 rows (xyz first, unit
    column stride, any row stride: DeviceDataset's [T,6]), offsets [B+1] int64 on pred's device
    (cloud b is rows offsets[b] .. offsets[b+1]). -> chamfer's dict with the gt side ragged:
    elem_bwd [T], idx_bwd [T] (the nearest predicted point of each gt point), idx_fwd [B,Mp]
    cloud-local rows. Cloud b's entries are chamfer's on that cloud alone; loss is the mean over
    clouds of the per-cloud means. Copies the offsets to the host (one synchronisation) and refuses
    bad offsets, an empty cloud (ValueError) and a cloud of 2^24 points or more before any launch."""
    _chk(pred, "predict_pc", torch.float32)
    _chk(offsets, "offsets", torch.int64)
    if not isinstance(points, torch.Tensor) or points.dtype != torch.float32 or not points.is_cuda:
        raise RuntimeError("points must be a float32 CUDA tensor")
    if pred.dim() != 3 or pred.shape[1] != 3 or pred.shape[0] < 1 or pred.shape[2] < 1:
        raise RuntimeError("chamfer_ragged: predict_pc must be [B,3,Mp] with B, Mp >= 1 (got %s)"
                           % (tuple(pred.shape),))
    if points.dim() != 2 or points.shape[1] < 3 or points.stride(1) != 1 \
            or (points.shape[0] > 1 and points.stride(0) < 3):
        raise RuntimeError("chamfer_ragged: points must be [T, >=3] rows with unit column stride "
                           "(got %s, strides %s)" % (tuple(points.shape), points.stride()))
    if points.device != pred.device or offsets.device != pred.device:
        raise RuntimeError("chamfer_ragged: predict_pc, points and offsets must be on one device "
                           "(got %s, %s, %s)" % (pred.device, points.device, offsets.device))
    B, _, Mp = pred.shape
    T = points.shape[0]
    off = ragged_offsets(offsets, T, B)
    counts = off[1:] - off[:-1]
    if (counts == 0).any():
        raise ValueError("chamfer_ragged: cloud %d has no points" % int((counts == 0).argmax()))
    if counts.max() > CHAMFER_RAGGED_MAX_POINTS:
        raise RuntimeError("chamfer_ragged: cloud %d has %d points, more than %d"
                           % (int(counts.argmax()), int(counts.max()), CHAMFER_RAGGED_MAX_POINTS))
    dev = pred.device
    with torch.cuda.device(dev):
        tile_start = torch.empty((B + 1,), dtype=torch.int32, device=dev)
        idx_f = torch.empty((B, Mp), dtype=torch.int32, device=dev) if want_idx else None
        idx_b = torch.empty((T,), dtype=torch.int32, device=dev) if want_idx else None
        ef = torch.empty((B, Mp), dtype=torch.float32, device=dev)
        eb = torch.empty((T,), dtype=torch.float32, device=dev)
        fa = torch.empty((B,), dtype=torch.float32, device=dev)
        ba = torch.empty((B,), dtype=torch.float32, device=dev)
        loss = torch.empty((3,), dtype=torch.float32, device=dev)
        _call("sonet_chamfer_ragged_f32", _C.ptr(pred), B, Mp, _C.ptr(points), T,
              points.stride(0), _C.ptr(offsets), off.ctypes.data, _C.ptr(tile_start), _C.ptr(idx_f),
              _C.ptr(idx_b), _C.ptr(ef), _C.ptr(eb), _C.ptr(fa), _C.ptr(ba), _C.ptr(loss),
              _stream(pred), kernels=4 if want_idx else 3)
    return dict(loss=loss, fwd_arr=fa, bwd_arr=ba, elem_fwd=ef, elem_bwd=eb, idx_fwd=idx_f,
                idx_bwd=idx_b)


def pointresnet_tc_pack(W, shifts, cin):
    """Host-side packing for pointresnet_tc: W = [W0 [64,cin], W1 [128,64], W2 [256,128],
    W3 [384,320]] folded fp32 weights, shifts = 4 folded shift vectors (any device).
    Returns (blob uint8 [bytes], fparams f32) as CPU tensors."""
    lib = _C.lib()
    Wc = [w.detach().to("cpu", torch.float32).contiguous() for w in W]
    Sc = [s.detach().to("cpu", torch.float32).contiguous() for s in shifts]
    want = [(64, cin), (128, 64), (256, 128), (384, 320)]
    for w, sh, s in zip(Wc, want, Sc):
        if tuple(w.shape) != sh or s.numel() != sh[0]:
            raise RuntimeError("pointresnet_tc_pack: unexpected layer shape %s" % (tuple(w.shape),))
    blob = torch.zeros(lib.sonet_pointresnet_tc_blob_bytes(), dtype=torch.uint8)
    fparams = torch.zeros(lib.sonet_pointresnet_tc_fparam_count(), dtype=torch.float32)
    _C.check(lib.sonet_pointresnet_tc_pack(Wc[0].data_ptr(), int(cin), Wc[1].data_ptr(),
                                           Wc[2].data_ptr(), Wc[3].data_ptr(), Sc[0].data_ptr(),
                                           Sc[1].data_ptr(), Sc[2].data_ptr(), Sc[3].data_ptr(),
                                           blob.data_ptr(), fparams.data_ptr()),
             "sonet_pointresnet_tc_pack")
    return blob, fparams


def pointresnet_tc(x, blob, fparams, f16=False, act=ACT_RELU):
    """x [B,Cin<=6,P] f32 -> [B,384,P]: the fused wgmma first PointResNet (f16: one fp16 product
    per MAC instead of the hi/lo split's three; act: the activation of layers 0-2, 'relu' or
    'elu')."""
    act = act_code(act)
    _chk(x, "x", torch.float32)
    _chk(blob, "blob", torch.uint8)
    _chk(fparams, "fparams", torch.float32)
    B, Cin, P = x.shape
    with torch.cuda.device(x.device):
        out = torch.empty((B, 384, P), dtype=torch.float32, device=x.device)
        if act == ACT_RELU:
            _call(_entry("sonet_pointresnet_tc_forward", f16), _C.ptr(x), Cin, B, P, _C.ptr(blob),
                  _C.ptr(fparams), _C.ptr(out), _stream(x))
        else:
            _call("sonet_pointresnet_tc_forward_act", _C.ptr(x), Cin, B, P, _C.ptr(blob),
                  _C.ptr(fparams), act, int(bool(f16)), _C.ptr(out), _stream(x))
    return out


def pointwise_tc_pack(W):
    """W [Cout,Cin] folded fp32 (any device) -> (blob uint8 CPU tensor, inv_scale float)."""
    import ctypes
    lib = _C.lib()
    Wc = W.detach().to("cpu", torch.float32).contiguous()
    Cout, Cin = Wc.shape
    blob = torch.zeros(int(lib.sonet_pointwise_tc_blob_bytes(Cout, Cin)), dtype=torch.uint8)
    inv = ctypes.c_float(0.0)
    _C.check(lib.sonet_pointwise_tc_pack(Wc.data_ptr(), Cout, Cin, blob.data_ptr(),
                                         ctypes.addressof(inv)), "sonet_pointwise_tc_pack")
    return blob, float(inv.value)


def pointwise_tc_pack_groups(Wg):
    """Wg [G,Cout,Cin] folded fp32 (any device) -> (blob uint8 CPU tensor of G consecutive blobs,
    bytes per blob, common inv_scale)."""
    import ctypes
    lib = _C.lib()
    Wc = Wg.detach().to("cpu", torch.float32).contiguous()
    G, Cout, Cin = Wc.shape
    per = int(lib.sonet_pointwise_tc_blob_bytes(Cout, Cin))
    blob = torch.zeros(per * G, dtype=torch.uint8)
    inv = ctypes.c_float(0.0)
    _C.check(lib.sonet_pointwise_tc_pack_groups(Wc.data_ptr(), G, Cout, Cin, blob.data_ptr(),
                                                ctypes.addressof(inv)),
             "sonet_pointwise_tc_pack_groups")
    return blob, per, float(inv.value)


def upconv_im2col(x):
    """x [B,Cin,H,W] -> xcol [4*B, 4*Cin, H*W]: the 2x2 low-resolution neighbourhoods of the four
    output parities of a nearest-x2 + 3x3 up-convolution (csrc/upconv.cu)."""
    _chk(x, "x", torch.float32)
    B, Cin, H, W = x.shape
    with torch.cuda.device(x.device):
        xcol = torch.empty((4 * B, 4 * Cin, H * W), dtype=torch.float32, device=x.device)
        _call("sonet_upconv_im2col_f32", _C.ptr(x), B, Cin, H, W, _C.ptr(xcol), _stream(x))
    return xcol


def upconv_conv_mode(Cin, H, W):
    """The parity GEMMs of an up-convolution read the three horizontal shifts (upconv_hshift)
    instead of the 16x im2col: H*W % 64 == 0 and Cin % 64 == 0, unless SONET_UPCONV_IM2COL=1."""
    return (H * W) % 64 == 0 and Cin % 64 == 0 and os.environ.get("SONET_UPCONV_IM2COL", "0") != "1"


def upconv_hshift(x):
    """x [B,Cin,H,W] -> [3*B, Cin, H*W]: the input shifted horizontally by -1, 0, +1 (zeros at the
    row ends) — the operand of the im2col-free up-convolution (csrc/upconv.cu)."""
    _chk(x, "x", torch.float32)
    B, Cin, H, W = x.shape
    with torch.cuda.device(x.device):
        out = torch.empty((3 * B, Cin, H * W), dtype=torch.float32, device=x.device)
        _call("sonet_upconv_hshift_f32", _C.ptr(x), B, Cin, H, W, _C.ptr(out), _stream(x))
    return out


def pick_splits(kchunks, base_items, target=120, cap=32):
    """K split of a wgmma launch: the smallest power of two dividing the number of 64-channel
    K chunks that brings the item count to ~one wave of SMs."""
    s = 1
    while s * 2 <= cap and kchunks % (s * 2) == 0 and base_items * s < target:
        s *= 2
    return s


def pointwise_tc_grouped(x, blob, per_bytes, inv_scale, shift, cout, act, groups, splits=1,
                         scat_w=0, out=None, scratch=None, conv=False, f16=False):
    """Grouped wgmma layer: x [G*B, C, P], G weight blobs -> out. scat_w = W > 0: the four groups
    are the output parities of an up-convolution over [H, W] maps, interleaved into
    out [B, cout, 4*P]; otherwise out [G*B, cout, P]. splits > 1: K split through `scratch`.
    act: activation (act_code).
    f16: one fp16 product per MAC instead of the hi/lo split's three."""
    _chk(x, "x", torch.float32)
    _chk(blob, "blob", torch.uint8)
    _chk(shift, "shift", torch.float32, optional=True)
    GB, C, P = x.shape
    B = GB // (3 if conv else groups)       # conv mode: x holds the 3 horizontally shifted copies
    dev = x.device
    with torch.cuda.device(dev):
        if scat_w > 0:
            P_out, gstride = 4 * P, 0
            if out is None:
                out = torch.empty((B, cout, P_out), dtype=torch.float32, device=dev)
        else:
            P_out, gstride = P, B * cout * P
            if out is None:
                out = torch.empty((GB, cout, P), dtype=torch.float32, device=dev)
        if splits > 1 and scratch is None:
            scratch = torch.empty((groups * splits * B * cout * P,), dtype=torch.float32, device=dev)
        _call(_entry("sonet_pointwise_tc_grouped_forward", f16), _C.ptr(x), C, B, P, _C.ptr(blob),
              int(per_bytes),
              float(inv_scale), _C.ptr(shift), int(cout), act_code(act), int(groups), int(splits),
              int(scat_w), int(scat_w) if conv else 0, int(P_out), int(gstride), _C.ptr(out),
              _C.ptr(scratch), _stream(x),
              kernels=2 if splits > 1 else 1)
    return out


def pointwise_layer_tc(x0, blob, inv_scale, shift, cout, act, x1=None, addend=None, gidx=None,
                       rows=False, f16=False):
    """wgmma variant of pointwise_layer: x0 [B,C0,P] (+ x1) -> [B,cout,P], or with rows=True the
    same values point-major, [B,P,cout]. act: activation (act_code). f16: one fp16 product per MAC
    instead of the hi/lo split's three."""
    _chk(x0, "x0", torch.float32)
    _chk(x1, "x1", torch.float32, optional=True)
    _chk(blob, "blob", torch.uint8)
    _chk(shift, "shift", torch.float32, optional=True)
    _chk(addend, "addend", torch.float32, optional=True)
    _chk(gidx, "gidx", torch.int32, optional=True)
    B, C0, P = x0.shape
    C1 = 0 if x1 is None else x1.shape[1]
    G = 0 if addend is None else addend.shape[2]
    with torch.cuda.device(x0.device):
        if rows:
            out = torch.empty((B, P, cout), dtype=torch.float32, device=x0.device)
            _call(_entry("sonet_pointwise_tc_forward_rows", f16), _C.ptr(x0), C0, _C.ptr(x1), C1, B, P,
                  _C.ptr(blob), float(inv_scale), _C.ptr(shift), int(cout), act_code(act),
                  _C.ptr(addend), _C.ptr(gidx), G, _C.ptr(out), _stream(x0))
        else:
            out = torch.empty((B, cout, P), dtype=torch.float32, device=x0.device)
            _call(_entry("sonet_pointwise_tc_forward", f16), _C.ptr(x0), C0, _C.ptr(x1), C1, B, P,
                  _C.ptr(blob),
                  float(inv_scale), _C.ptr(shift), int(cout), act_code(act), _C.ptr(addend),
                  _C.ptr(gidx), G, _C.ptr(out), _stream(x0))
    return out


# Row count up to which a two-layer PointNet takes nodegemm_pointnet. Below it the generic layer's
# per-chunk activation conversion dominates its items; the segmenter's 49 k-row layers amortise it.
NODEGEMM_MAX_ROWS = 16384


class NodeImages:
    """Per-owner (one per PointNet), per-(device, size, stream) buffers of nodegemm_pointnet's fp16
    operand images. They are static, so no forward allocates them and a captured CUDA graph
    replays on the buffers it was captured with."""

    def __init__(self):
        self._bufs = {}

    def get(self, dev, which, nbytes, stream):
        kk = (dev, which, int(nbytes), int(stream))
        buf = self._bufs.get(kk)
        if buf is None:
            buf = self._bufs[kk] = torch.empty(int(nbytes), dtype=torch.uint8, device=dev)
        return buf


_DEFAULT_NODE_IMAGES = NodeImages()   # for direct ops.nodegemm_pointnet callers (tests, tools)


def nodegemm_pointnet(x0, x1, params1, cout1, act, params2, cout2, f16=False, owner=None):
    """act(layer 1) then the bare layer 2 over cat(x0 [B,C0,P], x1 [B,C1,P] or None) -> [B,cout2,P]
    on the node-level wgmma GEMM (csrc/nodegemm_tc.cu), bit-identical to two pointwise_layer_tc
    calls. params1 / params2: (blob, inv_scale, shift) of the layers, as pointwise_tc_pack makes
    them. The input is split into fp16 operand images once; layer 1 writes its output as layer 2's
    images. f16: one fp16 product per MAC instead of the hi/lo split's three."""
    _chk(x0, "x0", torch.float32)
    _chk(x1, "x1", torch.float32, optional=True)
    for blob, _, shift in (params1, params2):
        _chk(blob, "blob", torch.uint8)
        _chk(shift, "shift", torch.float32, optional=True)
    B, C0, P = x0.shape
    C1 = 0 if x1 is None else x1.shape[1]
    dev, f16, stream = x0.device, int(bool(f16)), _stream(x0)
    lib = _C.lib()
    with torch.cuda.device(dev):
        imgs = owner or _DEFAULT_NODE_IMAGES
        img0 = imgs.get(dev, 0, lib.sonet_nodegemm_image_bytes(B * P, C0 + C1, f16), stream)
        img1 = imgs.get(dev, 1, lib.sonet_nodegemm_image_bytes(B * P, int(cout1), f16), stream)
        out = torch.empty((B, cout2, P), dtype=torch.float32, device=dev)
        _call("sonet_nodegemm_split_pack", _C.ptr(x0), C0, _C.ptr(x1), C1, B, P, f16, _C.ptr(img0),
              stream)
        _call("sonet_nodegemm_tc_forward", _C.ptr(img0), C0 + C1, B, P, _C.ptr(params1[0]),
              float(params1[1]), _C.ptr(params1[2]), int(cout1), act_code(act), f16, _C.ptr(img1),
              None, stream)
        _call("sonet_nodegemm_tc_forward", _C.ptr(img1), int(cout1), B, P, _C.ptr(params2[0]),
              float(params2[1]), _C.ptr(params2[2]), int(cout2), ACT_NONE, f16, None, _C.ptr(out),
              stream)
    return out


def knn_mlp_tc_pack(W2):
    """W2 [512,512] folded fp32 (any device) -> (blob uint8 CPU tensor, inv_scale float): the
    layer-2 weight stream of knn_mlp_tc."""
    import ctypes
    lib = _C.lib()
    Wc = W2.detach().to("cpu", torch.float32).contiguous()
    if tuple(Wc.shape) != (512, 512):
        raise RuntimeError("knn_mlp_tc_pack: expected W2 [512,512], got %s" % (tuple(Wc.shape),))
    blob = torch.zeros(int(lib.sonet_knn_mlp_tc_blob_bytes()), dtype=torch.uint8)
    inv = ctypes.c_float(0.0)
    _C.check(lib.sonet_knn_mlp_tc_pack(Wc.data_ptr(), blob.data_ptr(), ctypes.addressof(inv)),
             "sonet_knn_mlp_tc_pack")
    return blob, float(inv.value)


def knn_mlp_tc(coord, center, idx, K, Y, w1, blob, inv_scale, shift2, f16=False, act=ACT_RELU):
    """The KNN module's layer 1 (from the per-node Y = W1f x [B,512,M]) + layer 2 + max over the
    K neighbours in one wgmma kernel. coord, center [B,3,M]; idx [B,M,K'] i64; w1 [512,4] =
    (W1d | shift1); shift2 [512] -> knn_feature_1 [B,512,M]. Y is [B,512,M] either contiguous or
    the channel-fastest view y.transpose(1, 2) of a contiguous [B,M,512] (pointwise_layer_tc(...,
    rows=True)); the kernel reads the latter as float2 pairs, with bit-identical results.
    f16: layer 2 as one fp16 product per MAC instead of the hi/lo split's three. act: the
    activation of both layers, 'relu' or 'elu'."""
    act = act_code(act)
    _chk(coord, "coordinate", torch.float32)
    _chk(center, "center", torch.float32)
    _chk(idx, "knn_I", torch.int64)
    if Y.dim() == 3 and not Y.is_contiguous() and Y.transpose(1, 2).is_contiguous():
        _chk(Y.transpose(1, 2), "Y", torch.float32)
    else:
        _chk(Y, "Y", torch.float32)
    _chk(w1, "w1", torch.float32)
    _chk(blob, "blob", torch.uint8)
    _chk(shift2, "shift2", torch.float32)
    B, _, M = coord.shape
    if tuple(Y.shape) != (B, 512, M) or tuple(w1.shape) != (512, 4) or shift2.numel() != 512 \
            or tuple(idx.shape[:2]) != (B, M):
        raise RuntimeError("knn_mlp_tc: unexpected shapes coord %s Y %s w1 %s idx %s"
                           % (tuple(coord.shape), tuple(Y.shape), tuple(w1.shape), tuple(idx.shape)))
    with torch.cuda.device(coord.device):
        out = torch.empty((B, 512, M), dtype=torch.float32, device=coord.device)
        if act == ACT_RELU:
            _call(_entry("sonet_knn_mlp_tc_forward", f16), _C.ptr(coord), _C.ptr(center), _C.ptr(idx),
                  B, M, int(K), idx.shape[2], _C.ptr(Y), Y.stride(1), Y.stride(2), _C.ptr(w1),
                  _C.ptr(blob), float(inv_scale), _C.ptr(shift2), _C.ptr(out), _stream(coord))
        else:
            _call("sonet_knn_mlp_tc_forward_act", _C.ptr(coord), _C.ptr(center), _C.ptr(idx), B, M,
                  int(K), idx.shape[2], _C.ptr(Y), Y.stride(1), Y.stride(2), _C.ptr(w1), _C.ptr(blob),
                  float(inv_scale), _C.ptr(shift2), act, int(bool(f16)), _C.ptr(out), _stream(coord))
    return out


def som_sort_decenter(x, sn, cluster_mean, min_idx_i32, count, k):
    """-> (x_sorted [B,3(+3),kN], node_sorted [B,kN] i32, pos0 [B] i32): the stacked copies grouped
    by node, decentred (models/networks.py:168-172) — input of pointresnet_tc_pool."""
    _chk(x, "x", torch.float32)
    _chk(sn, "sn", torch.float32, optional=True)
    _chk(cluster_mean, "cluster_mean", torch.float32)
    _chk(min_idx_i32, "min_idx", torch.int32)
    _chk(count, "count", torch.int32)
    B, _, N = x.shape
    M = cluster_mean.shape[2]
    kN = k * N
    dev = x.device
    with torch.cuda.device(dev):
        xs = torch.empty((B, 6 if sn is not None else 3, kN), dtype=torch.float32, device=dev)
        ns = torch.empty((B, kN), dtype=torch.int32, device=dev)
        p0 = torch.empty((B,), dtype=torch.int32, device=dev)
        _call("sonet_som_sort_decenter", _C.ptr(x), _C.ptr(sn), _C.ptr(cluster_mean),
              _C.ptr(min_idx_i32), _C.ptr(count), B, N, M, int(k), _C.ptr(xs), _C.ptr(ns),
              _C.ptr(p0), _stream(x))
    return xs, ns, p0


_MAX_SMEM = {}
# sonet_som_group_mode results (include/sonet_b200.h)
SOM_GROUP_NONE = _C.CONSTANTS["SONET_SOM_GROUP_NONE"]
SOM_GROUP_UNSTAGED = _C.CONSTANTS["SONET_SOM_GROUP_UNSTAGED"]
SOM_GROUP_STAGED = _C.CONSTANTS["SONET_SOM_GROUP_STAGED"]


def som_group_mode(N, M, k, with_sn, dev):
    """How sonet_som_group_decenter runs on this device: SOM_GROUP_STAGED (cloud staged in shared
    memory), SOM_GROUP_UNSTAGED (read from global memory) or SOM_GROUP_NONE (does not fit)."""
    cap = _MAX_SMEM.get(dev)
    if cap is None:
        cap = _MAX_SMEM[dev] = torch.cuda.get_device_properties(dev).shared_memory_per_block_optin
    mode = _C.lib().sonet_som_group_mode(int(N), int(M), int(k), int(bool(with_sn)), int(cap))
    if mode < 0:
        _C.check(mode, "sonet_som_group_mode")
    return mode


def som_group_fits(N, M, k, dev):
    """Does sonet_som_group_decenter's per-cloud shared-memory footprint fit on this device?"""
    return som_group_mode(N, M, k, False, dev) != SOM_GROUP_NONE


def som_group_decenter(x, sn, min_idx_i32, M, k):
    """Cluster statistics + stable node sort + decentring in one launch (classifier path).
    -> (x_sorted [B,3(+3),kN], node_sorted [B,kN] i32, pos0 [B] i32, count [B,M] i32,
    cluster_mean [B,3,M])."""
    _chk(x, "x", torch.float32)
    _chk(sn, "sn", torch.float32, optional=True)
    _chk(min_idx_i32, "min_idx", torch.int32)
    B, _, N = x.shape
    kN = k * N
    dev = x.device
    with torch.cuda.device(dev):
        xs = torch.empty((B, 6 if sn is not None else 3, kN), dtype=torch.float32, device=dev)
        ns = torch.empty((B, kN), dtype=torch.int32, device=dev)
        p0 = torch.empty((B,), dtype=torch.int32, device=dev)
        count = torch.empty((B, M), dtype=torch.int32, device=dev)
        cmean = torch.empty((B, 3, M), dtype=torch.float32, device=dev)
        _call("sonet_som_group_decenter", _C.ptr(x), _C.ptr(sn), _C.ptr(min_idx_i32), B, N, int(M),
              int(k), _C.ptr(count), _C.ptr(cmean), _C.ptr(xs), _C.ptr(ns), _C.ptr(p0), _stream(x))
    return xs, ns, p0, count, cmean


class PoolKeys:
    """Per-owner (one per Encoder), per-(device, B, M, stream) key buffers of the fused per-node
    max. The kernels keep the invariant "keys are all-minimum between forwards" themselves
    (pool_finalize / knn_assemble_pool reset every key they read); `dirty` covers the failure
    window between the pool launch and its finalisation: if anything raises in between, the next
    acquire() re-initialises the buffer instead of silently maxing against a stale batch."""

    def __init__(self):
        self._bufs = {}

    def acquire(self, dev, B, M, stream):
        kk = (dev, int(B), int(M), int(stream))
        ent = self._bufs.get(kk)
        if ent is None:
            ent = self._bufs[kk] = dict(
                keys=torch.empty((B, 384, M), dtype=torch.int32, device=dev), dirty=True)
        if ent["dirty"]:
            _call("sonet_pool_keys_init", _C.ptr(ent["keys"]), ent["keys"].numel(), stream)
        ent["dirty"] = True          # until release()
        self._last = ent
        return ent["keys"]

    def release(self, keys):
        for ent in self._bufs.values():
            if ent["keys"] is keys:
                ent["dirty"] = False


_DEFAULT_POOL_KEYS = PoolKeys()   # for direct ops.pointresnet_tc_pool callers (tests, tools)


def pool_finalize(keys, p0, owner=None):
    """Pool keys [B,C,M] i32 + copy-0 features [B,C] -> first_pn_out_masked_max [B,C,M]; resets
    the keys."""
    B, C, M = keys.shape
    with torch.cuda.device(keys.device):
        out = torch.empty((B, C, M), dtype=torch.float32, device=keys.device)
        _call("sonet_pool_finalize", _C.ptr(keys), _C.ptr(p0), B, C, M, _C.ptr(out), _stream(keys))
    (owner or _DEFAULT_POOL_KEYS).release(keys)
    return out


def knn_assemble_pool(coord, keys, p0, idx, K, center_type, owner=None, want_x_aug=True):
    """knn_assemble reading the per-node maxima from the pool keys (pool_finalize folded in).
    -> (center [B,3,M], x_aug [B,3+C,M*K] or None with want_x_aug=False, masked_max [B,C,M])."""
    _chk(coord, "coordinate", torch.float32)
    _chk(keys, "pool_keys", torch.int32)
    _chk(p0, "p0", torch.float32)
    _chk(idx, "knn_I", torch.int64)
    B, C, M = keys.shape
    Kstride = idx.shape[2]
    ct = {"avg": 0, "center": 1}[center_type]
    dev = keys.device
    with torch.cuda.device(dev):
        center = torch.empty((B, 3, M), dtype=torch.float32, device=dev)
        x_aug = torch.empty((B, 3 + C, M * K), dtype=torch.float32, device=dev) \
            if want_x_aug else None
        mm = torch.empty((B, C, M), dtype=torch.float32, device=dev)
        _call("sonet_knn_assemble_pool_f32", _C.ptr(coord), _C.ptr(keys), _C.ptr(p0), _C.ptr(idx), B,
              C, M, int(K), Kstride, ct, _C.ptr(mm), _C.ptr(center), _C.ptr(x_aug), _stream(keys))
    (owner or _DEFAULT_POOL_KEYS).release(keys)
    return center, x_aug, mm


def pointresnet_tc_pool(x_sorted, blob, fparams, node_sorted, pos0, M, finalize=True, owner=None,
                        f16=False, act=ACT_RELU):
    """Fused wgmma PointResNet + per-node max: -> first_pn_out_masked_max [B,384,M], or with
    finalize=False the raw (keys [B,384,M] i32, p0 [B,384]) for knn_assemble_pool / pool_finalize.
    f16: one fp16 product per MAC instead of the hi/lo split's three. act: the activation of
    layers 0-2, 'relu' or 'elu'."""
    act = act_code(act)
    _chk(x_sorted, "x_sorted", torch.float32)
    _chk(blob, "blob", torch.uint8)
    _chk(fparams, "fparams", torch.float32)
    _chk(node_sorted, "node_sorted", torch.int32)
    _chk(pos0, "pos0", torch.int32)
    B, Cin, P = x_sorted.shape
    dev = x_sorted.device
    with torch.cuda.device(dev):
        keys = (owner or _DEFAULT_POOL_KEYS).acquire(dev, B, M, _stream(x_sorted))
        p0 = torch.empty((B, 384), dtype=torch.float32, device=dev)
        if act == ACT_RELU:
            _call(_entry("sonet_pointresnet_tc_pool_forward", f16), _C.ptr(x_sorted), Cin, B, P,
                  _C.ptr(blob),
                  _C.ptr(fparams), _C.ptr(node_sorted), _C.ptr(pos0), int(M), _C.ptr(keys),
                  _C.ptr(p0), _stream(x_sorted))
        else:
            _call("sonet_pointresnet_tc_pool_forward_act", _C.ptr(x_sorted), Cin, B, P, _C.ptr(blob),
                  _C.ptr(fparams), _C.ptr(node_sorted), _C.ptr(pos0), int(M), act, int(bool(f16)),
                  _C.ptr(keys), _C.ptr(p0), _stream(x_sorted))
    if not finalize:
        return keys, p0
    return pool_finalize(keys, p0, owner)


def som_query_topk(x, node, k):
    """BatchSOM.query_topk in one launch -> (mask [B,kN,M] i32, row_max [B,M] i32,
    min_idx [B,kN] i64, min_idx_i32 [B,kN])."""
    _chk(x, "x", torch.float32)
    _chk(node, "node", torch.float32)
    B, _, N = x.shape
    M = node.shape[2]
    dev = x.device
    with torch.cuda.device(dev):
        mask = torch.empty((B, k * N, M), dtype=torch.int32, device=dev)
        row_max = torch.empty((B, M), dtype=torch.int32, device=dev)
        idx64 = torch.empty((B, k * N), dtype=torch.int64, device=dev)
        idx32 = torch.empty((B, k * N), dtype=torch.int32, device=dev)
        _call("sonet_som_query_topk", _C.ptr(x), _C.ptr(node), B, N, M, int(k), _C.ptr(mask),
              _C.ptr(row_max), _C.ptr(idx64), _C.ptr(idx32), _stream(x))
    return mask, row_max, idx64, idx32
