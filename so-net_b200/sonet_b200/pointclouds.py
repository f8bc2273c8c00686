"""Datasets from bare point clouds: surface normals estimated on the device, then each shape's SOM.

The point-cloud counterpart of meshes.py, for clouds that come with no mesh and no normals (a scan,
a cloud sampled by another tool, any [P, 3] array). Every SO-Net model reads a normal per point.

1. k-NN (knn): the exact k nearest points of every point within its own cloud, brute force over a
   ragged batch in one launch (csrc/point_normals.cu).
2. Normals (estimate_normals): the unit normal of the plane fitted to each point's k neighbours, the
   eigenvector of the smallest eigenvalue of their covariance, in fp64. A PCA normal has no sign of
   its own: `orient` picks the rule (canonical, away from the cloud's centroid, or toward a
   viewpoint per cloud). Centroid orientation is only right for roughly star-shaped objects.
3. Orientation (orient_normals, or estimate_normals(orient="propagate")): signs propagated along
   the minimum spanning tree of each cloud's k-NN graph (Hoppe et al. 1992), anchored once per
   connected component, so that concave shapes (cups, chairs, the inner ring of a torus) get
   consistent normals. Borůvka rounds on the device (csrc/point_normals.cu).
4. SOM nodes: the notebook's procedure (data/build_som/save_som.ipynb), n of each cloud's points
   chosen without replacement, then BatchSOM(rows, cols).optimize, on ragged clouds.

build_dataset chains them into an augmentation.DeviceDataset; save_npz writes the notebook's
model_<name>.npz files (pc, sn, som_node).
"""
import os

import numpy as np
import torch

from . import ops
from .augmentation import DeviceDataset
from .som import BatchSOM

_ORIENT = {None: ops.NORMALS_CANONICAL, "centroid": ops.NORMALS_AWAY_FROM_CENTROID,
           "viewpoint": ops.NORMALS_TOWARD_VIEWPOINT}
# estimate_normals' tree rules: the canonical estimate, then orient_normals with this anchor
_PROPAGATE = {"propagate": ops.NORMALS_AWAY_FROM_CENTROID,
              "propagate-viewpoint": ops.NORMALS_TOWARD_VIEWPOINT}
_ANCHOR = {"centroid": ops.NORMALS_AWAY_FROM_CENTROID, "viewpoint": ops.NORMALS_TOWARD_VIEWPOINT}


def _check_k(k, what):
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 3 <= k <= ops.POINT_KNN_MAX_K:
        raise ValueError("%s: k=%r must be an integer in [3, %d]" % (what, k, ops.POINT_KNN_MAX_K))
    return int(k)


def _check_input(data, offsets, what, min_points=3, need="a normal needs at least 3"):
    """The host copy of offsets, after checking data [T, >=3] f32 and offsets [S+1] i64 on one
    CUDA device, the offsets within [0, T] and every cloud at least min_points long."""
    if not (torch.is_tensor(data) and torch.is_tensor(offsets) and data.is_cuda and offsets.is_cuda):
        raise ValueError("%s: data and offsets must be CUDA tensors" % what)
    if data.dtype != torch.float32 or data.dim() != 2 or data.shape[1] < 3:
        raise ValueError("%s: data must be f32 [T, >=3], got %s %s" % (what, data.dtype,
                                                                      tuple(data.shape)))
    if offsets.dtype != torch.int64 or offsets.dim() != 1 or offsets.shape[0] < 2:
        raise ValueError("%s: offsets must be i64 [S+1] with S >= 1" % what)
    off = offsets.cpu().numpy()
    if off[0] < 0 or off[-1] > data.shape[0]:
        raise ValueError("%s: offsets must lie in [0, %d]" % (what, data.shape[0]))
    counts = np.diff(off)
    if (counts < min_points).any():
        s = int(np.flatnonzero(counts < min_points)[0])
        raise ValueError("%s: cloud %d has %d points; %s" % (what, s, int(counts[s]), need))
    return off


def _viewpoint(viewpoint, S, device, what, orient):
    """viewpoint as a [S, 3] f32 device tensor; ValueError when it is missing or misshapen."""
    if viewpoint is None:
        raise ValueError("%s: %s needs viewpoint [S, 3]" % (what, orient))
    view = viewpoint if torch.is_tensor(viewpoint) else np.asarray(viewpoint, np.float32)
    view = torch.as_tensor(view).to(device, torch.float32).contiguous()
    if tuple(view.shape) != (S, 3):
        raise ValueError("%s: viewpoint must be [%d, 3], got %s" % (what, S, tuple(view.shape)))
    return view


def _max_points(off, what):
    """The largest cloud of the host offsets, which the orientation's round schedule needs."""
    P = int(np.diff(off).max())
    if P >= ops.POINT_ORIENT_MAX_POINTS:
        raise ValueError("%s: a cloud of %d points; orientation supports at most %d"
                         % (what, P, ops.POINT_ORIENT_MAX_POINTS - 1))
    return P


def knn(data, offsets, k):
    """[T, k] i32: the cloud-local indices of the k nearest points of every point of its own cloud
    (the point itself included), ascending distance, lowest index on ties. data [T, >=3] f32 (xyz in
    columns 0..2) and offsets [S+1] i64 on the device."""
    k = _check_k(k, "knn")
    _check_input(data, offsets, "knn")
    return ops.point_knn(data.contiguous(), offsets.contiguous(), k)[0]


def estimate_normals(data, offsets, k=16, orient="centroid", viewpoint=None, out=None,
                     want_curvature=False):
    """Unit surface normals [T, 3] f32 of every point of the ragged clouds data [T, >=3] f32 /
    offsets [S+1] i64 (CUDA tensors), from its k nearest neighbours within its cloud.
    orient: None (canonical: the component of largest magnitude is positive), "centroid" (pointing
    away from the cloud's mean), "viewpoint" (toward viewpoint [S, 3], one point per cloud, such as
    the sensor's position), or a sign propagated along the minimum spanning tree of the k-NN graph
    (orient_normals on the canonical estimate, reusing its k-NN): "propagate" anchors each
    component at its point farthest from the cloud's mean, "propagate-viewpoint" at its point
    nearest viewpoint. out: a [T, 3] f32 view to write into, such as data[:, 3:6]. With
    want_curvature returns (normals, curvature [T]), the surface variation l0 / (l0 + l1 + l2). A
    degenerate neighbourhood (coincident or collinear points, non-finite coordinates) gives the zero
    vector and NaN curvature. Raises ValueError for k outside [3, 32], an unknown orient, a missing
    viewpoint, or a cloud with fewer than 3 points."""
    k = _check_k(k, "estimate_normals")
    if not isinstance(orient, (str, type(None))) or (orient not in _ORIENT and orient not in _PROPAGATE):
        raise ValueError("estimate_normals: orient=%r is not None, 'centroid', 'viewpoint', "
                         "'propagate' or 'propagate-viewpoint'" % (orient,))
    off = _check_input(data, offsets, "estimate_normals")
    view = None
    if orient in ("viewpoint", "propagate-viewpoint"):
        view = _viewpoint(viewpoint, len(off) - 1, data.device, "estimate_normals", "orient=%r" % orient)
    data, offsets = data.contiguous(), offsets.contiguous()
    idx, _ = ops.point_knn(data, offsets, k)
    code = ops.NORMALS_CANONICAL if orient in _PROPAGATE else _ORIENT[orient]
    normals, curv = ops.estimate_normals(data, offsets, idx, code, view=view, out=out,
                                         want_curvature=want_curvature)
    if orient in _PROPAGATE:
        ops.orient_normals(data, offsets, idx, normals, _PROPAGATE[orient], view=view,
                           max_points=_max_points(off, "estimate_normals"))
    return (normals, curv) if want_curvature else normals


def orient_normals(data, offsets, normals, k=16, anchor="centroid", viewpoint=None, idx=None,
                   return_components=False):
    """Orient the normals [T, 3] f32 (a CUDA view such as data[:, 3:6]; from a scanner, another
    tool or estimate_normals) of the ragged clouds data [T, >=3] f32 / offsets [S+1] i64 in place,
    consistently within each cloud: signs propagate along the minimum spanning tree of the k-NN
    graph (weights 1 - |n_u . n_v|, Hoppe et al. 1992), and each connected component takes its
    sign from one anchor point: anchor="centroid", its point farthest from the cloud's mean, made
    to point away from it; anchor="viewpoint", its point nearest viewpoint [S, 3], made to point
    toward it. idx: a [T, K] i32 cloud-local k-NN (knn's) to reuse, else knn(data, offsets, k).
    Points with a non-finite coordinate or a zero or non-finite normal are left as they are.
    A k-NN graph that bridges two close sheets (a thin wall) can carry a flip across them.
    -> normals, or (normals, components [T] i32) with return_components: the cloud-local index
    of each point's anchor, -1 for the points left out."""
    if not isinstance(anchor, str) or anchor not in _ANCHOR:
        raise ValueError("orient_normals: anchor=%r is not 'centroid' or 'viewpoint'" % (anchor,))
    if idx is None:
        k = _check_k(k, "orient_normals")
    off = _check_input(data, offsets, "orient_normals", 1, "orienting needs at least 1")
    S = len(off) - 1
    view = None
    if anchor == "viewpoint":
        view = _viewpoint(viewpoint, S, data.device, "orient_normals", "anchor='viewpoint'")
    data, offsets = data.contiguous(), offsets.contiguous()
    if idx is None:
        idx, _ = ops.point_knn(data, offsets, k)
    elif not (torch.is_tensor(idx) and idx.is_cuda and idx.dtype == torch.int32 and idx.dim() == 2
              and idx.shape[0] == data.shape[0] and 1 <= idx.shape[1] <= ops.POINT_KNN_MAX_K):
        raise ValueError("orient_normals: idx must be a CUDA i32 [%d, K] tensor with K in [1, %d]"
                         % (data.shape[0], ops.POINT_KNN_MAX_K))
    normals, comp = ops.orient_normals(data, offsets, idx.contiguous(), normals, _ANCHOR[anchor],
                                       view=view, max_points=_max_points(off, "orient_normals"),
                                       want_component=return_components)
    return (normals, comp) if return_components else normals


def _to_device_rows(clouds, device):
    """(data [T, 6] f32 with xyz in columns 0..2 and zeros after, offsets [S+1] i64) on `device`."""
    if isinstance(clouds, tuple) and len(clouds) == 2 and np.ndim(clouds[1]) == 1:
        data, offsets = clouds
        data = torch.as_tensor(data).to(device, torch.float32)
        offsets = torch.as_tensor(offsets).to(device, torch.int64).contiguous()
        if data.dim() != 2 or data.shape[1] < 3:
            raise ValueError("build_dataset: data must be [T, >=3], got %s" % (tuple(data.shape),))
        rows = torch.zeros((data.shape[0], 6), dtype=torch.float32, device=device)
        rows[:, :3] = data[:, :3]
        return rows, offsets
    parts = []
    for i, c in enumerate(clouds):
        c = torch.as_tensor(c).to(device, torch.float32)
        if c.dim() != 2 or c.shape[1] != 3:
            raise ValueError("build_dataset: cloud %d has shape %s, expected [P, 3]"
                             % (i, tuple(c.shape)))
        parts.append(c)
    if not parts:
        raise ValueError("build_dataset: no clouds")
    counts = np.array([len(c) for c in parts], dtype=np.int64)
    rows = torch.zeros((int(counts.sum()), 6), dtype=torch.float32, device=device)
    rows[:, :3] = torch.cat(parts)
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)])).to(device)
    return rows, offsets


def som_nodes(data, offsets, rows=8, cols=8, n=4096, seed=0, rng=None):
    """The notebook's per-shape SOM for ragged clouds: data [T, 6] f32 and offsets [S+1] i64 on the
    device; n of each cloud's points are chosen without replacement (in the kernel, keyed by `seed`
    and the cloud's position, or with a numpy `rng` by rng.choice(P_i, n, replace=False) per cloud
    as the notebook does), then BatchSOM(rows, cols).optimize. -> [S, 3, rows*cols] f32. On clouds
    of one size it gives meshes.som_nodes's nodes."""
    counts = np.diff(offsets.cpu().numpy())
    S = len(counts)
    for s, P in enumerate(counts):
        if n > P:
            raise ValueError("som_nodes: cloud %d: cannot take a larger sample (%d) than population "
                             "(%d) when 'replace=False'" % (s, n, int(P)))
    dev = data.device
    max_P = int(counts.max())
    indices = None
    if rng is not None:
        sel = np.stack([rng.choice(int(P), n, replace=False) for P in counts]).astype(np.int32)
        indices = torch.from_numpy(sel).to(dev)
    elif max_P > ops.SAMPLE_MAX_P:
        raise ValueError("som_nodes: in-kernel choice supports P <= %d (got %d); pass rng"
                         % (ops.SAMPLE_MAX_P, max_P))
    ids = torch.arange(S, dtype=torch.int64, device=dev)
    pc, _, _ = ops.sample_points(data, offsets, ids, n, ops.SAMPLE_SUBSET, max_P, indices=indices,
                                 seed=seed)
    som = BatchSOM(rows, cols, 3, dev.index if dev.index is not None else 0, S)
    som.optimize(pc)
    return som.node.contiguous()


def build_dataset(clouds, labels, k=16, orient="centroid", viewpoint=None, rows=8, cols=None, n=4096,
                  seed=0, rng=None):
    """Bare point clouds -> an augmentation.DeviceDataset whose rows are xyz | estimated normal
    (estimate_normals with k and orient) and whose SOM nodes are som_nodes's (rows x cols, from n
    points of each cloud). clouds: a list of [P_i, 3] arrays or tensors (ragged sizes welcome) or
    a (data [T, >=3], offsets [S+1]) pair; labels: [S] class ids."""
    device = torch.device("cuda")
    first = clouds[0] if len(clouds) else None
    if torch.is_tensor(first) and first.is_cuda:
        device = first.device
    data, offsets = _to_device_rows(clouds, device)
    S = offsets.shape[0] - 1
    if len(labels) != S:
        raise ValueError("build_dataset: %d labels for %d clouds" % (len(labels), S))
    estimate_normals(data, offsets, k=k, orient=orient, viewpoint=viewpoint, out=data[:, 3:6])
    nodes = som_nodes(data, offsets, rows, rows if cols is None else cols, n, seed=seed, rng=rng)
    lab = torch.as_tensor(np.asarray(labels, dtype=np.int64))
    return DeviceDataset.from_device(data, offsets, lab, nodes)


def save_npz(folder, names, dataset_or_arrays):
    """The notebook's files for ragged clouds: folder/model_<name>.npz with pc [P_i, 3], sn [P_i, 3]
    and som_node [M, 3] (the keys data/modelnet_shrec_loader.py reads) per shape. dataset_or_arrays:
    a DeviceDataset (build_dataset's) or a pair (points, som_nodes) of lists of [P_i, 6] and [M, 3]
    arrays or tensors. -> the paths written."""
    host = lambda a: a.detach().cpu().numpy() if torch.is_tensor(a) else np.asarray(a)  # noqa: E731
    if isinstance(dataset_or_arrays, DeviceDataset):
        ds = dataset_or_arrays
        data, off = host(ds.data), host(ds.offsets)
        points = [data[off[s]:off[s + 1]] for s in range(len(ds))]
        nodes = list(host(ds.som_nodes).transpose(0, 2, 1))
    else:
        points, nodes = dataset_or_arrays
        points, nodes = [host(p) for p in points], [host(s) for s in nodes]
    if len(names) != len(points) or len(nodes) != len(points) or \
            any(p.ndim != 2 or p.shape[1] != 6 for p in points) or \
            any(s.ndim != 2 or s.shape[1] != 3 for s in nodes):
        raise ValueError("save_npz: expected names [S], points [P_i, 6] and som_nodes [M, 3] per shape")
    os.makedirs(folder, exist_ok=True)
    paths = []
    for name, p, s in zip(names, points, nodes):
        path = os.path.join(folder, "model_%s.npz" % name)
        np.savez(path, pc=p[:, 0:3], sn=p[:, 3:6], som_node=s)
        paths.append(path)
    return paths
