"""Batched, on-device counterpart of the loader-side preprocessing that feeds the hot path
(SURVEY.md §8f-3): data/augmentation.py:52-144 as applied by
data/modelnet_shrec_loader.py:218-261 — rotation about the up axis, perturbation rotation, jitter
of points / normals / SOM nodes, random scale, random shift — and the SOM-node kNN that the loader
computes per item with a CPU Faiss index (loader :116-150, 256-259).

The reference does this per item in DataLoader workers (six numpy passes + a Faiss index build per
cloud); `prepare_batch` does it for the whole batch in two kernel launches on the device that
already holds the batch: csrc/augment.cu and sonet_node_knn (csrc/pointwise.cu).

Randomness. The per-cloud scalars (angles, scale, shift: 8 numbers per cloud) are drawn on the host
from a numpy RandomState with the loader's own expressions, in the loader's order. The per-point
jitter draws are generated inside the kernel (Philox4x32-10, keyed by seed/cloud/array/point) —
or, with `host_noise=True`, drawn from the same RandomState in the loader's order and shipped to
the device, which reproduces the reference pipeline bit for bit (what the parity tests use).

`DeviceDataset` adds the head of the loaders' __getitem__, the random choice of each cloud's points
(csrc/sample_points.cu), for batches drawn from a dataset kept in device memory.
"""
import numpy as np
import torch

from . import ops

JITTER_PC = (0.01, 0.05)      # jitter_point_cloud defaults, augmentation.py:132 (points, normals)
JITTER_SOM = (0.04, 0.1)      # loader :233


def rotation_matrix_up_axis(angle):
    """augmentation.py:62-68: rotation about the y axis; data . R."""
    c, s = np.cos(angle), np.sin(angle)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def rotation_matrix_perturbation(angles):
    """augmentation.py:112-122: R = Rz . (Ry . Rx) for three small angles."""
    a = angles
    Rx = np.array([[1, 0, 0], [0, np.cos(a[0]), -np.sin(a[0])], [0, np.sin(a[0]), np.cos(a[0])]])
    Ry = np.array([[np.cos(a[1]), 0, np.sin(a[1])], [0, 1, 0], [-np.sin(a[1]), 0, np.cos(a[1])]])
    Rz = np.array([[np.cos(a[2]), -np.sin(a[2]), 0], [np.sin(a[2]), np.cos(a[2]), 0], [0, 0, 1]])
    return np.dot(Rz, np.dot(Ry, Rx))


def draw_params(rng, B, N, M, rot_horizontal=False, rot_perturbation=False,
                translation_perturbation=False, host_noise=False, angle_sigma=0.06,
                angle_clip=0.18):
    """Draw one batch of augmentation parameters from `rng` (np.random.RandomState or the
    np.random module) cloud by cloud in the loader's call order (loader :224-247):
    [angle] [3 perturbation angles] [randn(N,3) points] [randn(N,3) normals] [randn(M,3) nodes]
    scale [shift]. Returns host float64 arrays (None where the option is off)."""
    rot1 = np.empty((B, 3, 3)) if rot_horizontal else None
    rot2 = np.empty((B, 3, 3)) if rot_perturbation else None
    scale = np.empty((B,))
    shift = np.empty((B, 3)) if translation_perturbation else None
    noise = [np.empty((B, N, 3)), np.empty((B, N, 3)), np.empty((B, M, 3))] if host_noise else None
    for b in range(B):
        if rot_horizontal:
            rot1[b] = rotation_matrix_up_axis(rng.uniform() * 2 * np.pi)          # :62
        if rot_perturbation:
            rot2[b] = rotation_matrix_perturbation(
                np.clip(angle_sigma * rng.randn(3), -angle_clip, angle_clip))      # :112
        if host_noise:
            noise[0][b] = rng.randn(N, 3)                                         # :141
            noise[1][b] = rng.randn(N, 3)
            noise[2][b] = rng.randn(M, 3)
        scale[b] = rng.uniform(low=0.8, high=1.2)                                 # loader :236
        if translation_perturbation:
            shift[b] = rng.uniform(-0.1, 0.1, (1, 3))[0]                          # loader :243
    return dict(rot1=rot1, rot2=rot2, scale=scale, shift=shift, noise=noise)


def _dev(a, device):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(
        device, non_blocking=True)


def augment_batch(pc, sn, som, params, seed=0):
    """Apply `params` (from draw_params) to device tensors pc, sn [B,3,N], som [B,3,M]."""
    if not pc.is_cuda:
        raise RuntimeError("sonet_b200.augmentation runs on CUDA tensors only (no CPU fallback)")
    d = pc.device
    noise = params.get("noise") or (None, None, None)
    return ops.augment(pc.contiguous(), None if sn is None else sn.contiguous(),
                       None if som is None else som.contiguous(),
                       rot1=_dev(params.get("rot1"), d), rot2=_dev(params.get("rot2"), d),
                       scale=_dev(params.get("scale"), d), shift=_dev(params.get("shift"), d),
                       jitter_pc=JITTER_PC, jitter_sn=JITTER_PC, jitter_som=JITTER_SOM,
                       noise_pc=_dev(noise[0], d), noise_sn=_dev(noise[1], d),
                       noise_som=_dev(noise[2], d), seed=seed)


def som_knn(som_node, som_k, node_num=None):
    """Batched `som_knn_I` producer: exact kNN among the SOM nodes of every cloud, ascending
    distance, self first — what KNNBuilder.self_build_search returns per item through a CPU Faiss
    IndexFlatL2 (loader :116-150, 256-259). som_node [B,3,M] -> int64 [B,M,som_k]. For
    som_k < 2 the loader emits arange(node_num) as a [M,1] column (:260-261)."""
    B, _, M = som_node.shape
    if som_k >= 2:
        return ops.node_knn(som_node.detach().contiguous(), som_k)
    return torch.arange(M, dtype=torch.int64, device=som_node.device).view(1, M, 1).expand(
        B, M, 1).contiguous()


def prepare_batch(pc, sn, som, opt, train, rng=None, seed=0, host_noise=False):
    """The loader's per-item tail (loader :218-261) for a whole batch on the device:
    augmentation (train mode only) + SOM-node kNN. Returns (pc, sn, som, som_knn_I) ready for
    Model.set_input."""
    if train:
        rng = rng if rng is not None else np.random
        B, _, N = pc.shape
        p = draw_params(rng, B, N, som.shape[2],
                        rot_horizontal=bool(getattr(opt, "rot_horizontal", False)),
                        rot_perturbation=bool(getattr(opt, "rot_perturbation", False)),
                        translation_perturbation=bool(getattr(opt, "translation_perturbation", False)),
                        host_noise=host_noise)
        pc, sn, som = augment_batch(pc, sn, som, p, seed=seed)
    return pc, sn, som, som_knn(som, opt.som_k, opt.node_num)


def _draw_choice(rng, P, N, rule):
    """The loaders' choice of source points for one item, from `rng`: choice(P, N, replace=False)
    (modelnet_shrec_loader.py:198,212) or the ShapeNet rule (shapenet_loader.py:142-154)."""
    if rule == ops.SAMPLE_FILL and N >= P:
        return np.concatenate([np.arange(P), rng.choice(P, N - P, replace=True)])
    return rng.choice(P, N, replace=False)


def draw_batch_host(rng, counts, N, M, rule, train, **flags):
    """Every draw of a batch from `rng` in the loader's per-item order: item b's choice of points,
    then (train) item b's augmentation draws, then item b+1. -> (source indices [B,N] int32,
    draw_params-style dict with host noise, or None when not training)."""
    B = len(counts)
    sel = np.empty((B, N), dtype=np.int32)
    items = []
    for b in range(B):
        sel[b] = _draw_choice(rng, int(counts[b]), N, rule)
        if train:
            items.append(draw_params(rng, 1, N, M, host_noise=True, **flags))
    if not train:
        return sel, None
    cat = lambda k: None if items[0][k] is None else np.concatenate(  # noqa: E731
        [it[k] for it in items])
    params = dict((k, cat(k)) for k in ("rot1", "rot2", "scale", "shift"))
    params["noise"] = [np.concatenate([it["noise"][a] for it in items]) for a in range(3)]
    return sel, params


def _aug_flags(opt):
    """draw_params' flags of the train loader that opt.dataset selects: the ShapeNet loader neither
    rotates nor shifts (shapenet_loader.py:157-180)."""
    flags = dict(rot_horizontal=bool(getattr(opt, "rot_horizontal", False)),
                 rot_perturbation=bool(getattr(opt, "rot_perturbation", False)),
                 translation_perturbation=bool(getattr(opt, "translation_perturbation", False)))
    if getattr(opt, "dataset", None) == "shapenet":
        flags = dict.fromkeys(flags, False)
    return flags


class DeviceDataset:
    """A whole dataset in device memory, drawn from batch by batch: the loaders' complete
    __getitem__ (random point choice, augmentation, SOM-node kNN) plus the collation, on the device.

    points: list of [P_i, 6] arrays (xyz | normal, the column order of the ModelNet .npy files and of
    pc / sn in the npz files); labels: [S] class ids; som_nodes: list of [M, 3]; seg: list of [P_i]
    part labels (ShapeNet) or None. Everything is uploaded once, as fp32 (int32 part labels).

    A float64 source (SHREC's np.loadtxt data) is rounded to fp32 here, once. The loader instead adds
    its jitter and applies the rotations and scale in float64 before its one rounding, so in train
    mode an output value can differ from the loader's by the input rounding carried through
    (at most 2^-24 * scale * |v|, v the point's or node's 3-vector) plus one fp32 ulp of the result.
    Test-mode outputs are the loader's bits."""

    def __init__(self, points, labels, som_nodes, seg=None, device="cuda"):
        S = len(points)
        if S == 0 or len(labels) != S or len(som_nodes) != S or (seg is not None and len(seg) != S):
            raise ValueError("DeviceDataset: points, labels, som_nodes (and seg) need one entry per "
                             "cloud, at least one")
        counts = np.array([np.shape(p)[0] for p in points], dtype=np.int64)
        for i, p in enumerate(points):
            if np.ndim(p) != 2 or np.shape(p)[1] != 6:
                raise ValueError("DeviceDataset: cloud %d has shape %s, expected [P, 6]"
                                 % (i, np.shape(p)))
        if (counts == 0).any():
            raise ValueError("DeviceDataset: cloud %d is empty" % int(np.flatnonzero(counts == 0)[0]))
        M = np.shape(som_nodes[0])[0]
        if any(np.shape(s) != (M, 3) for s in som_nodes):
            raise ValueError("DeviceDataset: every som_nodes entry must be [M, 3] with one M")
        if seg is not None and any(np.shape(s) != (c,) for s, c in zip(seg, counts)):
            raise ValueError("DeviceDataset: seg[i] must be [P_i]")
        self.device = torch.device(device)
        self.counts = counts
        self.max_P = int(counts.max())
        self.node_num = M
        offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        host = np.concatenate([np.asarray(p, dtype=np.float32) for p in points])
        self.data = torch.from_numpy(host).to(self.device)
        self.offsets = torch.from_numpy(offsets).to(self.device)
        self.labels = torch.from_numpy(np.asarray(labels, dtype=np.int64).reshape(S)).to(self.device)
        nodes = np.stack([np.asarray(s, dtype=np.float32).T for s in som_nodes])
        self.som_nodes = torch.from_numpy(np.ascontiguousarray(nodes)).to(self.device)
        self.seg = None if seg is None else torch.from_numpy(
            np.concatenate([np.asarray(s, dtype=np.int32) for s in seg])).to(self.device)

    @classmethod
    def from_device(cls, data, offsets, labels, som_nodes):
        """A dataset from tensors already in device memory (meshes.build_dataset's), without a host
        round trip: data [sum P, 6] f32, offsets [S+1] i64, labels [S] i64, som_nodes [S, 3, M]
        f32, all on one device; no part labels. counts are read back once (S integers)."""
        ds = cls.__new__(cls)
        ds.device = data.device
        ds.counts = np.diff(offsets.cpu().numpy()).astype(np.int64)
        if len(ds.counts) == 0 or (ds.counts <= 0).any():
            raise ValueError("DeviceDataset: every cloud needs at least one point")
        ds.max_P = int(ds.counts.max())
        ds.node_num = som_nodes.shape[2]
        ds.data = data.float().contiguous()
        ds.offsets = offsets.contiguous()
        ds.labels = labels.to(data.device, torch.int64).contiguous()
        ds.som_nodes = som_nodes.float().contiguous()
        ds.seg = None
        return ds

    def __len__(self):
        return len(self.counts)

    def full_clouds(self, index):
        """(points [sum P_i, 6] f32, offsets [len(index)+1] int64, seg [sum P_i] int64 or None) of
        the clouds `index`, all their points, in index order, on the dataset's device: the ragged
        input of segmenter.Model.score_points and losses.compute_iou_full for the batch that
        batch(index, ...) draws. A run of consecutive clouds is a view of the resident points;
        otherwise the rows are gathered."""
        index = np.asarray(index, dtype=np.int64).reshape(-1)
        if len(index) == 0 or index.min() < 0 or index.max() >= len(self.counts):
            raise ValueError("full_clouds: index must name clouds in [0, %d)" % len(self.counts))
        counts = self.counts[index]
        offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)) \
            .to(self.device)
        starts = np.concatenate([[0], np.cumsum(self.counts)])[index]
        if (np.diff(index) == 1).all():
            rows = slice(int(starts[0]), int(starts[0] + counts.sum()))
        else:
            rows = torch.from_numpy(np.concatenate(
                [np.arange(s, s + c) for s, c in zip(starts, counts)])).to(self.device)
        seg = None if self.seg is None else self.seg[rows].long()
        return self.data[rows], offsets, seg

    def full_batch(self, index, opt, train=False, rng=None, seed=0):
        """(points [sum P_i, 6] f32, offsets [len(index)+1] int64, label [len(index)] int64,
        som_node [len(index),3,M] f32, som_knn_I [len(index),M,som_k] int64) of the clouds `index`:
        every point of each (full_clouds), with the loader's SOM nodes and their kNN — the input of
        classifier.Model.score_clouds and networks.Encoder.forward_ragged.
        train=False: no augmentation (the test-mode loader's). train=True: the train loader's
        augmentation of whole clouds, the input of classifier.Model.optimize_clouds: the per-cloud
        scalars from `rng` by draw_params, in the order and with the dataset's flags that
        batch(train=True, host_noise=False) draws them, the jitter in the kernel keyed by `seed`
        (cloud b's row n gets the draws of point n of cloud b in batch()), and the kNN of the
        augmented nodes."""
        points, offsets, _ = self.full_clouds(index)
        cid = torch.from_numpy(np.asarray(index, dtype=np.int64).reshape(-1)).to(self.device)
        som = self.som_nodes.index_select(0, cid)
        if train:
            rng = rng if rng is not None else np.random
            p = draw_params(rng, len(cid), 0, self.node_num, host_noise=False, **_aug_flags(opt))
            d = self.device
            points, som = ops.augment_ragged(
                points.contiguous(), offsets, som, rot1=_dev(p["rot1"], d), rot2=_dev(p["rot2"], d),
                scale=_dev(p["scale"], d), shift=_dev(p["shift"], d), jitter_pc=JITTER_PC,
                jitter_sn=JITTER_PC, jitter_som=JITTER_SOM, seed=seed)
        return (points, offsets, self.labels.index_select(0, cid), som,
                som_knn(som, opt.som_k, self.node_num))

    def batch(self, index, opt, train, rng=None, seed=0, host_noise=False, shard=None):
        """The collated batch of the loader `opt.dataset` selects (autoencoder/train.py:25-36) for
        the clouds `index`, ready for Model.set_input(*...):
          modelnet / shrec: (pc, sn, label, som_node, som_knn_I)        N distinct points per cloud
          shapenet:         (pc, sn, label, seg, som_node, som_knn_I)   the ShapeNet fill rule
        with N = opt.input_pc_num; train=True adds the loader's augmentation (prepare_batch's).
        host_noise=True draws everything from `rng` in the loader's per-item order (the choice of
        item b, then item b's augmentation, then item b+1) and reproduces the loader bit for bit;
        host_noise=False draws the choice and the jitter in the kernels (keyed by `seed`) and only
        the per-cloud scalars from `rng`.
        shard=(rank, world): rows shard_bounds(len(index), rank, world) of the batch the same call
        returns without it (dist.DataParallelTraining's shard). The whole batch is drawn and sliced,
        so every rank must pass the same index, seed and identically seeded `rng`."""
        if shard is not None:
            from .dist import shard_bounds
            lo, hi = shard_bounds(len(np.asarray(index).reshape(-1)), *shard)
            full = self.batch(index, opt, train, rng=rng, seed=seed, host_noise=host_noise)
            return tuple(t[lo:hi] for t in full)
        if opt.dataset in ("modelnet", "shrec"):
            rule = ops.SAMPLE_SUBSET
        elif opt.dataset == "shapenet":
            rule = ops.SAMPLE_FILL
            if self.seg is None:
                raise ValueError("DeviceDataset: the shapenet batch needs seg")
        else:
            raise ValueError("DeviceDataset: unknown dataset %r" % (opt.dataset,))
        ids = np.asarray(index, dtype=np.int64).reshape(-1)
        S = len(self.counts)
        if ((ids < 0) | (ids >= S)).any():
            raise IndexError("DeviceDataset: cloud index out of range [0, %d)" % S)
        B, N, M = len(ids), int(opt.input_pc_num), self.node_num
        P = self.counts[ids]
        if rule == ops.SAMPLE_SUBSET and (P < N).any():
            raise ValueError("Cannot take a larger sample than population when 'replace=False' "
                             "(cloud %d has %d points, N=%d)" % (ids[P < N][0], P[P < N][0], N))
        rng = rng if rng is not None else np.random
        flags = _aug_flags(opt)
        params = None
        indices = None
        if host_noise:
            sel, params = draw_batch_host(rng, P, N, M, rule, train, **flags)
            indices = torch.from_numpy(sel).to(self.device)
        elif train:
            params = draw_params(rng, B, N, M, host_noise=False, **flags)
        cid = torch.from_numpy(ids).to(self.device)
        pc, sn, seg = ops.sample_points(self.data, self.offsets, cid, N, rule, int(P.max()),
                                        labels=self.seg if rule == ops.SAMPLE_FILL else None,
                                        indices=indices, seed=seed)
        som = self.som_nodes.index_select(0, cid)
        if train:
            pc, sn, som = augment_batch(pc, sn, som, params, seed=seed)
        knn = som_knn(som, opt.som_k, M)
        label = self.labels.index_select(0, cid)
        if rule == ops.SAMPLE_FILL:
            return pc, sn, label, seg, som, knn
        return pc, sn, label, som, knn
