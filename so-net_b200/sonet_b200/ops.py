"""Tensor-level wrappers over the C-ABI: validate, allocate outputs, pass the current stream.

Every function here launches hand-written sm_90a kernels from libsonet_b200.so on the tensors'
device and the current torch stream. Inputs must be CUDA, contiguous, of the stated dtype — the
same checks the reference plugin does with CHECK_INPUT (models/index_max_ext/index_max.cpp:119-121),
raised as RuntimeError. Nothing here falls back to PyTorch or the CPU.
"""
import ctypes

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
    [B,N] i32)."""
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


def pointwise_layer(x0, Wt, scale, shift, relu, x1=None, addend=None, gidx=None, out=None):
    """x0 [B,C0,P] (+ x1 [B,C1,P]) -> [B,Cout,P]; Wt [C0+C1,Cout] transposed folded weights."""
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
              _C.ptr(scale), _C.ptr(shift), Cout, int(bool(relu)), _C.ptr(addend), _C.ptr(gidx), G,
              _C.ptr(out), _stream(x0))
    return out


def linear(x, W, scale, shift, relu):
    """x [B,Cin], W [Cout,Cin] -> [B,Cout]."""
    _chk(x, "x", torch.float32)
    _chk(W, "W", torch.float32)
    _chk(scale, "scale", torch.float32, optional=True)
    _chk(shift, "shift", torch.float32, optional=True)
    B, Cin = x.shape
    Cout = W.shape[0]
    with torch.cuda.device(x.device):
        out = torch.empty((B, Cout), dtype=torch.float32, device=x.device)
        _call("sonet_linear_f32", _C.ptr(x), B, Cin, _C.ptr(W), _C.ptr(scale), _C.ptr(shift),
              Cout, int(bool(relu)), _C.ptr(out), _stream(x))
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


def pointresnet_tc(x, blob, fparams, f16=False):
    """x [B,Cin<=6,P] f32 -> [B,384,P]: the fused wgmma first PointResNet (f16: one fp16 product
    per MAC instead of the hi/lo split's three)."""
    _chk(x, "x", torch.float32)
    _chk(blob, "blob", torch.uint8)
    _chk(fparams, "fparams", torch.float32)
    B, Cin, P = x.shape
    with torch.cuda.device(x.device):
        out = torch.empty((B, 384, P), dtype=torch.float32, device=x.device)
        _call(_entry("sonet_pointresnet_tc_forward", f16), _C.ptr(x), Cin, B, P, _C.ptr(blob),
              _C.ptr(fparams), _C.ptr(out), _stream(x))
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


def upconv_hshift(x):
    """x [B,Cin,H,W] -> [3*B, Cin, H*W]: the input shifted horizontally by -1, 0, +1 (zeros at the
    row ends) — the operand of the im2col-free up-convolution (csrc/upconv.cu)."""
    _chk(x, "x", torch.float32)
    B, Cin, H, W = x.shape
    with torch.cuda.device(x.device):
        out = torch.empty((3 * B, Cin, H * W), dtype=torch.float32, device=x.device)
        _call("sonet_upconv_hshift_f32", _C.ptr(x), B, Cin, H, W, _C.ptr(out), _stream(x))
    return out


def pointwise_tc_grouped(x, blob, per_bytes, inv_scale, shift, cout, relu, groups, splits=1,
                         scat_w=0, out=None, scratch=None, conv=False, f16=False):
    """Grouped wgmma layer: x [G*B, C, P], G weight blobs -> out. scat_w = W > 0: the four groups
    are the output parities of an up-convolution over [H, W] maps, interleaved into
    out [B, cout, 4*P]; otherwise out [G*B, cout, P]. splits > 1: K split through `scratch`.
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
              float(inv_scale), _C.ptr(shift), int(cout), int(bool(relu)), int(groups), int(splits),
              int(scat_w), int(scat_w) if conv else 0, int(P_out), int(gstride), _C.ptr(out),
              _C.ptr(scratch), _stream(x),
              kernels=2 if splits > 1 else 1)
    return out


def pointwise_layer_tc(x0, blob, inv_scale, shift, cout, relu, x1=None, addend=None, gidx=None,
                       rows=False, f16=False):
    """wgmma variant of pointwise_layer: x0 [B,C0,P] (+ x1) -> [B,cout,P], or with rows=True the
    same values point-major, [B,P,cout]. f16: one fp16 product per MAC instead of the hi/lo
    split's three."""
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
                  _C.ptr(blob), float(inv_scale), _C.ptr(shift), int(cout), int(bool(relu)),
                  _C.ptr(addend), _C.ptr(gidx), G, _C.ptr(out), _stream(x0))
        else:
            out = torch.empty((B, cout, P), dtype=torch.float32, device=x0.device)
            _call(_entry("sonet_pointwise_tc_forward", f16), _C.ptr(x0), C0, _C.ptr(x1), C1, B, P,
                  _C.ptr(blob),
                  float(inv_scale), _C.ptr(shift), int(cout), int(bool(relu)), _C.ptr(addend),
                  _C.ptr(gidx), G, _C.ptr(out), _stream(x0))
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


def knn_mlp_tc(coord, center, idx, K, Y, w1, blob, inv_scale, shift2, f16=False):
    """The KNN module's layer 1 (from the per-node Y = W1f x [B,512,M]) + layer 2 + max over the
    K neighbours in one wgmma kernel. coord, center [B,3,M]; idx [B,M,K'] i64; w1 [512,4] =
    (W1d | shift1); shift2 [512] -> knn_feature_1 [B,512,M]. Y is [B,512,M] either contiguous or
    the channel-fastest view y.transpose(1, 2) of a contiguous [B,M,512] (pointwise_layer_tc(...,
    rows=True)); the kernel reads the latter as float2 pairs, with bit-identical results.
    f16: layer 2 as one fp16 product per MAC instead of the hi/lo split's three."""
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
        _call(_entry("sonet_knn_mlp_tc_forward", f16), _C.ptr(coord), _C.ptr(center), _C.ptr(idx), B,
              M, int(K), idx.shape[2], _C.ptr(Y), Y.stride(1), Y.stride(2), _C.ptr(w1), _C.ptr(blob),
              float(inv_scale), _C.ptr(shift2), _C.ptr(out), _stream(coord))
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
SOM_GROUP_NONE, SOM_GROUP_UNSTAGED, SOM_GROUP_STAGED = 0, 1, 2


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
                        f16=False):
    """Fused wgmma PointResNet + per-node max: -> first_pn_out_masked_max [B,384,M], or with
    finalize=False the raw (keys [B,384,M] i32, p0 [B,384]) for knn_assemble_pool / pool_finalize.
    f16: one fp16 product per MAC instead of the hi/lo split's three."""
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
        _call(_entry("sonet_pointresnet_tc_pool_forward", f16), _C.ptr(x_sorted), Cin, B, P,
              _C.ptr(blob),
              _C.ptr(fparams), _C.ptr(node_sorted), _C.ptr(pos0), int(M), _C.ptr(keys), _C.ptr(p0),
              _stream(x_sorted))
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
