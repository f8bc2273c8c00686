"""oracle.py — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

CPU restatement (torch-CPU ATen calls + plain C for the index arithmetic) of the reference's
per-batch forward hot path. It exists only to check the CUDA path: it may be imported by tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs, never by anything
under so-net_b200/.

The functions are written from the reference's *dataflow* (cited per function, paths relative to
lijx10/SO-Net) using the same ATen operators the reference calls (conv1d, batch_norm, topk, sum,
gather), so that it is both the parity checker and a faithful CPU baseline ("port") of the
reference PyTorch-CPU path. Weights are passed as a flat state_dict with the reference's keys.

Pinning (SURVEY.md §8c): the reference has no tests or golden vectors. This oracle is pinned by
tests/golden/*.npz — outputs of the REFERENCE ITSELF (/root/reference imported unmodified with
the three shims of oracle/ref_shims.py) generated in the build container by
oracle/make_golden.py — and by the reference's own compiled index_max plugin (oracle/_ref).
Chamfer's nearest-neighbour search is Faiss in the reference (not vendored, no version pin):
restated as exact brute force => "parity unpinned" at that boundary for near-tie index choices.
"""
import ctypes
import importlib.util
import os

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
_clib = None
_ref_plugin = None


def clib():
    global _clib
    if _clib is None:
        path = os.path.join(HERE, "_build", "liboracle_c.so")
        if not os.path.exists(path):
            from . import build as _b
            _b.build_c()
        _clib = ctypes.CDLL(path)
    return _clib


def ref_plugin():
    """The reference's own compiled `index_max` module (oracle/_ref), or None if not built."""
    global _ref_plugin
    if _ref_plugin is None:
        from . import build as _b
        path = _b.ref_plugin_path()
        if path is None:
            return None
        spec = importlib.util.spec_from_file_location("index_max", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _ref_plugin = mod
    return _ref_plugin


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


# ---- index_max --------------------------------------------------------------------------------------
def index_max(data, index, K):
    """models/index_max_ext/index_max.cpp:73-112. data [B,C,N] f32, index [B,N] i32 -> [B,C,K] i32."""
    data = data.contiguous().float()
    index = index.contiguous().to(torch.int32)
    B, C, N = data.shape
    out = torch.zeros((B, C, K), dtype=torch.int32)
    clib().oracle_index_max(_p(data), _p(index), B, C, N, int(K), _p(out))
    return out


def index_max_fast(data, index, K, threads=None):
    """Fastest CPU implementation available for baseline timing: the reference's compiled plugin
    (forward_multi_thread_cpu, index_max.cpp:33-70) when oracle/_ref exists, else the C port."""
    m = ref_plugin()
    if m is not None:
        threads = threads or os.cpu_count() or 1
        threads = max(1, min(threads, data.shape[1]))
        return m.forward_multi_thread_cpu(data.contiguous(), index.contiguous().to(torch.int32),
                                          int(K), int(threads))
    return index_max(data, index, K)


# ---- SOM assignment ------------------------------------------------------------------------------------
def som_topk(x, node, k):
    """util/som.py:245-253 via the C restatement. -> min_idx [B,kN] int32 (slot-major, ascending
    distance), min_dist [B,kN] f32."""
    x = x.contiguous().float()
    node = node.contiguous().float()
    B, _, N = x.shape
    M = node.shape[2]
    idx = torch.zeros((B, k * N), dtype=torch.int32)
    dist = torch.zeros((B, k * N), dtype=torch.float32)
    clib().oracle_som_topk(_p(x), _p(node), B, N, M, int(k), _p(idx), _p(dist))
    return idx, dist


def query_topk(x, node, k, sorted_slots=False):
    """BatchSOM.query_topk, util/som.py:237-269, with the same ATen ops -> (mask [B,kN,M] int32,
    mask_row_max [B,M] int32, min_idx [B,kN] int64).

    sorted_slots: the reference calls topk(sorted=False), whose slot order is implementation
    defined (it differs between torch's CPU and CUDA kernels and between sizes). The order only
    matters through one quirk: an EMPTY node gathers "the feature of stacked copy 0"
    (models/networks.py:185), i.e. of point 0 decentred by whatever node topk put in slot 0.
    sorted_slots=True picks the instance "slot order = ascending distance" — the order the CUDA
    path emits — so that tensors downstream of empty nodes can be compared exactly."""
    M = node.shape[2]
    node_e = node.unsqueeze(2).expand(x.size(0), x.size(1), x.size(2), M)
    diff = x.unsqueeze(3).expand_as(node_e) - node_e
    diff_norm = (diff ** 2).sum(dim=1)
    _, min_idx = torch.topk(diff_norm, k=k, dim=2, largest=False, sorted=bool(sorted_slots))   # B,N,k
    ids = torch.arange(M, dtype=torch.int64).view(1, 1, M, 1)
    mask = torch.eq(min_idx.unsqueeze(2).expand(-1, -1, M, -1), ids).int()        # B,N,M,k
    mask = torch.cat([mask[..., i] for i in range(k)], dim=1)                      # B,kN,M
    min_idx = torch.cat([min_idx[..., i] for i in range(k)], dim=1)                # B,kN
    mask_row_max, _ = torch.max(mask, dim=1)
    return mask, mask_row_max, min_idx


def canon_sets(min_idx, k):
    """Per-point sorted k-set of node indices: [B,kN] slot-major -> [B,N,k] sorted (the parity
    definition for the assignment, SURVEY.md Appendix C)."""
    B, kN = min_idx.shape
    N = kN // k
    return torch.sort(min_idx.view(B, k, N).permute(0, 2, 1).long(), dim=2)[0]


# ---- batch-SOM training (§8f-4) -------------------------------------------------------------------
def som_init_weighting_matrix(rows, cols, sigma=0.4):
    """BatchSOM.gaussian / get_init_weighting_matrix, util/som.py:214-229 -> [M, rows, cols]."""
    d = 2 * np.pi * sigma * sigma
    w = torch.empty(rows * cols, rows, cols)
    for idx in range(rows * cols):
        i, j = idx // cols, idx % cols
        ax = np.exp(-np.power(np.arange(rows) - i, 2) / d)
        ay = np.exp(-np.power(np.arange(cols) - j, 2) / d)
        w[idx] = torch.from_numpy(np.outer(ax, ay).astype(np.float32))
    return w


def som_batch_update(node, x, init_w, learning_rate, sigma, sigma0=0.4):
    """BatchSOM.batch_update, util/som.py:295-347, with the same ATen ops. node [B,3,M] (a new
    tensor is returned), x [B,3,N], init_w [M,rows,cols]."""
    B, C, N = x.shape
    M, rows, cols = init_w.shape
    node_e = node.unsqueeze(2).expand(B, C, N, M)                               # :301
    x_e = x.unsqueeze(3).expand_as(node_e)
    diff_norm = ((x_e - node_e) ** 2).sum(dim=1)                                # :305-306
    _, min_idx = torch.min(diff_norm, dim=2)                                    # :309
    ids = torch.arange(M, dtype=torch.int64).view(1, 1, M)
    mask = torch.eq(min_idx.unsqueeze(2).expand(B, N, M), ids).float()          # :310-314
    mask_row_sum = torch.sum(mask, dim=1) + 0.00001                             # :315
    mask_row_max, _ = torch.max(mask, dim=1)                                    # :316
    masked_sum = torch.sum(x_e * mask.unsqueeze(1).expand_as(x_e), dim=2)       # :319-320
    mean = masked_sum / mask_row_sum.unsqueeze(1).expand_as(masked_sum)         # :321-322
    mean_e = mean.unsqueeze(3).expand(B, C, M, M)                               # :326-328
    diff = mean_e - node.unsqueeze(2).expand_as(mean_e)                         # :329-330
    diff = diff * mask_row_max.unsqueeze(2).unsqueeze(1).expand_as(diff)        # :331
    scale = 1.0 / ((sigma / sigma0) ** 2)                                       # :232-235
    W = torch.exp(torch.log(init_w) * scale)
    W = W.unsqueeze(0).unsqueeze(1).expand(B, C, M, rows, cols)                 # :337-342
    delta = (diff.view(B, C, M, rows, cols) * W * learning_rate).sum(dim=2)     # :343-347
    return (node.view(B, C, rows, cols) + delta).view(B, C, M), min_idx


def som_optimize(x, node_init_value, rows, cols, lr0=0.5, sigma0=0.4, max_iteration=60):
    """BatchSOM.optimize, util/som.py:352-366. node_init_value [3,M] (the potential-field start,
    which tests take from the golden file — it is numpy-RNG-seeded host preprocessing)."""
    init_w = som_init_weighting_matrix(rows, cols, sigma0)
    node = node_init_value.unsqueeze(0).expand(x.shape[0], -1, -1).contiguous()
    for _ in range(int(max_iteration / 3)):
        node, _ = som_batch_update(node, x, init_w, lr0, sigma0, sigma0)
    for it in range(max_iteration):
        node, _ = som_batch_update(node, x, init_w, lr0 / (1 + 2 * it / max_iteration),
                                   sigma0 / (1 + 2 * it / max_iteration), sigma0)
    return node


# ---- layers (eval mode) -------------------------------------------------------------------------------
def _bn(y, st, prefix):
    return F.batch_norm(y, st[prefix + ".running_mean"], st[prefix + ".running_var"],
                        st[prefix + ".weight"], st[prefix + ".bias"], False, 0.1, 1e-5)


def equivariant(x, st, prefix):
    """EquivariantLayer.forward, models/layers.py:282-296: conv1d(k=1) -> BN (if present) -> ReLU
    (if present). A layer has BN+ReLU iff its state has norm.* (PointNet's last layer is bare)."""
    y = F.conv1d(x, st[prefix + ".conv.weight"], st[prefix + ".conv.bias"])
    if prefix + ".norm.weight" in st:
        y = F.relu(_bn(y, st, prefix + ".norm"))
    return y


def conv2d_1x1(x, st, prefix):
    """MyConv2d.forward, models/layers.py:203-210."""
    y = F.conv2d(x, st[prefix + ".conv.weight"], st[prefix + ".conv.bias"])
    if prefix + ".norm.weight" in st:
        y = F.relu(_bn(y, st, prefix + ".norm"))
    return y


def mylinear(x, st, prefix):
    """MyLinear.forward, models/layers.py:155-166."""
    y = F.linear(x, st[prefix + ".linear.weight"], st[prefix + ".linear.bias"])
    if prefix + ".norm.weight" in st:
        y = F.relu(_bn(y, st, prefix + ".norm"))
    return y


def _n_layers(st, prefix):
    n = 0
    while "%s.layers.%d.conv.weight" % (prefix, n) in st:
        n += 1
    return n


def pointnet(x, st, prefix):
    """PointNet.forward, models/layers.py:384-387."""
    for i in range(_n_layers(st, prefix)):
        x = equivariant(x, st, "%s.layers.%d" % (prefix, i))
    return x


def pointresnet(x, st, prefix):
    """PointResNet.forward, models/layers.py:419-432."""
    n = _n_layers(st, prefix)
    l0 = equivariant(x, st, prefix + ".layers.0")
    t = l0
    for i in range(1, n - 1):
        t = equivariant(t, st, "%s.layers.%d" % (prefix, i))
    return equivariant(torch.cat((l0, t), dim=1), st, "%s.layers.%d" % (prefix, n - 1))


def knn_gather(src, knn_I):
    """operations.knn_gather_by_indexing, models/operations.py:38-54."""
    B, C, N = src.shape
    K = knn_I.shape[2]
    idx = knn_I.unsqueeze(1).expand(B, C, N, K).contiguous().view(B, C, N * K)
    return torch.gather(src, 2, idx).view(B, C, N, K)


def node_knn(coord, K):
    """The precomputed_knn_I=None branch, models/layers.py:334-337."""
    d = torch.sum((coord.unsqueeze(3) - coord.unsqueeze(2)) ** 2, dim=1)
    return torch.topk(d, k=K, dim=2, largest=False, sorted=True)[1]


def knn_module(coord, x, knn_I, K, center_type, st, prefix):
    """KNNModule.forward, models/layers.py:313-367."""
    knn_I = knn_I[:, :, 0:K] if knn_I is not None else node_knn(coord, K)
    neighbors = knn_gather(coord, knn_I)
    if center_type == 'avg':
        center = torch.mean(neighbors, dim=3, keepdim=True)
    else:
        center = coord.unsqueeze(3)
    h = torch.cat((neighbors - center, knn_gather(x, knn_I)), dim=1)
    for i in range(_n_layers(st, prefix)):
        h = conv2d_1x1(h, st, "%s.layers.%d" % (prefix, i))
    return center.squeeze(3), torch.max(h, dim=3)[0]


# ---- networks -----------------------------------------------------------------------------------------
def encoder_forward(st, opt, x, sn, node, node_knn_I, fast_pool=False, sorted_slots=False):
    """Encoder.forward, models/networks.py:111-199 (eval mode). Returns a dict of every cached
    attribute. `st` = encoder state_dict. fast_pool: use the fastest CPU index_max (baseline
    timing) instead of the single-thread restatement."""
    k = opt.k
    M = node.shape[2]
    # index decisions always in fp32 (the reference's arithmetic); the value path follows x.dtype,
    # so a float64 state + float64 inputs give the fp64 evaluation the precision tests compare with
    mask, mask_row_max, min_idx = query_topk(x.float(), node.float(), k, sorted_slots)   # networks.py:127
    mask_row_sum = torch.sum(mask, dim=1)                                   # :128
    maskf = mask.unsqueeze(1).to(x.dtype)
    x_stack = torch.cat((x,) * k, dim=2)                                    # :132-137
    sn_stack = torch.cat((sn,) * k, dim=2)
    cluster_mean = torch.sum(x_stack.unsqueeze(3) * maskf, dim=2) / \
        (mask_row_sum.unsqueeze(1).to(x.dtype) + 1e-5)                      # :140-142
    som_node = cluster_mean
    centers = torch.sum(maskf * som_node.unsqueeze(2), dim=3)               # :168-169
    x_dec = x_stack - centers                                               # :171
    x_aug = torch.cat((x_dec, sn_stack), dim=1) if opt.surface_normal else x_dec
    first = pointresnet(x_aug, st, "first_pointnet")                        # :176
    if fast_pool:   # baseline timing; an int selects the thread count
        gather_index = index_max_fast(first.float(), min_idx.int(), M,
                                      None if fast_pool is True else int(fast_pool)).long()
    else:
        gather_index = index_max(first.float().contiguous(), min_idx.int(), M).long()   # :181-184
    masked_max = first.gather(2, gather_index * mask_row_max.unsqueeze(1).long())  # :185
    out = dict(mask=mask, mask_row_max=mask_row_max, min_idx=min_idx, mask_row_sum=mask_row_sum,
               som_node=som_node, centers=centers, x_decentered=x_dec, first_pn_out=first,
               gather_index=gather_index, first_pn_out_masked_max=masked_max)
    if opt.som_k >= 2:
        kc, kf = knn_module(som_node, masked_max, node_knn_I, opt.som_k, opt.som_k_type, st,
                            "knnlayer")                                     # :189
        final = pointnet(torch.cat((kc, kf), dim=1), st, "final_pointnet")  # :192
        out.update(knn_center_1=kc, knn_feature_1=kf)
    else:
        final = pointresnet(torch.cat((som_node, masked_max), dim=1), st, "final_pointnet")  # :195
    out["final_pn_out"] = final
    out["feature"] = torch.max(final, dim=2)[0]                             # :197
    return out


def classifier_forward(st, feature):
    """Classifier.forward, models/networks.py:218-227 (eval: dropout = identity)."""
    return mylinear(mylinear(mylinear(feature, st, "fc1"), st, "fc2"), st, "fc3")


def segmenter_forward(st, opt, enc, x, sn, label):
    """models/segmenter.py:90-109 (per-point gathers) + Segmenter.forward,
    models/networks.py:259-344. `enc` = encoder_forward() result."""
    B, N = x.shape[0], x.shape[2]
    k = opt.k
    kN = k * N
    idx = torch.max(enc["mask"], dim=2)[1].unsqueeze(1)                     # segmenter.py:90-91
    g = lambda t: torch.gather(t, 2, idx.expand(B, t.shape[1], kN))         # noqa: E731  :96-98
    onehot = torch.zeros(B, 16, dtype=x.dtype).scatter_(1, label.unsqueeze(1), 1) \
        .unsqueeze(2).expand(B, 16, kN)
    parts = [enc["x_decentered"], torch.cat((x,) * k, dim=2), enc["centers"]]
    if opt.surface_normal:
        parts.append(torch.cat((sn,) * k, dim=2))
    parts += [onehot, enc["first_pn_out"], g(enc["first_pn_out_masked_max"])]
    if opt.som_k >= 2:
        parts.append(g(enc["knn_feature_1"]))
    parts += [g(enc["final_pn_out"]), enc["feature"].unsqueeze(2).expand(B, -1, kN)]
    h = torch.cat(parts, dim=1)                                             # networks.py:300-305
    for name in ("layer1", "layer2", "layer3"):
        h = equivariant(h, st, name)
    sp = torch.split(h, N, dim=2)                                           # :331-336
    avg = 0.5 * (sp[0] + sp[1]) if k == 2 else (1.0 / 3.0) * (sp[0] + sp[1] + sp[2])
    return equivariant(equivariant(avg, st, "layer4"), st, "layer5")


# ---- Chamfer -------------------------------------------------------------------------------------------
def nn_search(query, db):
    """faiss.IndexFlatL2 k=1 (models/losses.py:209-235) as exact brute force.
    query [3,Q], db [3,D] -> (idx [Q] int32, dist2 [Q] float32).

    dist2 is the fp32 squared distance of the selected pair, ((dx*dx + dy*dy) + dz*dz) with every
    op rounded separately: the scan's minimum, or, for a query no candidate beats +inf for (index
    0, every distance NaN or +inf), the distance to db point 0 (NaN or +inf)."""
    query = query.contiguous().float()
    db = db.contiguous().float()
    Q, D = query.shape[1], db.shape[1]
    idx = torch.zeros(Q, dtype=torch.int32)
    dist2 = torch.zeros(Q, dtype=torch.float32)
    clib().oracle_nn_search(_p(query), Q, _p(db), D, _p(idx), _p(dist2))
    none = torch.isinf(dist2)
    if bool(none.any()):
        dist2[none] = pair_dist2(query[:, none], db[:, :1].expand(3, int(none.sum())))
    return idx, dist2


def pair_dist2(a, b):
    """fp32 ((dx*dx + dy*dy) + dz*dz) of a [3,P] and b [3,P] point by point, every op rounded
    separately (numpy float32 ops are correctly rounded and never contracted)."""
    with np.errstate(all="ignore"):     # NaN and overflow are part of what is checked
        d = a.numpy().astype(np.float32) - b.numpy().astype(np.float32)
        return torch.from_numpy((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])


def chamfer_elem(dist2):
    """The kernel's per-point term sqrt(dist2 + 1e-8) in fp32, each op correctly rounded."""
    d = dist2.numpy().astype(np.float32)
    with np.errstate(all="ignore"):
        return torch.from_numpy(np.sqrt(d + np.float32(1e-8)))


def chamfer(predict_pc, gt_pc):
    """ChamferLoss.forward, models/losses.py:237-290. -> dict(loss, forward_loss, backward_loss,
    forward_loss_array, backward_loss_array, loss_array, idx_fwd, idx_bwd, dist2_fwd, dist2_bwd);
    dist2_* [B,P] are nn_search's fp32 squared distances of the selected pairs."""
    B = predict_pc.shape[0]
    sel_gt, sel_pr, i_f, i_b, d_f, d_b = [], [], [], [], [], []
    for i in range(B):                                                      # losses.py:260-276
        fi, df = nn_search(predict_pc[i], gt_pc[i])
        bi, db = nn_search(gt_pc[i], predict_pc[i])
        fi, bi = fi.long(), bi.long()
        sel_gt.append(gt_pc[i].index_select(1, fi))
        sel_pr.append(predict_pc[i].index_select(1, bi))
        i_f.append(fi)
        i_b.append(bi)
        d_f.append(df)
        d_b.append(db)
    sel_gt = torch.stack(sel_gt).unsqueeze(1)                               # B,1,3,M
    sel_pr = torch.stack(sel_pr).unsqueeze(1)
    rn = lambda v: ((v ** 2).sum(dim=2) + 1e-8).sqrt()                      # noqa: E731  :17-27
    f_el = rn(sel_gt - predict_pc.unsqueeze(1))                             # :281
    b_el = rn(sel_pr - gt_pc.unsqueeze(1))                                  # :286
    fa, ba = f_el.mean(dim=1).mean(dim=1), b_el.mean(dim=1).mean(dim=1)
    return dict(loss=f_el.mean() + b_el.mean(), forward_loss=f_el.mean(),
                backward_loss=b_el.mean(), forward_loss_array=fa, backward_loss_array=ba,
                loss_array=fa + ba, idx_fwd=torch.stack(i_f), idx_bwd=torch.stack(i_b),
                dist2_fwd=torch.stack(d_f), dist2_bwd=torch.stack(d_b))


def split_state(state, prefix):
    """Sub-state_dict of a module: keys starting with `prefix.` with the prefix removed."""
    p = prefix + "."
    return {k[len(p):]: v for k, v in state.items() if k.startswith(p)}


def to_numpy_tree(d):
    return {k: (v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v))
            for k, v in d.items()}
