"""The reference's models/losses.py API on our kernels.

ChamferLoss (losses.py:17-27, 192-296): the reference builds two Faiss IndexFlatL2 per cloud and
round-trips through host numpy (losses.py:247-276). Here both nearest-neighbour searches of the
whole batch, the sqrt(d^2 + 1e-8) terms and all means run on the device in four launches
(csrc/chamfer.cu). No Faiss dependency. chamfer_ragged: the same numbers against whole
ground-truth clouds of any size, for evaluation; seg_loss_ragged: CrossEntropyLossSeg's evaluation
loss over whole shapes of any size (csrc/seg_loss.cu).

compute_iou_np_array / compute_iou (losses.py:73-189), the part-segmentation metric of
part-seg/train.py:95: one kernel for CUDA tensors, the same arithmetic in C++ for host tensors
(csrc/seg_iou.cu); PartSegIoU accumulates it over an evaluation loop without a sync per batch.
"""
import json
import os
from collections import OrderedDict, namedtuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _C, ops

SHAPENET_PART_TABLE = ops.SHAPENET_PART_TABLE


def robust_norm(var):
    """var [B,C,H,W] -> sqrt(sum over dim 2 of var^2 + 1e-8), [B,C,W] (losses.py:17-27)."""
    return ((var ** 2).sum(dim=2) + 1e-8).sqrt()


class CrossEntropyLossSeg(nn.Module):
    """Per-point NLL over [B,classes,N] scores and [B,N] targets (models/losses.py:30-43).
    Evaluation (no gradient asked for, fp32 CUDA scores, no class weights): one fused kernel +
    a deterministic final sum (csrc/seg_loss.cu); training: PyTorch's differentiable op."""

    def __init__(self, weight=None, size_average=True):
        super().__init__()
        self.weight = weight
        self.reduction = 'mean' if size_average else 'sum'

    def forward(self, inputs, targets):
        if (self.weight is None and inputs.is_cuda and inputs.dtype == torch.float32
                and inputs.dim() == 3 and targets.dtype == torch.int64 and targets.is_cuda
                and not (torch.is_grad_enabled() and inputs.requires_grad)):
            return ops.seg_loss(inputs.contiguous(), targets.contiguous(),
                                size_average=self.reduction == 'mean')
        return F.cross_entropy(inputs, targets, weight=self.weight, reduction=self.reduction)


class ChamferLoss(nn.Module):
    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.dimension = 3
        self.k = 1
        self.forward_loss = torch.FloatTensor([0])
        self.backward_loss = torch.FloatTensor([0])

    def forward(self, predict_pc, gt_pc):
        """predict_pc [B,3,M], gt_pc [B,3,N] (CUDA) -> scalar loss; also sets forward_loss,
        backward_loss, forward_loss_array, backward_loss_array, loss_array (losses.py:281-289).

        Nearest neighbours are exact, lowest index on ties. A point with no finite nearest
        neighbour (every candidate's squared distance is NaN or overflows to +inf) is paired with
        the other cloud's point 0, as a brute-force scan from (+inf, index 0) would: its term is
        NaN if either point has a NaN coordinate, +inf on overflow. So non-finite inputs give a
        NaN or inf loss, in training as in evaluation, and nn_idx_fwd / nn_idx_bwd stay in range."""
        if not predict_pc.is_cuda:
            raise RuntimeError("sonet_b200.ChamferLoss runs on CUDA tensors only (no CPU fallback)")
        need_grad = torch.is_grad_enabled() and (predict_pc.requires_grad or gt_pc.requires_grad)
        r = ops.chamfer(predict_pc.detach().contiguous().float(),
                        gt_pc.detach().contiguous().float(), want_idx=need_grad)
        self.nn_idx_fwd, self.nn_idx_bwd = r["idx_fwd"], r["idx_bwd"]
        if not need_grad:
            self.forward_loss, self.backward_loss = r["loss"][0], r["loss"][1]
            self.forward_loss_array, self.backward_loss_array = r["fwd_arr"], r["bwd_arr"]
            self.loss_array = self.forward_loss_array + self.backward_loss_array
            return r["loss"][2]
        # training: the search is the kernel's; the loss is re-expressed with differentiable
        # gathers (gradient w.r.t. predict_pc as in losses.py:269, 276)
        i_f = r["idx_fwd"].long().unsqueeze(1).expand(-1, 3, -1)
        i_b = r["idx_bwd"].long().unsqueeze(1).expand(-1, 3, -1)
        sel_gt = torch.gather(gt_pc, 2, i_f).unsqueeze(1)          # B x 1 x 3 x M
        sel_pr = torch.gather(predict_pc, 2, i_b).unsqueeze(1)     # B x 1 x 3 x N
        f_el = robust_norm(sel_gt - predict_pc.unsqueeze(1))
        b_el = robust_norm(sel_pr - gt_pc.unsqueeze(1))
        self.forward_loss = f_el.mean()
        self.forward_loss_array = f_el.mean(dim=1).mean(dim=1)
        self.backward_loss = b_el.mean()
        self.backward_loss_array = b_el.mean(dim=1).mean(dim=1)
        self.loss_array = self.forward_loss_array + self.backward_loss_array
        return self.forward_loss + self.backward_loss

    def __call__(self, predict_pc, gt_pc):
        return self.forward(predict_pc, gt_pc)


ChamferRagged = namedtuple("ChamferRagged", ("loss", "forward_loss", "backward_loss", "loss_array",
                                             "fwd_arr", "bwd_arr"))


def chamfer_ragged(predict_pc, points, offsets):
    """ChamferLoss's evaluation numbers against whole clouds of any size: predict_pc [B,3,Mp] (CUDA)
    against ground-truth clouds points [T,>=3] (xyz first; DeviceDataset's [T,6]), cloud b rows
    offsets[b] .. offsets[b+1]. Returns ChamferRagged(loss, forward_loss, backward_loss, loss_array,
    fwd_arr, bwd_arr), the values ChamferLoss.forward returns and sets in evaluation.

    Cloud b's numbers are ChamferLoss's on that cloud alone, at N = P_b. forward_loss and
    backward_loss are means over the clouds of the per-cloud means, so each cloud counts once
    whatever its size: with equal sizes that is the reference's b_el.mean(), and with ragged sizes
    it keeps large clouds from dominating. Evaluation only: a gradient cannot flow through it, so
    predict_pc or points requiring one with grad mode on is refused."""
    if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad
                                       for t in (predict_pc, points)):
        raise RuntimeError("chamfer_ragged is evaluation only: no gradient flows through it "
                           "(call it under torch.no_grad() or on detached tensors)")
    if not isinstance(predict_pc, torch.Tensor) or not predict_pc.is_cuda:
        raise RuntimeError("sonet_b200.chamfer_ragged runs on CUDA tensors only (no CPU fallback)")
    r = ops.chamfer_ragged(predict_pc.detach().contiguous(), points.detach(), offsets)
    return ChamferRagged(r["loss"][2], r["loss"][0], r["loss"][1], r["fwd_arr"] + r["bwd_arr"],
                         r["fwd_arr"], r["bwd_arr"])


def seg_loss_ragged(score, seg, offsets):
    """CrossEntropyLossSeg's evaluation loss over whole shapes of any size: score [T,classes] (CUDA,
    point-major, as segmenter.Model.segment_clouds and score_points return it), seg [T] int64 part
    labels (-100: not counted), cloud b rows offsets[b] .. offsets[b+1]. Returns (loss,
    loss_array): loss is the mean over every counted point of the batch, CrossEntropyLossSeg's rule
    (with equal sizes, its bits on the [B,classes,N] scores); loss_array [B] is each shape's own
    mean, so loss_array.mean() weighs every shape once whatever its size. An out-of-range label
    other than -100 makes its shape's mean and loss NaN. Evaluation only: a score requiring a
    gradient with grad mode on is refused."""
    if torch.is_grad_enabled() and isinstance(score, torch.Tensor) and score.requires_grad:
        raise RuntimeError("seg_loss_ragged is evaluation only: no gradient flows through it "
                           "(call it under torch.no_grad() or on a detached score)")
    if not isinstance(score, torch.Tensor) or not score.is_cuda:
        raise RuntimeError("sonet_b200.seg_loss_ragged runs on CUDA tensors only (no CPU fallback)")
    return ops.seg_loss_ragged(score.detach().contiguous(), seg.contiguous(), offsets.contiguous())


def _seg_iou(score, seg, label, table=None, want_correct=False):
    """Per-shape IoU [B] float64 (and correct-point counts [B] int32) on score's device: the sm_90a
    kernel for CUDA scores (no sync; a label outside the table gives NaN), the library's host entry
    for CPU scores (a label outside the table raises)."""
    if score.dtype != torch.float32:
        raise RuntimeError("seg_iou: score must be float32 (got %s)" % score.dtype)
    score = score.detach().contiguous()
    seg = seg.detach().to(score.device, torch.int64).contiguous()
    label = label.detach().to(score.device, torch.int64).contiguous()
    if score.is_cuda:
        iou, _, correct = ops.seg_iou(score, seg, label, table, want_correct=want_correct)
        return iou, correct
    B, C, N = ops._seg_iou_args(score, seg, label)
    offsets, ids, K = ops.part_table_csr(table, C, score.device)
    iou = torch.empty((B,), dtype=torch.float64)
    correct = torch.empty((B,), dtype=torch.int32) if want_correct else None
    _C.check(_C.lib().sonet_seg_iou_cpu_f32(score.data_ptr(), seg.data_ptr(), label.data_ptr(), B, C,
                                            N, offsets.data_ptr(), ids.data_ptr(), K, iou.data_ptr(),
                                            None, _C.ptr(correct), torch.get_num_threads()),
             "sonet_seg_iou_cpu_f32")
    return iou, correct


def _host_iou(iou):
    out = iou.cpu().numpy()
    if np.isnan(out).any():
        raise RuntimeError("seg_iou: label outside the part table (cloud %d)"
                           % int(np.flatnonzero(np.isnan(out))[0]))
    return out


def compute_iou_np_array(score, seg, label, visualizer, opt, input_pc):
    """score [B,C,N] float32, seg [B,N], label [B] (integer) -> per-shape IoU, float64 numpy [B]
    (models/losses.py:73-116): for each part of the shape's ShapeNetPart category, I / (U + 1e-4)
    of the predicted (argmax over C) and ground-truth point sets, or 1.0 if the part is absent
    from both; their mean. Bit-equal to the reference. CUDA scores run one kernel, host scores the
    library's C++ entry. visualizer, opt and input_pc are accepted and ignored, as in the reference.
    Unlike the reference, whose list indexing wraps negative labels, a label outside [0, 16) raises
    RuntimeError."""
    return _host_iou(_seg_iou(score, seg, label)[0])


def compute_iou(score, seg, label, visualizer, opt, input_pc):
    """Mean over the batch of compute_iou_np_array (models/losses.py:119-189), as np.float64."""
    return compute_iou_np_array(score, seg, label, visualizer, opt, input_pc).mean()


def compute_iou_full(score, seg, label, offsets, table=None):
    """Per-shape IoU over ALL points of each shape, float64 numpy [B]: compute_iou_np_array's rule
    (argmax over all classes, then per part of the shape's category I / (U + 0.0001), 1.0 for an
    empty union, averaged over the parts) on ragged shapes. score [sum P_i, C] f32 (what
    segmenter.Model.score_points returns), seg [sum P_i], label [B], offsets [B+1] int64. CUDA
    scores run one kernel, host scores the library's C++ entry; both give the same bits. Its mean
    is compute_iou's number at full resolution. Bad offsets or a label outside the table raise."""
    if score.dtype != torch.float32 or score.dim() != 2:
        raise RuntimeError("compute_iou_full: score must be float32 [T, C] (got %s %s)"
                           % (score.dtype, tuple(score.shape)))
    score = score.detach().contiguous()
    seg = seg.detach().to(score.device, torch.int64).contiguous()
    label = label.detach().to(score.device, torch.int64).contiguous()
    ops.ragged_offsets(offsets, score.shape[0], label.shape[0])
    offsets = offsets.detach().to(score.device).contiguous()
    if score.is_cuda:
        return _host_iou(ops.seg_iou_ragged(score, seg, label, offsets, table)[0])
    if tuple(seg.shape) != (score.shape[0],):
        raise RuntimeError("compute_iou_full: seg must be [T] (got %s)" % (tuple(seg.shape),))
    T, C = score.shape
    B = label.shape[0]
    poff, ids, K = ops.part_table_csr(table, C, score.device)
    iou = torch.empty((B,), dtype=torch.float64)
    _C.check(_C.lib().sonet_seg_iou_ragged_cpu_f32(
        score.data_ptr(), seg.data_ptr(), label.data_ptr(), offsets.data_ptr(), B, C, T,
        poff.data_ptr(), ids.data_ptr(), K, iou.data_ptr(), None, None, torch.get_num_threads()),
        "sonet_seg_iou_ragged_cpu_f32")
    return iou.numpy()


def visualize_pc_seg(score, seg, label, visualizer, opt, input_pc, batch_num):
    """Show one cloud coloured by predicted and by ground-truth part (models/losses.py:46-70):
    score [C,N], seg [N], input_pc [3,N]; colours from <opt.dataroot>/part_color_mapping.json
    (RGB in [0,1], scaled to int 0..255); ground-truth part 49 is drawn as (1,1,1). label and
    batch_num are unused, as in the reference."""
    xyz = input_pc.detach().cpu().numpy().transpose()                        # N x 3
    predicted = torch.max(score.detach().cpu(), dim=0)[1].numpy()
    gt = seg.detach().cpu().numpy()
    with open(os.path.join(opt.dataroot, "part_color_mapping.json")) as f:
        colors = np.fabs(np.asarray(json.load(f)) * 255).astype(int)
    gt_colors = colors[gt]
    gt_colors[gt == 49] = 1
    visualizer.display_current_results(OrderedDict([("pc_colored_predicted", [xyz, colors[predicted]]),
                                                    ("pc_colored_gt", [xyz, gt_colors])]), 1, 1)


class PartSegIoU:
    """Part-segmentation metrics over an evaluation loop, without a host sync per batch.

        meter = PartSegIoU()
        for batch in loader:
            ...; meter.update(model.score_segmenter, model.input_seg, model.input_label)
        r = meter.compute()

    update() runs the seg_iou kernel (the host entry for CPU tensors) and keeps the per-shape IoUs,
    categories and correct-point counts on the scores' device. compute() copies them once and
    returns, all computed in float64 numpy in a fixed order (the same batches in the same order give
    the same bits):
      instance_miou  mean IoU over all shapes (what part-seg/train.py accumulates in test_iou)
      category_miou  {category: mean IoU of its shapes} for every category seen
      class_miou     mean of category_miou over the categories seen, in ascending order
      accuracy       correct points / all points
    table: category -> part ids (default: the 16 ShapeNetPart categories)."""

    def __init__(self, table=None):
        self.table = table
        self.reset()

    def reset(self):
        self._iou, self._label, self._correct = [], [], []
        self._points = 0

    def update(self, score, seg, label):
        iou, correct = _seg_iou(score, seg, label, self.table, want_correct=True)
        self._iou.append(iou)
        self._label.append(label.detach().to(iou.device, torch.int64, copy=True))
        self._correct.append(correct)
        self._points += seg.numel()

    def compute(self):
        if not self._iou:
            raise RuntimeError("PartSegIoU.compute() before any update()")
        iou = _host_iou(torch.cat(self._iou))
        label = torch.cat(self._label).cpu().numpy()
        correct = torch.cat(self._correct).cpu().numpy().astype(np.int64)
        cats = np.unique(label)
        per_cat = OrderedDict((int(c), iou[label == c].mean()) for c in cats)
        return dict(instance_miou=iou.mean(), category_miou=per_cat,
                    class_miou=np.asarray(list(per_cat.values())).mean(),
                    accuracy=correct.sum() / float(self._points))
