"""Encoder / Classifier / Segmenter / Decoder with the reference's API (models/networks.py:20-462):
same constructor (`opt` namespace), same forward signatures, same cached attributes, same
state_dict keys — so reference checkpoints load and models/{classifier,segmenter,autoencoder}.py
call these unchanged.

Eval/no-grad forward = the H100 hot path: SOM assignment, cluster statistics, decentring, the
point-wise MLPs, the per-node arg-max pool, node kNN grouping and the heads all run as
hand-written sm_90a kernels (libsonet_b200). Compared with the reference dataflow
(models/networks.py:111-199) the dense one-hot mask [B,kN,M] and the two [B,3,kN,M] products are
never built: statistics and centres come straight from the assignment indices; `mask`, `centers`
remain available as lazily materialised attributes for callers that read them
(models/segmenter.py:90).
"""
import math

import numpy as np
import torch
import torch.nn as nn

from . import augmentation, ops, som, train_ops
from .layers import (EquivariantLayer, KNNModule, MyConv2d, MyLinear, PointNet, PointResNet,
                     UpConv, _Cache, _fast_ok, tc_enabled, tc_f16)


def _bn_kwargs(opt):
    return dict(momentum=opt.bn_momentum, bn_momentum_decay_step=opt.bn_momentum_decay_step,
                bn_momentum_decay=opt.bn_momentum_decay)


class Transformer(nn.Module):
    """Rotation regressor (models/networks.py:20-68). Its call is commented out in the reference
    encoder (networks.py:147-164); the sub-module exists so that encoder state_dicts match."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        act, norm, bn = opt.activation, opt.normalization, _bn_kwargs(opt)
        self.first_pointnet = PointNet(3, (32, 64, 128), activation=act, normalization=norm, **bn)
        self.second_pointnet = PointNet(128 + 128, (256, 256), activation=act, normalization=norm,
                                        **bn)
        self.fc1 = MyLinear(256, 128, activation=act, normalization=norm, **bn)
        self.fc2 = MyLinear(128, 64, activation=act, normalization=norm, **bn)
        self.fc3 = MyLinear(64, 1, activation=None, normalization=None)
        self.dropout1 = nn.Dropout(p=opt.dropout)
        self.dropout2 = nn.Dropout(p=opt.dropout)

    def forward(self, x, sn=None, epoch=None):
        first_pn_out = self.first_pointnet(x, epoch)
        feature_1, _ = torch.max(first_pn_out, dim=2, keepdim=False)
        second_pn_out = self.second_pointnet(
            torch.cat((first_pn_out, feature_1.unsqueeze(2).expand_as(first_pn_out)), dim=1), epoch)
        feature_2, _ = torch.max(second_pn_out, dim=2, keepdim=False)
        fc1_out = self.fc1(feature_2, epoch)
        if self.opt.dropout > 0.1:
            fc1_out = self.dropout1(fc1_out)
        self.fc2_out = self.fc2(fc1_out, epoch)
        if self.opt.dropout > 0.1:
            self.fc2_out = self.dropout2(self.fc2_out)
        return torch.tanh(self.fc3(self.fc2_out, epoch))


class Encoder(nn.Module):
    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.feature_num = opt.feature_num
        act, norm, bn = opt.activation, opt.normalization, _bn_kwargs(opt)

        self.transformer = Transformer(opt)
        in_ch = 6 if self.opt.surface_normal == True else 3  # noqa: E712 (reference semantics)
        self.first_pointnet = PointResNet(in_ch, [64, 128, 256, 384], activation=act,
                                          normalization=norm, **bn)
        if self.opt.som_k >= 2:
            self.knnlayer = KNNModule(3 + 384, (512, 512), activation=act, normalization=norm, **bn)
            self.final_pointnet = PointNet(3 + 512, (768, self.feature_num), activation=act,
                                           normalization=norm, **bn)
        else:
            self.final_pointnet = PointResNet(3 + 384, (512, 512, 768, self.feature_num),
                                              activation=act, normalization=norm, **bn)

        rows = int(math.sqrt(self.opt.node_num))
        self.som_builder = som.BatchSOM(rows, rows, 3, self.opt.gpu_id, self.opt.batch_size)
        self.zero_pad = torch.nn.ZeroPad2d(padding=1)

        self._assign = None
        self._mask = None
        self._centers = None
        self._x_aug = None
        self._first_pn_out = None
        self._lazy_src = None
        # True (default): when first_pn_out itself is not needed, fuse the per-node max into the
        # wgmma PointResNet and never write it. Callers that read encoder.first_pn_out every
        # forward (the segmenter) set this to False to avoid the lazy recomputation.
        self.fuse_pool = True
        self._fpo_demand = False     # set once a caller has read first_pn_out lazily (see below)
        self._pool_keys = ops.PoolKeys()
        self._ragged_keys = ops.PoolKeys()   # forward_ragged's own: the graphed forward's stay put

    # ---- lazily materialised public attributes (API of models/networks.py:127, 169) -----------
    @property
    def mask(self):
        """[B,kN,M] int32 one-hot assignment (util/som.py:255-265)."""
        if self._mask is None and self._assign is not None:
            self._mask = ops.som_mask(self._assign["min_idx_i32"], self.som_node.shape[2])
        return self._mask

    @property
    def centers(self):
        """[B,3,kN] centre of each stacked point copy (models/networks.py:168-169)."""
        if self._centers is None and self._assign is not None:
            self._centers = ops.gather_points(self.som_node.detach().contiguous(),
                                              self._assign["min_idx_i32"])
        return self._centers

    def _materialise_x_aug(self):
        if self._x_aug is None and self._lazy_src is not None:
            xd, snd, idx32, k, _ = self._lazy_src
            self._x_aug, _ = ops.som_decenter(xd, snd, self.som_node.detach(), idx32, k)
        return self._x_aug

    @property
    def x_decentered(self):
        """[B,3,kN] stacked points minus their node centre (models/networks.py:171)."""
        xa = self._materialise_x_aug()
        return None if xa is None else xa[:, 0:3, :]

    @property
    def first_pn_out(self):
        """[B,384,kN] output of the first PointResNet (models/networks.py:176). On the fused
        path it is only computed when somebody reads it."""
        if self._first_pn_out is None and self._lazy_src is not None:
            # a caller that reads first_pn_out after a fused forward (the reference's unmodified
            # models/segmenter.py:100-105 does, every forward) pays one recomputation; from the
            # next forward on the encoder keeps the unfused path for it
            self._fpo_demand = True
            with torch.no_grad():
                self._first_pn_out = self.first_pointnet(self._materialise_x_aug(),
                                                         self._lazy_src[4])
        return self._first_pn_out

    @property
    def min_idx(self):
        """[B,kN] int32 node index of each stacked point copy (slot-major)."""
        return None if self._assign is None else self._assign["min_idx_i32"]

    def forward(self, x, sn, node, node_knn_I, is_train=False, epoch=None):
        """x, sn [B,3,N]; node [B,3,M]; node_knn_I [B,M,som_k] int64 -> feature [B,feature_num]."""
        if not x.is_cuda:
            raise RuntimeError("sonet_b200.Encoder runs on CUDA tensors only (no CPU fallback)")
        opt = self.opt
        k = opt.k
        M = node.size()[2]
        use_sn = opt.surface_normal == True  # noqa: E712
        fast = _fast_ok(self, x, sn if use_sn else x)    # eval mode, no input gradient

        # SOM nodes come from the loader (models/networks.py:123-124)
        self.som_builder.node = node.detach().to(torch.float32).contiguous()

        # assignment + cluster statistics (networks.py:127-143) — always the CUDA kernels: the
        # reference computes these on .data (no gradient flows through them)
        xd = x.detach().contiguous()
        snd = sn.detach().contiguous() if use_sn else None
        fpn = self.first_pointnet
        fused = (fast and self.fuse_pool and not self._fpo_demand and M <= 256
                 and fpn.layers[0].fast(xd)
                 and fpn._tc_eligible(6 if use_sn else 3, None))
        group = fused and ops.som_group_fits(xd.shape[2], M, k, xd.device)
        a = ops.som_assign(xd, self.som_builder.node, k, want_stats=not group)
        idx32, mask_row_max = a["min_idx_i32"], a["row_max"]
        if group:
            # statistics + stable node sort + decentring in one launch
            xs, ns, p0, a["count"], a["cluster_mean"] = ops.som_group_decenter(xd, snd, idx32, M, k)
        self._assign, self._mask, self._centers = a, None, None
        self.som_builder.node = a["cluster_mean"]
        self.som_node = self.som_builder.node

        self._lazy_src = (xd, snd, idx32, k, epoch)
        self._x_aug, self._first_pn_out = None, None
        pooled = None
        if fused:
            # fused path: node-sorted copies -> wgmma PointResNet -> per-node max. Neither
            # x_augmented nor first_pn_out [B,384,kN] is materialised (they stay available as
            # lazily recomputed attributes for callers that read them).
            if not group:
                xs, ns, p0 = ops.som_sort_decenter(xd, snd, self.som_node, idx32, a["count"], k)
            blob, fpar = fpn._tc_params()
            pooled = ops.pointresnet_tc_pool(xs, blob, fpar, ns, p0, M, finalize=False,
                                             owner=self._pool_keys, f16=tc_f16(),
                                             act=fpn.layers[0].activation)
            done = None
            if opt.som_k >= 2:   # pool_finalize folds into the KNN module's input assembly
                done = self.knnlayer.forward_pooled(self.som_node, pooled, node_knn_I, opt.som_k,
                                                    opt.som_k_type, epoch, owner=self._pool_keys)
            if done is None:
                self.first_pn_out_masked_max = ops.pool_finalize(*pooled, owner=self._pool_keys)
                pooled = None
            else:
                self.knn_center_1, self.knn_feature_1, self.first_pn_out_masked_max = done
        elif fast:
            x_aug, _ = ops.som_decenter(xd, snd, self.som_node, idx32, k)
            self._x_aug = x_aug
            self._first_pn_out = self.first_pointnet(x_aug, epoch)
            _, self.first_pn_out_masked_max = ops.index_max(self._first_pn_out, idx32, M,
                                                            with_values=True)
        else:
            # differentiable composition (training): same math with gathers instead of the
            # dense mask products
            idx64 = idx32.long()
            centers = torch.gather(self.som_node, 2, idx64.unsqueeze(1).expand(-1, 3, -1))
            self._centers = centers.detach()
            x_stack = torch.cat((x,) * k, dim=2)
            x_dec = (x_stack - self._centers).detach()
            x_in = torch.cat((x_dec, torch.cat((sn,) * k, dim=2)), dim=1) if use_sn else x_dec
            self._x_aug = x_in
            self._first_pn_out = self.first_pointnet(x_in, epoch)
            if train_ops.ENABLED:
                # arg-max kernel forward (values fused) + deterministic scatter backward
                self.first_pn_out_masked_max = train_ops.IndexMaxGather.apply(
                    self._first_pn_out, idx32, M)
            else:
                gather_index = ops.index_max(self._first_pn_out.detach().contiguous(), idx32,
                                             M).long()
                self.first_pn_out_masked_max = self._first_pn_out.gather(
                    dim=2, index=gather_index * mask_row_max.unsqueeze(1).long())

        if opt.som_k >= 2:
            if pooled is None:
                self.knn_center_1, self.knn_feature_1 = self.knnlayer(
                    self.som_node, self.first_pn_out_masked_max, node_knn_I, opt.som_k,
                    opt.som_k_type, epoch)
            self.final_pn_out = self.final_pointnet.forward_pair(self.knn_center_1,
                                                                 self.knn_feature_1, epoch)
        else:
            # som_k < 2 (shrec16/options.py:40): PointResNet on cat(som_node, masked_max)
            self.final_pn_out = self.final_pointnet(self.som_node, epoch,
                                                    x1=self.first_pn_out_masked_max)

        if fast:
            self.feature = ops.rowmax(self.final_pn_out)
        else:
            self.feature, _ = torch.max(self.final_pn_out, dim=2, keepdim=False)
        return self.feature

    # ---- whole clouds of any size ------------------------------------------------------------
    # device bytes per stacked copy of a point in one chunk: the decentred copy, its node ids and
    # the unfused route's four layer outputs
    _RAGGED_COPY_BYTES = 4 * (6 + 2 + 64 + 128 + 256 + 384)
    # som_group_decenter_ragged packs a chunk's point index into 24 bits
    _RAGGED_MAX_POINTS = (1 << 24) - 1

    def check_ragged(self, points, offsets, node, node_knn_I=None, chunk_points=None,
                     what="forward_ragged", train=False):
        """The refusals of forward_ragged (RuntimeError; ValueError for an empty cloud), raised
        before any launch; with train, those of forward_ragged_train instead: the same but for the
        train-mode refusal, plus k*T >= 2^31 stacked columns, train_ops.ENABLED off, an installed
        DataParallelTraining and a random point dropout. Returns the offsets as a host numpy
        array."""
        opt = self.opt
        if train:
            if not train_ops.ENABLED:
                raise RuntimeError("%s: the train kernels are off (train_ops.ENABLED = False)" % what)
            if train_ops.EXCHANGE is not None:
                raise RuntimeError("%s: a DataParallelTraining is installed; ragged batches train in "
                                   "one process" % what)
            if opt.random_pc_dropout_lower_limit < 0.99:
                raise RuntimeError("%s: random point dropout (random_pc_dropout_lower_limit=%s) is not "
                                   "applied to whole clouds" % (what, opt.random_pc_dropout_lower_limit))
        elif self.training:
            raise RuntimeError("%s: the encoder is in train mode; call eval() first" % what)
        if opt.normalization == 'instance':
            raise RuntimeError("%s: --normalization instance has no ragged per-cloud statistics"
                               % what)
        if not all(l._fast_eligible() for l in self.first_pointnet.layers):
            raise RuntimeError("%s: activation %r / normalization %r have no kernels"
                               % (what, opt.activation, opt.normalization))
        dev = self.first_pointnet.layers[0].conv.weight.device
        if not (1 <= opt.k <= 4):
            raise RuntimeError("%s: k=%d outside [1, 4]" % (what, opt.k))
        for name, t, dt, dim in (("points", points, torch.float32, 2), ("node", node, torch.float32, 3),
                                 ("offsets", offsets, torch.int64, 1),
                                 ("node_knn_I", node_knn_I, torch.int64, 3)):
            if t is None and name == "node_knn_I":
                continue
            if not isinstance(t, torch.Tensor) or t.dtype != dt or t.dim() != dim:
                raise RuntimeError("%s: %s must be a %d-D %s tensor (got %s)" % (
                    what, name, dim, dt, (t.dtype, tuple(t.shape)) if isinstance(t, torch.Tensor)
                    else type(t).__name__))
            if t.device != dev:
                raise RuntimeError("%s: %s must be on the model's device %s (got %s)"
                                   % (what, name, dev, t.device))
        if points.shape[1] != 6:
            raise RuntimeError("%s: points must be [T, 6] (got %s)" % (what, tuple(points.shape)))
        B, M = node.shape[0], node.shape[2]
        if node.shape[1] != 3 or B < 1:
            raise RuntimeError("%s: node must be [B, 3, M] (got %s)" % (what, tuple(node.shape)))
        if not (opt.k <= M <= 256):
            raise RuntimeError("%s: M=%d nodes outside [k=%d, 256]" % (what, M, opt.k))
        if node_knn_I is not None and (node_knn_I.shape[:2] != (B, M)
                                       or node_knn_I.shape[2] < max(opt.som_k, 1)):
            raise RuntimeError("%s: node_knn_I must be [%d, %d, >=%d] (got %s)"
                               % (what, B, M, max(opt.som_k, 1), tuple(node_knn_I.shape)))
        if chunk_points is not None and int(chunk_points) < 1:
            raise RuntimeError("%s: chunk_points must be >= 1 (got %s)" % (what, chunk_points))
        off = ops.ragged_offsets(offsets, points.shape[0], B)
        counts = np.diff(off)
        if (counts == 0).any():
            raise ValueError("%s: cloud %d has no points" % (what, int(np.flatnonzero(counts == 0)[0])))
        if counts.max() > self._RAGGED_MAX_POINTS:
            raise RuntimeError("%s: cloud %d has %d points, more than %d"
                               % (what, int(counts.argmax()), int(counts.max()),
                                  self._RAGGED_MAX_POINTS))
        if train and opt.k * points.shape[0] >= (1 << 31):
            raise RuntimeError("%s: k*T = %d stacked columns, 2^31 or more"
                               % (what, opt.k * points.shape[0]))
        return off

    def forward_ragged_train(self, points, offsets, node, node_knn_I, epoch=None):
        """The global feature [B,feature_num] of every cloud of a ragged batch from ALL of its points,
        in train mode and differentiable w.r.t. the encoder's parameters (classifier.Model.
        optimize_clouds). Inputs as forward_ragged; node_knn_I None: computed (augmentation.som_knn).

        The ragged SOM assignment and the group route's cluster means (forward_ragged's, the whole
        cloud's), the decentred copies x_aug [1,Cin,k*T] (detached, as in forward()), the first
        PointResNet on the train kernels with cols = k*offsets, so that its BatchNorm statistics
        cover every stacked copy of the batch (a cloud weighs its size), the per-cloud per-node max
        (IndexMaxGatherRagged), then forward()'s train-mode node-level stage on [B,.,M]. No chunks:
        BatchNorm needs the whole batch. Writes no encoder attribute; the BatchNorm running
        statistics are updated as in a train step (with n = k*T in the first PointResNet).
        Refused before any launch: eval mode and check_ragged(train=True)'s cases."""
        if not self.training:
            raise RuntimeError("forward_ragged_train: the encoder is in eval mode; call train() first")
        self.check_ragged(points, offsets, node, node_knn_I, what="forward_ragged_train", train=True)
        opt = self.opt
        k, M = opt.k, node.shape[2]
        use_sn = opt.surface_normal == True  # noqa: E712
        points = points.detach().contiguous()
        node = node.detach().contiguous()
        with torch.no_grad():
            if node_knn_I is None:
                node_knn_I = augmentation.som_knn(node, opt.som_k, M)
            idx, _, _ = ops.som_assign_ragged(points, offsets, node, k)
            _, _, _, som_node = ops.som_group_decenter_ragged(points, offsets, idx, M, k, use_sn)
            x_aug = ops.som_decenter_ragged(points, offsets, idx, som_node, k, use_sn)
            cols = offsets * k
        fpo = self.first_pointnet(x_aug, epoch, cols=cols)
        masked_max = train_ops.IndexMaxGatherRagged.apply(fpo, idx, offsets, cols, M, k)
        if opt.som_k >= 2:
            center, knn_feature = self.knnlayer(som_node, masked_max, node_knn_I, opt.som_k,
                                                opt.som_k_type, epoch)
            final = self.final_pointnet.forward_pair(center, knn_feature, epoch)
        else:
            final = self.final_pointnet(som_node, epoch, x1=masked_max)
        feature, _ = torch.max(final, dim=2, keepdim=False)
        return feature

    def forward_ragged(self, points, offsets, node, node_knn_I, chunk_points=None,
                       return_nodes=False):
        """The global feature of every cloud of a ragged batch from ALL of its points, in eval mode.

        points [T,6] f32 on the model's device (xyz | normal, DeviceDataset.data's layout; the
        normals are ignored unless surface_normal), offsets [B+1] int64 (cloud b is rows
        offsets[b] .. offsets[b+1], P_b points), node [B,3,M] the loader's SOM nodes, node_knn_I
        [B,M,som_k] int64. Returns feature [B,feature_num]; with return_nodes also a dict of
        som_node, first_pn_out_masked_max, knn_center_1, knn_feature_1 (None when som_k < 2) and
        final_pn_out, each [B,.,M].

        Cloud b is the dense forward at N = P_b: its k stacked copies in the reference's x_stack
        order, assigned with sonet_som_assign's arithmetic, cluster means summed in the group
        route's order, the first PointResNet and index_max's per-node max (> -1000, else the cloud's
        copy 0). From the pooled features on, the node-level stage runs on [B,.,M] as in forward().
        Routes: the first PointResNet's from the batch's k*T columns, the node-level stage's from
        its B*M rows. A cloud's results depend only on its own points and nodes and those routes:
        permuting the clouds permutes the outputs bit for bit, and chunk_points (default: from the
        free device memory) changes no bit, since chunks are whole clouds.

        The encoder attributes of the last forward() (som_node, feature, ...) are left untouched.
        Refused before any launch: check_ragged."""
        off = self.check_ragged(points, offsets, node, node_knn_I, chunk_points)
        opt, fpn = self.opt, self.first_pointnet
        k, M, T = opt.k, node.shape[2], points.shape[0]
        use_sn = opt.surface_normal == True  # noqa: E712
        fused = fpn._tc_eligible(6 if use_sn else 3, None)
        if chunk_points:
            chunk = int(chunk_points)
        else:
            free, _ = torch.cuda.mem_get_info(points.device)
            chunk = (free // 4) // (k * self._RAGGED_COPY_BYTES)
        chunk = max(1, min(chunk, self._RAGGED_MAX_POINTS))
        with torch.no_grad():
            points = points.contiguous()
            node = node.detach().contiguous()
            cms, mms = [], []
            for b0, b1 in _ragged_chunks(off, chunk):
                o0 = int(off[b0])
                pts = points[o0:int(off[b1])]
                offc = (offsets[b0:b1 + 1] - o0).contiguous()
                idx, _, _ = ops.som_assign_ragged(pts, offc, node[b0:b1], k)
                xs, ns, p0s, cm = ops.som_group_decenter_ragged(pts, offc, idx, M, k, use_sn)
                if fused:
                    blob, fpar = fpn._tc_params()
                    pooled = ops.pointresnet_tc_pool_ragged(xs, blob, fpar, ns, p0s, M,
                                                            owner=self._ragged_keys, f16=tc_f16(),
                                                            act=fpn.layers[0].activation)
                    mm = ops.pool_finalize(*pooled, owner=self._ragged_keys)
                else:
                    x_aug = ops.som_decenter_ragged(pts, offc, idx, cm, k, use_sn)
                    fpo = fpn(x_aug, route_rows=k * T)
                    _, mm = ops.index_max_ragged(fpo[0], idx, offc, M, k)
                cms.append(cm)
                mms.append(mm)
            som_node = cms[0] if len(cms) == 1 else torch.cat(cms)
            masked_max = mms[0] if len(mms) == 1 else torch.cat(mms)
            center = knn_feature = None
            if opt.som_k >= 2:
                center, knn_feature = self.knnlayer(som_node, masked_max, node_knn_I, opt.som_k,
                                                    opt.som_k_type)
                final = self.final_pointnet.forward_pair(center, knn_feature)
            else:
                final = self.final_pointnet(som_node, x1=masked_max)
            feature = ops.rowmax(final)
        if not return_nodes:
            return feature
        return feature, dict(som_node=som_node, first_pn_out_masked_max=masked_max,
                             knn_center_1=center, knn_feature_1=knn_feature, final_pn_out=final)


def _ragged_chunks(off, chunk):
    """(b0, b1) runs of whole clouds of the host offsets `off` with at most `chunk` points each;
    a larger cloud is a run of its own."""
    B, b0 = len(off) - 1, 0
    while b0 < B:
        b1 = b0 + 1
        while b1 < B and off[b1 + 1] - off[b0] <= chunk:
            b1 += 1
        yield b0, b1
        b0 = b1


class Classifier(nn.Module):
    """FC 1024 -> 512 -> 256 -> classes (models/networks.py:202-227)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.feature_num = opt.feature_num
        act, norm, bn = opt.activation, opt.normalization, _bn_kwargs(opt)
        self.fc1 = MyLinear(self.feature_num, 512, activation=act, normalization=norm, **bn)
        self.fc2 = MyLinear(512, 256, activation=act, normalization=norm, **bn)
        self.fc3 = MyLinear(256, self.opt.classes, activation=None, normalization=None)
        self.dropout1 = nn.Dropout(p=self.opt.dropout)
        self.dropout2 = nn.Dropout(p=self.opt.dropout)

    def forward(self, feature, epoch=None, store=True):
        """store=False: leave the fc2_out attribute alone (classifier.Model.optimize_clouds)."""
        fc1_out = self.fc1(feature, epoch)
        if self.opt.dropout > 0.1:
            fc1_out = self.dropout1(fc1_out)
        fc2_out = self.fc2(fc1_out, epoch)
        if self.opt.dropout > 0.1:
            fc2_out = self.dropout2(fc2_out)
        if store:
            self.fc2_out = fc2_out
        return self.fc3(fc2_out, epoch)


class Segmenter(nn.Module):
    """Per-point segmentation head (models/networks.py:230-344)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.feature_num = opt.feature_num
        base = (12 if self.opt.surface_normal == True else 9) + 16 + 384 + 384  # noqa: E712
        in_channels = base + (512 if self.opt.som_k >= 2 else 0) + self.feature_num * 2
        act, norm = self.opt.activation, self.opt.normalization
        self.layer1 = EquivariantLayer(in_channels, 1024, activation=act, normalization=norm)
        self.layer2 = EquivariantLayer(1024, 512, activation=act, normalization=norm)
        self.layer3 = EquivariantLayer(512, 256, activation=act, normalization=norm)
        self.drop3 = nn.Dropout(p=self.opt.dropout)
        self.layer4 = EquivariantLayer(256, 128, activation=act, normalization=norm)
        self.drop4 = nn.Dropout(p=self.opt.dropout)
        self.layer5 = EquivariantLayer(128, self.opt.classes, activation=None, normalization=None)
        self._l1 = _Cache()

    def _onehot(self, label, B, device):
        onehot = torch.zeros(B, 16, dtype=torch.float32, device=device)
        onehot.scatter_(1, label.unsqueeze(1), 1)
        return onehot

    def _tail(self, layer2_out, k, N, route_rows=None):
        """layer3 + k-copy average + layer4/5 (models/networks.py:326-341). An instance-norm
        layer 3 takes the k-copy mean inside its normalisation pass. route_rows: the point count
        B*N whose routes layers 3-5 take (forward_rows), None for this launch's own."""
        if (self.layer3.normalization == 'instance' and k in (2, 3) and layer2_out.dim() == 3
                and self.layer3.fast(layer2_out) and self.layer4.fast(layer2_out)):
            return self._tail_avg(self.layer3.forward_points(layer2_out.contiguous(), kcopy=k))
        layer3_out = self.layer3(layer2_out,
                                 route_rows=None if route_rows is None else k * route_rows)
        fast = self.layer4.fast(layer3_out)
        if fast and k in (2, 3):
            avg = ops.kcopy_mean(layer3_out.contiguous(), k)
        else:
            parts = torch.split(layer3_out, N, dim=2)
            assert len(parts) == k
            if k == 1:     # one copy per point: its own layer-3 output
                avg = parts[0]
            elif k == 2:
                avg = 0.5 * (parts[0] + parts[1])
            elif k == 3:
                avg = (1.0 / 3.0) * (parts[0] + parts[1] + parts[2])
        return self._tail_avg(avg, route_rows)

    def _tail_avg(self, avg, route_rows=None):
        out4 = self.layer4(avg, route_rows=route_rows)
        if self.opt.dropout > 0.1:
            out4 = self.drop4(out4)
        return self.layer5(out4, route_rows=route_rows)

    def forward(self, x_decentered, x, centers, sn, label, first_pn_out, feature_max_first_pn_out,
                feature_max_knn_feature_1, feature_max_final_pn_out, feature):
        """Reference signature: per-point tensors already gathered by the caller
        (models/segmenter.py:90-98). The 3356-channel concat is materialised as in the reference,
        the five layers run on the point-wise kernel."""
        B, N = x.size()[0], x.size()[2]
        k = self.opt.k
        kN = round(k * N)
        x_st = torch.cat((x,) * k, dim=2)
        parts = [x_decentered, x_st, centers]
        if self.opt.surface_normal == True:  # noqa: E712
            parts.append(torch.cat((sn,) * k, dim=2))
        parts.append(self._onehot(label, B, x.device).unsqueeze(2).expand(B, 16, kN).detach())
        parts += [first_pn_out, feature_max_first_pn_out]
        if self.opt.som_k >= 2:
            parts.append(feature_max_knn_feature_1)
        parts += [feature_max_final_pn_out, feature.unsqueeze(2).expand(B, self.feature_num, kN)]
        layer1_in = torch.cat(parts, dim=1)
        return self._tail(self.layer2(self.layer1(layer1_in)), k, self.opt.input_pc_num)

    # ---- fast entry: node-level features + assignment, no per-point gathers ----------------
    def _zero_idx(self, B, M, dev):
        z = getattr(self, "_zidx", None)
        if z is None or z.shape != (B, M) or z.device != dev:
            z = self._zidx = torch.zeros((B, M), dtype=torch.int32, device=dev)
        return z

    def _pack_layer1(self, n_pt_a, n_onehot, n_pp, n_node):
        """Split the folded layer-1 weight (transposed [Cin,1024]) by input-channel role."""
        w, shift = self.layer1.folded(transpose=True)

        def build():
            o0 = n_pt_a
            o1 = o0 + n_onehot
            o2 = o1 + n_pp
            o3 = o2 + n_node
            w_point = torch.cat((w[0:o0], w[o1:o2]), dim=0).contiguous()     # coords | first_pn_out
            w_node = w[o2:o3].contiguous()                                    # node-level features
            # per-cloud inputs (one-hot label | global feature): a [B,1040]x[1040,1024] fp32 GEMM
            # whose result enters the node-level GEMM as a broadcast addend
            w_cloud = torch.cat((w[o0:o1], w[o3:]), dim=0).t().contiguous()   # [1024, 1040]
            bp, ip = ops.pointwise_tc_pack(w_point.t().contiguous())
            # node-level GEMM: one launch of the grouped entry (K split to fill the SMs)
            bn, pern, inn = ops.pointwise_tc_pack_groups(w_node.t().contiguous().unsqueeze(0))
            tc = (bp.to(w.device), ip, bn.to(w.device), pern, inn)
            return w_point, w_node, w_cloud, tc, shift
        return self._l1.get((self.layer1._folded.version, n_pt_a, n_onehot, n_pp, n_node), build)

    def forward_nodes(self, x_decentered, x, centers, sn, label, first_pn_out, node_first, node_knn,
                      node_final, feature, min_idx_i32):
        """Same result as forward(), given the node-level features [B,C,M] and the point->node
        assignment min_idx_i32 [B,kN] instead of per-point gathered copies.

        Layer 1 is split algebraically (SURVEY.md §8a-10): of its 3356 input channels only 396
        vary per point; 1920 vary per node and 1040 per cloud. The cloud part is one [B,1040] fp32
        GEMM, broadcast-added inside the node-level GEMM over the M nodes, whose result is in turn
        gathered per point inside the epilogue of the per-point GEMM — 6.85 instead of 25.2 GFLOP per cloud, and the [B,3356,kN] concat
        (1.3 GB at B=32,N=1024) is never written.
        """
        if not (self.layer1.fast(first_pn_out) and self.opt.som_k >= 2):
            if self.layer1.fast(node_first, node_final):
                g = lambda t: ops.gather_points(t.contiguous(), min_idx_i32)  # noqa: E731
            else:
                # training / grad mode: torch.gather as in models/segmenter.py:96-98, so that the
                # encoder receives gradient through the three node-level feature maps
                i64 = min_idx_i32.long().unsqueeze(1)
                g = lambda t: torch.gather(t, 2, i64.expand(-1, t.shape[1], -1))  # noqa: E731
            return self.forward(x_decentered, x, centers, sn, label, first_pn_out, g(node_first),
                                g(node_knn), g(node_final), feature)
        B, N = x.size()[0], x.size()[2]
        k = self.opt.k
        use_sn = self.opt.surface_normal == True  # noqa: E712
        small = [x_decentered, torch.cat((x,) * k, dim=2), centers]
        if use_sn:
            small.append(torch.cat((sn,) * k, dim=2))
        pt = torch.cat(small, dim=1).contiguous()                       # [B,12,kN]
        addend, packed = self._node_addend(pt.shape[1], first_pn_out.shape[1], node_first,
                                           node_knn, node_final, feature, label)
        out1 = self._layer1_points(pt, first_pn_out, addend, min_idx_i32, packed)
        if self.layer1.normalization == 'instance':
            out1 = self.layer1.instance_norm(out1)
        return self._tail(self.layer2(out1), k, N)

    def _node_addend(self, n_pt, n_pp, node_first, node_knn, node_final, feature, label,
                     zero_idx=None):
        """(addend, packed): layer 1's node- and cloud-level part [B,1024,M] (the node GEMM over
        cat(node_first, node_knn, node_final) plus the broadcast [B,1040] cloud GEMM) and the
        packed split weights for _layer1_points. zero_idx: the fp32 route's zero [B,M] int32
        gather index, or None for the module's cached one (a caller that must not rebind the cache
        a captured graph reads passes its own)."""
        B, M = node_first.shape[0], node_first.shape[2]
        packed = self._pack_layer1(
            n_pt, 16, n_pp, node_first.shape[1] + node_knn.shape[1] + node_final.shape[1])
        w_point, w_node, w_cloud, tc, shift = packed
        cloud = torch.cat((self._onehot(label, B, feature.device), feature), dim=1)   # [B,1040]
        cloud_add = ops.linear(cloud.contiguous(), w_cloud, None, None, False).unsqueeze(2)  # [B,1024,1]
        if tc_enabled():
            bp, ip, bn, pern, inn = tc
            cout = w_point.shape[1]
            # [B,1920,M] -> [B,1024,M]: 16 row tiles x 4 column tiles would leave the GPU to 64
            # CTAs that each walk all 30 K chunks; the K split brings it to one wave
            node_in = torch.cat((node_first, node_knn, node_final), dim=1).contiguous()
            kch = (node_in.shape[1] + 63) // 64
            splits = ops.pick_splits(kch, ((B * M + 127) // 128) * ((cout + 255) // 256))
            addend = ops.pointwise_tc_grouped(node_in, bn, pern, inn, None, cout, False, groups=1,
                                              splits=splits, f16=tc_f16()) + cloud_add
            return addend, packed
        node_a = torch.cat((node_first, node_knn), dim=1).contiguous()
        addend = ops.pointwise_layer(node_a, w_node, None, None, False, x1=node_final.contiguous(),
                                     addend=cloud_add,
                                    gidx=self._zero_idx(B, M, feature.device) if zero_idx is None
                                    else zero_idx)
        return addend, packed

    def _layer1_points(self, pt, first_pn_out, addend, gidx, packed):
        """Layer 1 over per-point rows pt [B',12,P] | first_pn_out [B',384,P], the node-level
        addend gathered per column by gidx [B',P] (the split GEMM of forward_nodes); pre-norm z for
        an instance-norm layer 1."""
        w_point, _, _, tc, shift = packed
        # the split is linear up to the pre-norm z: an instance-norm layer 1 normalises it after
        act1 = None if self.layer1.normalization == 'instance' else self.layer1.activation
        if tc_enabled():
            bp, ip = tc[0], tc[1]
            return ops.pointwise_layer_tc(pt, bp, ip, shift, w_point.shape[1], act1,
                                          x1=first_pn_out.contiguous(), addend=addend, gidx=gidx,
                                          f16=tc_f16())
        return ops.pointwise_layer(pt, w_point, None, shift, act1, x1=first_pn_out.contiguous(),
                                   addend=addend, gidx=gidx)

    def forward_rows(self, pt, first_pn_out, addend_flat, gidx, k, packed, route_rows):
        """The per-point head over one chunk of ragged rows laid out as ONE batch row, copy-major
        (csrc/seg_points.cu): pt [1,12,k*R], first_pn_out [1,384,k*R], gidx [1,k*R] flat
        cloud*M+node ids into addend_flat [1,1024,B*M] (_node_addend's [B,1024,M] with the clouds
        side by side; packed: its second value) -> scores [1,classes,R]. Every layer is a
        per-column GEMM, so a row's scores do not depend on the other rows of the chunk.
        route_rows: the B*N points of the sampled forward. Each layer takes the kernel that
        forward_nodes took for them (layers 2-3 over k*B*N columns, 4-5 over B*N), whatever the
        chunk's size, so that a point's scores keep the sampled forward's bits."""
        out1 = self._layer1_points(pt, first_pn_out, addend_flat, gidx, packed)
        out2 = self.layer2(out1, route_rows=k * route_rows)
        return self._tail(out2, k, pt.shape[2] // k, route_rows=route_rows)


class DecoderLinear(nn.Module):
    """FC decoder branch (models/networks.py:347-369)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.feature_num = opt.feature_num
        self.output_point_number = opt.output_fc_pc_num
        n, act, norm = self.output_point_number, opt.activation, opt.normalization
        self.linear1 = MyLinear(self.feature_num, n * 2, activation=act, normalization=norm)
        self.linear2 = MyLinear(n * 2, n * 3, activation=act, normalization=norm)
        self.linear3 = MyLinear(n * 3, n * 4, activation=act, normalization=norm)
        self.linear_out = MyLinear(n * 4, n * 3, activation=None, normalization=None)
        self.linear_out.linear.bias.data.uniform_(-1, 1)

    def forward(self, x):
        x = self.linear_out(self.linear3(self.linear2(self.linear1(x))))
        return x.view(-1, 3, self.output_point_number)


class ConvToPC(nn.Module):
    """1x1 conv head producing xyz per pixel (models/networks.py:372-391)."""

    def __init__(self, in_channels, opt):
        super().__init__()
        self.in_channels = in_channels
        self.opt = opt
        self.conv1 = MyConv2d(in_channels, int(in_channels), kernel_size=1, stride=1, padding=0,
                              bias=True, activation=opt.activation,
                              normalization=opt.normalization)
        self.conv2 = MyConv2d(int(in_channels), 3, kernel_size=1, stride=1, padding=0, bias=True,
                              activation=None, normalization=None)
        self.conv2.conv.bias.data.uniform_(-1, 1)

    def forward(self, x):
        return self.conv2(self.conv1(x))


class DecoderConv(nn.Module):
    """Up-convolution pyramid 1x1 -> 64x64 (models/networks.py:394-431). PyTorch/cuDNN 3x3 convs:
    out of the hand-written-kernel scope (SURVEY.md §2 row 9, §8f rank 1)."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.feature_num = opt.feature_num
        self.output_point_num = opt.output_conv_pc_num
        f, act, norm = self.feature_num, opt.activation, opt.normalization
        self.deconv1 = UpConv(f, int(f), activation=act, normalization=norm)
        self.deconv2 = UpConv(int(f), int(f / 2), activation=act, normalization=norm)
        self.deconv3 = UpConv(int(f / 2), int(f / 4), activation=act, normalization=norm)
        self.deconv4 = UpConv(int(f / 4), int(f / 8), activation=act, normalization=norm)
        self.conv2pc4 = ConvToPC(int(f / 8), opt)
        self.deconv5 = UpConv(int(f / 8), int(f / 8), activation=act, normalization=norm)
        self.conv2pc5 = ConvToPC(int(f / 8), opt)
        self.deconv6 = UpConv(int(f / 8), int(f / 8), activation=act, normalization=norm)
        self.conv2pc6 = ConvToPC(int(f / 8), opt)

    def outputs(self, x):
        """(pc4, pc5, pc6), the point sets of the 16x16, 32x32 and 64x64 levels, without storing
        them on the module."""
        x = x.view(-1, self.feature_num, 1, 1)
        x = self.deconv4(self.deconv3(self.deconv2(self.deconv1(x))))
        pc4 = self.conv2pc4(x)
        x = self.deconv5(x)
        pc5 = self.conv2pc5(x)
        x = self.deconv6(x)
        return pc4, pc5, self.conv2pc6(x)

    def forward(self, x):
        self.pc4, self.pc5, self.pc6 = self.outputs(x)
        return self.pc6


class Decoder(nn.Module):
    """models/networks.py:434-462."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        if self.opt.output_fc_pc_num > 0:
            self.fc_decoder = DecoderLinear(opt)
        self.conv_decoder = DecoderConv(opt)

    def outputs(self, x):
        """(predicted point set, parts) without storing anything on this module or its submodules:
        parts holds linear_pc when output_fc_pc_num > 0 and conv_pc4 / conv_pc5 / conv_pc6 when
        output_conv_pc_num > 0, the tensors forward() stores under those names."""
        return self._outputs(x, self.conv_decoder.outputs)

    def _stored_pyramid(self, x):
        self.conv_decoder(x)
        return self.conv_decoder.pc4, self.conv_decoder.pc5, self.conv_decoder.pc6

    def _outputs(self, x, pyramid):
        parts = {}
        if self.opt.output_fc_pc_num > 0:
            parts["linear_pc"] = self.fc_decoder(x)
        if self.opt.output_conv_pc_num > 0:
            pc4, pc5, pc6 = pyramid(x)
            parts["conv_pc6"] = pc6.view(-1, 3, 4096)
            parts["conv_pc4"] = pc4.view(-1, 3, 256)
            parts["conv_pc5"] = pc5.view(-1, 3, 1024)
        out = None
        if self.opt.output_fc_pc_num == 0:
            if self.opt.output_conv_pc_num == 4096:
                out = parts["conv_pc6"]
            elif self.opt.output_conv_pc_num == 1024:
                out = parts["conv_pc5"]
        else:
            if self.opt.output_conv_pc_num == 4096:
                out = torch.cat([parts["linear_pc"], parts["conv_pc6"]], 2)
            elif self.opt.output_conv_pc_num == 1024:
                out = torch.cat([parts["linear_pc"], parts["conv_pc5"]], 2)
            else:
                out = parts["linear_pc"]
        return out, parts

    def forward(self, x):
        out, parts = self._outputs(x, self._stored_pyramid)
        for name, t in parts.items():
            setattr(self, name, t)
        return out
