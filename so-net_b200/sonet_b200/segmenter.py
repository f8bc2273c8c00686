"""segmenter.Model — caller-facing wrapper of models/segmenter.py:14-192 on the H100 networks.

forward() hands the Segmenter the node-level features and the point->node assignment directly
(Segmenter.forward_nodes) instead of the three per-point torch.gather copies of
models/segmenter.py:90-98. Double-buffered asynchronous set_input and CUDA-graph replay of
test_model() and optimize(): _model_base.GraphedModel.
"""
import torch

from . import losses, networks, ops
from ._model_base import ENCODER_SNAPSHOT, GraphedModel


class Model(GraphedModel):
    _SNAPSHOT = {"": ("feature", "score_segmenter", "loss_segmenter", "loss"),
                 "encoder": ENCODER_SNAPSHOT}

    def __init__(self, opt):
        self.opt = opt
        dev = opt.device if isinstance(opt.device, torch.device) else torch.device(opt.device)
        self.encoder = networks.Encoder(opt).to(dev)
        self.segmenter = networks.Segmenter(opt).to(dev)
        self.softmax_segmenter = losses.CrossEntropyLossSeg().to(dev)
        self.encoder.fuse_pool = False   # the head reads first_pn_out of every forward
        B, N, M, K = opt.batch_size, opt.input_pc_num, opt.node_num, max(opt.som_k, 1)
        self._INPUT_SPEC = (
            ("input_pc", lambda d: torch.empty(B, 3, N, dtype=torch.float32, device=d)),
            ("input_sn", lambda d: torch.empty(B, 3, N, dtype=torch.float32, device=d)),
            ("input_label", lambda d: torch.ones(B, dtype=torch.int64, device=d)),
            ("input_seg", lambda d: torch.ones(B, 50, dtype=torch.int64, device=d)),
            ("input_node", lambda d: torch.empty(B, 3, M, dtype=torch.float32, device=d)),
            ("input_node_knn_I", lambda d: torch.zeros(B, M, K, dtype=torch.int64, device=d)))
        self._init_io(dev)
        self._evaluated = False      # test_model() has run on the bound batch (score_points)

    def _state_modules(self):
        return (self.encoder, self.segmenter)

    def _after_bind(self, s):
        self.pc, self.sn = self.input_pc.detach(), self.input_sn.detach()
        self.seg, self.label = self.input_seg.detach(), self.input_label.detach()

    def set_input(self, input_pc, input_sn, input_label, input_seg, input_node, input_node_knn_I):
        """models/segmenter.py:66-77."""
        self._set_input(input_pc, input_sn, input_label, input_seg, input_node, input_node_knn_I)
        self._evaluated = False

    def _forward(self, is_train, epoch):
        enc = self.encoder
        self.feature = enc(self.pc, self.sn, self.input_node, self.input_node_knn_I, is_train, epoch)
        self.score_segmenter = self.segmenter.forward_nodes(
            enc.x_decentered, self.pc, enc.centers, self.sn, self.input_label, enc.first_pn_out,
            enc.first_pn_out_masked_max, enc.knn_feature_1, enc.final_pn_out, self.feature,
            enc.min_idx)

    def forward(self, is_train=False, epoch=None):
        s = self._wait_inputs()
        self._forward(is_train, epoch)
        self._mark_consumed(s)

    def _loss(self):
        # models/segmenter.py:129-131; computed only when the targets match the scores' point
        # axis (the placeholder input_seg of the constructor does not)
        if self.seg.dim() == 2 and self.seg.shape[1] == self.score_segmenter.shape[2]:
            self.loss_segmenter = self.softmax_segmenter(self.score_segmenter, self.seg)
            self.loss = self.loss_segmenter

    def _eval_forward(self):
        self._forward(False, None)
        self._loss()

    def test_model(self):
        self.encoder.eval()
        self.segmenter.eval()
        if self._use_graph:
            self._test_model_graph()
        else:
            with torch.no_grad():
                self.forward(is_train=False)
                self._loss()
        self._evaluated = True

    def _make_optimizers(self):
        return (torch.optim.Adam(self.encoder.parameters(), lr=self.opt.lr,
                                 betas=(0.9, 0.999), weight_decay=0),
                torch.optim.Adam(self.segmenter.parameters(), lr=self.opt.lr,
                                 betas=(0.9, 0.999), weight_decay=0))

    def _train_step(self, epoch, forward):
        """One training step (models/segmenter.py:111-123) on the differentiable PyTorch path;
        optimize() runs it (GraphedModel.optimize)."""
        self._evaluated = False
        self.encoder.train()
        self.segmenter.train()
        with torch.enable_grad():
            forward(True, epoch)
            self.encoder.zero_grad()
            self.segmenter.zero_grad()
            self.loss_segmenter = self.softmax_segmenter(self.score_segmenter, self.seg)
            self.loss_segmenter.backward()
        for o in self._optim:
            o.step()

    # ---- every point of each shape -----------------------------------------------------------
    # device bytes per stacked copy of a row in one chunk: pt, x_aug, first_pn_out and layers 1-3
    _COPY_BYTES = 4 * (12 + 6 + 384 + 1024 + 512 + 256) + 4
    # padding unit of a chunk's rows (whole wgmma row tiles). It decides no kernel route: every
    # layer takes the route of the sampled forward (Segmenter.forward_rows)
    _ROW_QUANTUM = 256

    def _default_chunk_rows(self, total):
        free, _ = torch.cuda.mem_get_info(self._dev)
        per_row = self.opt.k * self._COPY_BYTES + 4 * (256 + 128 + 2 * self.opt.classes)
        rows = (free // 4) // per_row
        rows = max(self._ROW_QUANTUM, rows // self._ROW_QUANTUM * self._ROW_QUANTUM)
        return int(min(rows, total))

    def score_points(self, points, offsets, chunk_rows=None):
        """Scores of EVERY point of each shape of the batch just evaluated by test_model():
        points [sum P_i, 6] f32 on the model's device (xyz | normal, DeviceDataset.data's layout),
        offsets [B+1] int64 (cloud b of the ragged set is row b of the sampled batch). Returns
        score [sum P_i, classes] f32: per point what score_segmenter [B, classes, N] holds per
        sampled point.

        A point's score depends only on its coordinates and normal, its k nearest of the cloud's
        loader SOM nodes, the cloud's node-level features [B,C,M] and its per-cloud vector
        (one-hot label, global feature), all kept from the sampled forward. Each point is assigned
        to its k nearest loader nodes with the encoder's arithmetic, decentred by those nodes'
        cluster means (encoder.som_node), and run through the first PointResNet, the split layer 1
        with the node/cloud addend, layers 2-5 and the k-copy mean. Rows go in chunks of
        chunk_rows (default: a quarter of the free device memory); the chunking changes no bit.
        Each layer runs on the kernel the sampled forward ran it on for its B*N points, so the
        sampled points themselves get score_segmenter's bits at every batch size.

        Refused (RuntimeError, before any launch): train mode; instance normalisation (layer 1's
        per-row statistics would depend on the point set); som_k < 2; a batch test_model() has not
        evaluated; offsets that do not match the batch or the points."""
        enc, seg, opt = self.encoder, self.segmenter, self.opt
        if enc.training or seg.training:
            raise RuntimeError("score_points: the model is in train mode; call test_model() first")
        if opt.normalization == 'instance':
            raise RuntimeError("score_points: --normalization instance normalises layer 1 over each "
                               "cloud's rows, so a point's score depends on the point set")
        if opt.som_k < 2:
            raise RuntimeError("score_points: needs the KNN module's node features (som_k >= 2)")
        if not self._evaluated:
            raise RuntimeError("score_points: the bound batch has not been evaluated by test_model()")
        if points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] != 6:
            raise RuntimeError("score_points: points must be float32 [T, 6] (got %s %s)"
                               % (points.dtype, tuple(points.shape)))
        B = self.input_pc.shape[0]
        T = points.shape[0]
        ops.ragged_offsets(offsets, T, B)
        if points.device != self.input_pc.device or not points.is_cuda:
            raise RuntimeError("score_points: points must be on the model's device %s (got %s)"
                               % (self.input_pc.device, points.device))
        if chunk_rows is not None and chunk_rows < 1:
            raise RuntimeError("score_points: chunk_rows must be >= 1 (got %d)" % chunk_rows)
        k = opt.k
        BN = B * self.input_pc.shape[2]      # the sampled forward's points: the layers' routes
        use_sn = opt.surface_normal == True  # noqa: E712
        with torch.no_grad():
            points = points.contiguous()
            offsets = offsets.to(points.device).contiguous()
            addend, packed = seg._node_addend(12 if use_sn else 9, 384, enc.first_pn_out_masked_max,
                                              enc.knn_feature_1, enc.final_pn_out, self.feature,
                                              self.input_label)
            C, M = addend.shape[1], addend.shape[2]
            addend_flat = addend.permute(1, 0, 2).reshape(1, C, B * M).contiguous()
            node = self.input_node.detach().to(torch.float32).contiguous()
            score = torch.empty((T, opt.classes), dtype=torch.float32, device=points.device)
            chunk = min(int(chunk_rows), T) if chunk_rows else self._default_chunk_rows(T)
            q = self._ROW_QUANTUM
            for r0 in range(0, T, max(chunk, 1)):
                R = min(chunk, T - r0)
                gidx, x_aug, pt = ops.seg_points_assign(points, offsets, node, enc.som_node, k,
                                                        use_sn, r0, R, (R + q - 1) // q * q)
                fpo = enc.first_pointnet(x_aug, route_rows=k * BN)
                y = seg.forward_rows(pt, fpo, addend_flat, gidx, k, packed, BN)   # [1,classes,Rp]
                score[r0:r0 + R].copy_(y[0, :, :R].t())
        return score
