"""segmenter.Model — caller-facing wrapper of models/segmenter.py:14-192 on the H100 networks.

forward() hands the Segmenter the node-level features and the point->node assignment directly
(Segmenter.forward_nodes) instead of the three per-point torch.gather copies of
models/segmenter.py:90-98. Double-buffered asynchronous set_input and CUDA-graph replay of
test_model() and optimize(): _model_base.GraphedModel.
"""
import torch

from . import losses, networks
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

    def _state_modules(self):
        return (self.encoder, self.segmenter)

    def _after_bind(self, s):
        self.pc, self.sn = self.input_pc.detach(), self.input_sn.detach()
        self.seg, self.label = self.input_seg.detach(), self.input_label.detach()

    def set_input(self, input_pc, input_sn, input_label, input_seg, input_node, input_node_knn_I):
        """models/segmenter.py:66-77."""
        self._set_input(input_pc, input_sn, input_label, input_seg, input_node, input_node_knn_I)

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
            return self._test_model_graph()
        with torch.no_grad():
            self.forward(is_train=False)
            self._loss()

    def _make_optimizers(self):
        return (torch.optim.Adam(self.encoder.parameters(), lr=self.opt.lr,
                                 betas=(0.9, 0.999), weight_decay=0),
                torch.optim.Adam(self.segmenter.parameters(), lr=self.opt.lr,
                                 betas=(0.9, 0.999), weight_decay=0))

    def _train_step(self, epoch, forward):
        """One training step (models/segmenter.py:111-123) on the differentiable PyTorch path;
        optimize() runs it (GraphedModel.optimize)."""
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
