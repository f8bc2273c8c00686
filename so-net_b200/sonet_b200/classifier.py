"""classifier.Model — the caller-facing wrapper of models/classifier.py:15-153 (set_input /
forward / test_model / optimize), built on the H100 networks. This is the public API bench.py
times end to end: host tensors in through set_input, scores out.

set_input is double-buffered and asynchronous, test_model() and optimize() can each replay as one
CUDA graph (enable_cuda_graph, enable_train_graph) — see _model_base.GraphedModel.
"""
import torch
import torch.nn as nn

from . import augmentation, networks
from ._model_base import ENCODER_SNAPSHOT, GraphedModel


class Model(GraphedModel):
    _SNAPSHOT = {"": ("feature", "score", "loss"), "encoder": ENCODER_SNAPSHOT}

    def __init__(self, opt):
        self.opt = opt
        dev = opt.device if isinstance(opt.device, torch.device) else torch.device(opt.device)
        self.encoder = networks.Encoder(opt).to(dev)
        self.classifier = networks.Classifier(opt).to(dev)
        self.softmax_criteria = nn.CrossEntropyLoss().to(dev)
        B, N, M, K = opt.batch_size, opt.input_pc_num, opt.node_num, max(opt.som_k, 1)
        self._INPUT_SPEC = (
            ("input_pc", lambda d: torch.empty(B, 3, N, dtype=torch.float32, device=d)),
            ("input_sn", lambda d: torch.empty(B, 3, N, dtype=torch.float32, device=d)),
            ("input_label", lambda d: torch.ones(B, dtype=torch.int64, device=d)),
            ("input_node", lambda d: torch.empty(B, 3, M, dtype=torch.float32, device=d)),
            ("input_node_knn_I", lambda d: torch.zeros(B, M, K, dtype=torch.int64, device=d)))
        self._init_io(dev)
        self.test_loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self.test_accuracy = torch.zeros(1, dtype=torch.float32)

    def _state_modules(self):
        return (self.encoder, self.classifier)

    def _after_bind(self, s):
        self.pc, self.sn, self.label = (self.input_pc.detach(), self.input_sn.detach(),
                                        self.input_label.detach())

    def _eval_forward(self):
        self.feature = self.encoder(self.pc, self.sn, self.input_node, self.input_node_knn_I,
                                    False, None)
        self.score = self.classifier(self.feature, None)
        self.loss = self.softmax_criteria(self.score, self.label)

    def set_input(self, input_pc, input_sn, input_label, input_node, input_node_knn_I):
        """models/classifier.py:64-72."""
        self._set_input(input_pc, input_sn, input_label, input_node, input_node_knn_I)

    def _forward(self, is_train, epoch):
        self.feature = self.encoder(self.pc, self.sn, self.input_node, self.input_node_knn_I,
                                    is_train, epoch)
        self.score = self.classifier(self.feature, epoch)

    def forward(self, is_train=False, epoch=None):
        s = self._wait_inputs()
        self._forward(is_train, epoch)
        self._mark_consumed(s)

    def test_model(self):
        self.encoder.eval()
        self.classifier.eval()
        if self._use_graph:
            return self._test_model_graph()
        with torch.no_grad():
            self.forward(is_train=False)
            self.loss = self.softmax_criteria(self.score, self.label)

    def score_clouds(self, points, offsets, node, node_knn_I=None, chunk_points=None):
        """Class scores [B, classes] of whole clouds of any size, from all of their points, in eval
        mode: points [T,6] f32, offsets [B+1] int64, node [B,3,M] (the test-mode loader's SOM nodes,
        DeviceDataset.full_batch), node_knn_I [B,M,som_k] int64 or None to compute it with
        augmentation.som_knn. Encoder.forward_ragged, then the classifier head (dropout is the
        identity in eval mode). Reads no bound input and writes no attribute of the model: score,
        the encoder's state and a captured eval graph stay as test_model() left them. Refused before
        any launch: train mode and Encoder.check_ragged's cases."""
        enc, head, opt = self.encoder, self.classifier, self.opt
        if enc.training or head.training:
            raise RuntimeError("score_clouds: the model is in train mode; call test_model() or "
                               "eval() first")
        enc.check_ragged(points, offsets, node, node_knn_I, chunk_points, what="score_clouds")
        with torch.no_grad():
            if node_knn_I is None:
                node_knn_I = augmentation.som_knn(node.detach().contiguous(), opt.som_k,
                                                  node.shape[2])
            feature = enc.forward_ragged(points, offsets, node, node_knn_I, chunk_points)
            return head.fc3(head.fc2(head.fc1(feature)))

    def optimize_clouds(self, points, offsets, label, node, node_knn_I=None, epoch=None):
        """One training step (optimize()'s: forward, zero_grad, CrossEntropyLoss, backward, both
        Adam steps) on whole clouds of any size: points [T,6] f32, offsets [B+1] int64, label [B]
        int64 in [0, classes), node [B,3,M] and node_knn_I [B,M,som_k] int64 or None to compute it
        (DeviceDataset.full_batch(train=True) draws such batches). The encoder runs
        Encoder.forward_ragged_train; the loss is the mean over the B clouds, so each cloud counts
        once whatever its size. Returns dict(loss, score [B,classes]), both detached.

        Shares optimize()'s optimizers, so interleaving the two is one training run. Always eager
        (every batch has its own shapes), also after enable_train_graph(True) has made Adam
        capturable; reads no bound input, rebinds no buffer of a captured graph and writes no model
        attribute but the parameters, their gradients, the optimizer state and the BatchNorm running
        statistics. Refused before any launch: Encoder.check_ragged(train=True)'s cases and a label
        that is not [B] int64 on the model's device with values in [0, classes)."""
        enc, opt = self.encoder, self.opt
        enc.check_ragged(points, offsets, node, node_knn_I, what="optimize_clouds", train=True)
        B = node.shape[0]
        if not isinstance(label, torch.Tensor) or label.dtype != torch.int64 \
                or tuple(label.shape) != (B,) or label.device != node.device:
            raise RuntimeError("optimize_clouds: label must be a [%d] int64 tensor on %s (got %s)" % (
                B, node.device, (label.dtype, tuple(label.shape), str(label.device))
                if isinstance(label, torch.Tensor) else type(label).__name__))
        lo, hi = (int(v) for v in torch.stack((label.min(), label.max())).cpu())
        if lo < 0 or hi >= opt.classes:
            raise RuntimeError("optimize_clouds: label values must lie in [0, %d) (got %d .. %d)"
                               % (opt.classes, lo, hi))
        if self._optim is None:
            self._optim = self._make_optimizers()
        enc.train()
        self.classifier.train()
        with torch.enable_grad():
            feature = enc.forward_ragged_train(points, offsets, node, node_knn_I, epoch)
            score = self.classifier(feature, epoch, store=False)
            enc.zero_grad()
            self.classifier.zero_grad()
            loss = self.softmax_criteria(score, label)
            loss.backward()
        for o in self._optim:
            o.step()
        return dict(loss=loss.detach(), score=score.detach())

    def _make_optimizers(self):
        return (torch.optim.Adam(self.encoder.parameters(), lr=self.opt.lr,
                                 betas=(0.9, 0.999), weight_decay=0),
                torch.optim.Adam(self.classifier.parameters(), lr=self.opt.lr,
                                 betas=(0.9, 0.999), weight_decay=0))

    def _train_step(self, epoch, forward):
        """One training step (models/classifier.py:78-99) on the differentiable PyTorch path;
        optimize() runs it (GraphedModel.optimize)."""
        self.encoder.train()
        self.classifier.train()
        with torch.enable_grad():
            forward(True, epoch)
            self.encoder.zero_grad()
            self.classifier.zero_grad()
            self.loss = self.softmax_criteria(self.score, self.label)
            self.loss.backward()
        for o in self._optim:
            o.step()
