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
