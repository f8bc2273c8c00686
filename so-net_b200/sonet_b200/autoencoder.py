"""autoencoder.Model — caller-facing wrapper of models/autoencoder.py:13-161 on the H100
networks: encoder + decoder + Chamfer, all on the hand-written kernels in eval mode.
Double-buffered asynchronous set_input and CUDA-graph replay of test_model() and
optimize(): _model_base.GraphedModel."""
import torch

from . import augmentation, losses, networks
from ._model_base import ENCODER_SNAPSHOT, GraphedModel


class Model(GraphedModel):
    _SNAPSHOT = {"": ("feature", "predicted_pc", "loss_chamfer", "loss_chamfer_conv4",
                      "loss_chamfer_conv5", "loss"),
                 "encoder": ENCODER_SNAPSHOT,
                 "decoder": ("linear_pc", "conv_pc4", "conv_pc5", "conv_pc6"),
                 "chamfer_criteria": ("forward_loss", "backward_loss", "forward_loss_array",
                                      "backward_loss_array", "loss_array", "nn_idx_fwd",
                                      "nn_idx_bwd")}

    def __init__(self, opt):
        self.opt = opt
        dev = opt.device if isinstance(opt.device, torch.device) else torch.device(opt.device)
        self.encoder = networks.Encoder(opt).to(dev)
        self.decoder = networks.Decoder(opt).to(dev)
        self.chamfer_criteria = losses.ChamferLoss(opt).to(dev)
        B, N, M, K = opt.batch_size, opt.input_pc_num, opt.node_num, max(opt.som_k, 1)
        self._INPUT_SPEC = (
            ("input_pc", lambda d: torch.empty(B, 3, N, dtype=torch.float32, device=d)),
            ("input_sn", lambda d: torch.empty(B, 3, N, dtype=torch.float32, device=d)),
            ("input_label", lambda d: torch.ones(B, dtype=torch.int64, device=d)),
            ("input_node", lambda d: torch.empty(B, 3, M, dtype=torch.float32, device=d)),
            ("input_node_knn_I", lambda d: torch.zeros(B, M, K, dtype=torch.int64, device=d)))
        self._init_io(dev)
        self.test_loss = torch.zeros(1, dtype=torch.float32, device=dev)

    def _state_modules(self):
        return (self.encoder, self.decoder)

    def _after_bind(self, s):
        self.pc, self.sn, self.label = (self.input_pc.detach(), self.input_sn.detach(),
                                        self.input_label.detach())

    def set_input(self, input_pc, input_sn, input_label, input_node, input_node_knn_I):
        """models/autoencoder.py:56-64."""
        self._set_input(input_pc, input_sn, input_label, input_node, input_node_knn_I)

    def _forward(self, is_train, epoch):
        self.feature = self.encoder(self.pc, self.sn, self.input_node, self.input_node_knn_I,
                                    is_train, epoch)
        self.predicted_pc = self.decoder(self.feature)

    def forward(self, is_train=False, epoch=None):
        s = self._wait_inputs()
        self._forward(is_train, epoch)
        self._mark_consumed(s)

    def _losses(self, train):
        """models/autoencoder.py:82-99 (train: conv5 always) / :109-126 (test: conv5 for 4096)."""
        n_conv = self.opt.output_conv_pc_num
        if n_conv > 0:
            if train or n_conv == 4096:
                self.loss_chamfer_conv5 = self.chamfer_criteria(self.decoder.conv_pc5, self.pc)
            self.loss_chamfer_conv4 = self.chamfer_criteria(self.decoder.conv_pc4, self.pc)
        self.loss_chamfer = self.chamfer_criteria(self.predicted_pc, self.pc)
        if n_conv == 1024:
            self.loss = self.loss_chamfer + self.loss_chamfer_conv4
        elif n_conv == 4096:
            self.loss = self.loss_chamfer + self.loss_chamfer_conv5 + self.loss_chamfer_conv4
        else:
            self.loss = self.loss_chamfer

    def _eval_forward(self):
        self._forward(False, None)
        self._losses(train=False)

    def test_model(self):
        """models/autoencoder.py:105-126."""
        self.encoder.eval()
        self.decoder.eval()
        if self._use_graph:
            return self._test_model_graph()
        with torch.no_grad():
            self.forward(is_train=False)
            self._losses(train=False)

    def reconstruct_clouds(self, points, offsets, node, node_knn_I=None, chunk_points=None):
        """The auto-encoder's evaluation against whole clouds of any size, in eval mode: points
        [T,6] f32, offsets [B+1] int64 (cloud b is rows offsets[b] .. offsets[b+1]), node [B,3,M]
        (the test-mode loader's SOM nodes, DeviceDataset.full_batch), node_knn_I [B,M,som_k] int64
        or None to compute it with augmentation.som_knn.

        Encoder.forward_ragged encodes every point of each cloud; the decoder runs once over all B
        features, as test_model() runs it; then test_model()'s combination of Chamfer terms, each
        measured against the WHOLE clouds (losses.chamfer_ragged): predicted_pc, conv_pc4 when
        output_conv_pc_num > 0, conv_pc5 when it is 4096. Each cloud counts once in every term
        whatever its size. Returns a dict: feature [B,F], predicted_pc [B,3,Mp], loss_chamfer,
        loss_chamfer_conv4 and loss_chamfer_conv5 (None when test_model() computes no such term),
        loss, and loss_array [B], predicted_pc's per-cloud loss. With equal-size clouds and the same
        nodes every value is test_model()'s bits.

        Reads no bound input and writes no attribute of the model, its modules or chamfer_criteria:
        what test_model() left, and a captured eval graph, stay as they were. Refused before any
        launch: train mode and Encoder.check_ragged's cases, --normalization instance among them
        (instance statistics have no ragged kernels)."""
        enc, dec, opt = self.encoder, self.decoder, self.opt
        if enc.training or dec.training:
            raise RuntimeError("reconstruct_clouds: the model is in train mode; call test_model() "
                               "or eval() first")
        enc.check_ragged(points, offsets, node, node_knn_I, chunk_points, what="reconstruct_clouds")
        with torch.no_grad():
            if node_knn_I is None:
                node_knn_I = augmentation.som_knn(node.detach().contiguous(), opt.som_k,
                                                  node.shape[2])
            feature = enc.forward_ragged(points, offsets, node, node_knn_I, chunk_points)
            predicted_pc, parts = dec.outputs(feature)
            n_conv = opt.output_conv_pc_num
            conv4 = conv5 = None
            if n_conv > 0:
                if n_conv == 4096:
                    conv5 = losses.chamfer_ragged(parts["conv_pc5"], points, offsets).loss
                conv4 = losses.chamfer_ragged(parts["conv_pc4"], points, offsets).loss
            main = losses.chamfer_ragged(predicted_pc, points, offsets)
            if n_conv == 1024:
                loss = main.loss + conv4
            elif n_conv == 4096:
                loss = main.loss + conv5 + conv4
            else:
                loss = main.loss
        return dict(feature=feature, predicted_pc=predicted_pc, loss_chamfer=main.loss,
                    loss_chamfer_conv4=conv4, loss_chamfer_conv5=conv5, loss=loss,
                    loss_array=main.loss_array)

    def _make_optimizers(self):
        return (torch.optim.Adam(self.encoder.parameters(), lr=self.opt.lr, betas=(0.9, 0.999)),
                torch.optim.Adam(self.decoder.parameters(), lr=self.opt.lr, betas=(0.9, 0.999)))

    def _train_step(self, epoch, forward):
        """One training step (models/autoencoder.py:70-103) on the differentiable PyTorch path;
        optimize() runs it (GraphedModel.optimize)."""
        self.encoder.train()
        self.decoder.train()
        with torch.enable_grad():
            forward(True, epoch)
            self.encoder.zero_grad()
            self.decoder.zero_grad()
            self._losses(train=True)
            self.loss.backward()
        for o in self._optim:
            o.step()
