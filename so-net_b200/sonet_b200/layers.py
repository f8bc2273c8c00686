"""Layer classes with the reference's constructor signatures and state_dict keys
(models/layers.py:22-432), running on the sm_90a kernels of libsonet_b200 in eval/no-grad mode.

Dispatch rule (SURVEY.md §8b "Autograd"): the hand-written forward kernels run whenever the module
is in eval() mode and no INPUT tensor carries a gradient — with or without torch.no_grad(), because
the reference's own test loop (models/classifier.py:101-105, modelnet/train.py:72-76) calls
test_model() in eval mode WITHOUT no_grad and must still land on the hot path. An eval-mode forward
therefore returns tensors without grad_fn: calling backward() on them fails loudly ("does not
require grad") instead of silently dropping parameter gradients. In train() mode, when an input
requires grad (saliency / adversarial use in eval mode), or when EVAL_AUTOGRAD is set, the layers
compose differentiable PyTorch ops on the GPU exactly as the reference does — the reference's own
training path, not a CPU fallback. Both activations of the reference's options (relu, elu) run on
the kernels, as does no activation; swish and leakyrelu always take the PyTorch path.

Both normalizations of the reference's options (batch, instance) run on the kernels too. BatchNorm
folds into the layer's GEMM in eval mode. Instance norm (track_running_stats=False: eval and train
compute the same forward) needs each row's statistics over all its points first: an instance layer
runs its GEMM with the conv bias and no activation, then ops.instance_norm applies the per-row
statistics, gamma, beta and the activation in one pass, fused with the KNN module's max over
neighbours or the segmenter's k-copy mean where those follow. MyLinear with instance norm keeps the
PyTorch path: on a [B, C] input nn.InstanceNorm1d raises in the reference, and so it does here. The
fused first-PointResNet and KNN kernels are BatchNorm-only; instance models take the per-layer chain.
"""
import itertools
import math
import os

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.modules.batchnorm import _BatchNorm

from . import operations, ops, train_ops


# Set to True to make eval-mode forwards differentiable w.r.t. the parameters as well (the
# PyTorch composition); the default keeps eval() = inference kernels.
EVAL_AUTOGRAD = False


def _fast_ok(module, *tensors):
    if module.training:
        return False
    if torch.is_grad_enabled() and (EVAL_AUTOGRAD or any(t is not None and t.requires_grad
                                                         for t in tensors)):
        return False
    return all(t is not None and t.is_cuda and t.dtype == torch.float32 for t in tensors)


class Swish(nn.Module):
    """x * sigmoid(x) (models/layers.py:14-19)."""

    def forward(self, x):
        return x * torch.sigmoid(x)


class _MomentumDecayBatchNorm(_BatchNorm):
    """BatchNorm whose momentum decays with the epoch (models/layers.py:22-70, 73-120)."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True,
                 momentum_decay_step=None, momentum_decay=1):
        super().__init__(num_features, eps, momentum, affine)
        self.momentum_decay_step = momentum_decay_step
        self.momentum_decay = momentum_decay
        self.momentum_original = self.momentum

    def momentum_at(self, epoch):
        """The momentum a train forward at `epoch` uses: the decayed one from epoch 1 on when a
        decay step is set, else the current one (the last epoch's, or the constructor's)."""
        step = self.momentum_decay_step
        if epoch is not None and epoch >= 1 and step is not None and step > 0:
            return max(self.momentum_original * (self.momentum_decay ** (epoch // step)), 0.01)
        return self.momentum

    def forward(self, input, epoch=None):
        self.momentum = self.momentum_at(epoch)
        if self.training and train_ops.EXCHANGE is not None:
            # data-parallel training synchronises the BatchNorms on the train kernels only; this
            # one would normalise each rank's shard by its own statistics
            raise RuntimeError("a data-parallel train step reached a BatchNorm outside the train "
                               "kernels (train_ops.norm_act_train)")
        return F.batch_norm(input, self.running_mean, self.running_var, self.weight, self.bias,
                            self.training, self.momentum, self.eps)


class MyBatchNorm1d(_MomentumDecayBatchNorm):
    def _check_input_dim(self, input):
        if input.dim() not in (2, 3):
            raise ValueError('expected 2D or 3D input (got {}D input)'.format(input.dim()))


class MyBatchNorm2d(_MomentumDecayBatchNorm):
    def _check_input_dim(self, input):
        if input.dim() != 4:
            raise ValueError('expected 4D input (got {}D input)'.format(input.dim()))


# activations with a kernel epilogue (ops.act_code); others compose PyTorch ops
KERNEL_ACTIVATIONS = (None, 'relu', 'elu')
# normalizations with a kernel: BatchNorm folded into the GEMM, instance norm by ops.instance_norm
KERNEL_NORMALIZATIONS = (None, 'batch', 'instance')


def _norm_on_kernels(normalization, norm):
    """A layer's normalization runs on the kernels: None, BatchNorm, or instance norm without
    running statistics (the reference's nn.InstanceNorm*d default; with running statistics eval
    mode would normalise by those instead)."""
    if normalization not in KERNEL_NORMALIZATIONS:
        return False
    return normalization != 'instance' or not norm.track_running_stats


def _make_act(activation):
    if activation == 'relu':
        return nn.ReLU()
    if activation == 'elu':
        return nn.ELU(alpha=1.0)
    if activation == 'swish':
        return Swish()
    if activation == 'leakyrelu':
        return nn.LeakyReLU(0.1)
    return None


def tc_mode():
    """The eval-mode precision of the tensor-core layers, from SONET_TC, read at call time so a
    change applies from the next forward on (a captured CUDA graph is re-captured):
      "fp32"  SONET_TC=0: every layer on the exact-fp32 CUDA-core kernels;
      "fp16"  SONET_TC=fp16: every wgmma GEMM as one fp16 product per MAC (the `_f16` entries);
      "split" anything else, unset and 1 included: the fp16 hi/lo 3-product split (default).
    Train mode ignores it. No other module reads the variable."""
    v = os.environ.get("SONET_TC", "1")
    if v == "0":
        return "fp32"
    if v == "fp16":
        return "fp16"
    return "split"


def tc_enabled():
    """True unless SONET_TC=0, which routes every layer to the exact-fp32 CUDA-core kernels."""
    return tc_mode() != "fp32"


def tc_f16():
    """True under SONET_TC=fp16: the eval wgmma launches take their one-product `_f16` entries."""
    return tc_mode() == "fp16"


_stamps = itertools.count(1)


class _Cache:
    """A value derived from module parameters, rebuilt by get() when its key (never None)
    changes. Values derived from this one key on `version`, a stamp of the current value unique
    across all caches, so such a key also changes when a source layer is swapped for another."""
    _key = _value = version = None

    def clear(self):
        self._key = self._value = self.version = None

    def get(self, key, build):
        if key != self._key:
            self._value = build()
            self._key, self.version = key, next(_stamps)
        return self._value


class _FoldedParams(_Cache):
    """Eval-mode conv/linear + BatchNorm folded into (weights, shift), re-folded only when a
    parameter or running statistic changes (tracked through tensor version counters).

      y = gamma * (W x + bias - mean) / sqrt(var + eps) + beta  =  (s*W) x + ((bias-mean)*s + beta)

    get() takes the fold's sources instead of a key and builder: it derives both from them.
    """

    def __init__(self):
        self._wt = _Cache()     # [Cin, Cout] (the point-wise kernel wants K-major slabs)

    def get(self, weight2d, bias, norm, transpose):
        srcs = [weight2d, bias]
        if norm is not None:
            srcs += [norm.weight, norm.bias, norm.running_mean, norm.running_var]
        key = tuple((t.data_ptr(), t._version, t.device) for t in srcs if t is not None)

        def build():
            with torch.no_grad():
                w = weight2d.detach().float()
                shift = bias.detach().float() if bias is not None else \
                    torch.zeros(w.shape[0], device=w.device)
                if norm is not None:
                    s = norm.weight.detach() / torch.sqrt(norm.running_var.detach() + norm.eps)
                    shift = (shift - norm.running_mean.detach()) * s + norm.bias.detach()
                    w = w * s[:, None]
                return w.contiguous(), shift.contiguous()      # [Cout, Cin], [Cout]
        w, shift = super().get(key, build)
        if not transpose:
            return w, shift
        return self._wt.get(self.version, lambda: w.t().contiguous()), shift


def invalidate(module):
    """Drop every derived weight cache (BN-folded weights, wgmma packings) below `module`.

    The BN fold is keyed on (data_ptr, tensor._version, device) of the parameters and BN
    statistics, which optimizer steps, load_state_dict() and in-place tensor ops all bump; the
    packings derived from a fold are keyed on its version. Writes through `.data`
    (`p.data.mul_(..)`, `w.data.copy_(..)` — an idiom of the reference code base,
    e.g. models/networks.py:366) do NOT bump the version counter: call this after such edits."""
    for m in module.modules():
        for v in vars(m).values():
            if isinstance(v, _Cache):
                v.clear()


class MyLinear(nn.Module):
    """Linear + BN1d + act (models/layers.py:123-166)."""

    def __init__(self, in_features, out_features, activation=None, normalization=None,
                 momentum=0.1, bn_momentum_decay_step=None, bn_momentum_decay=1):
        super().__init__()
        self.activation = activation
        self.normalization = normalization
        self.linear = nn.Linear(in_features, out_features, bias=True)
        if normalization == 'batch':
            self.norm = MyBatchNorm1d(out_features, momentum=momentum, affine=True,
                                      momentum_decay_step=bn_momentum_decay_step,
                                      momentum_decay=bn_momentum_decay)
        elif normalization == 'instance':
            self.norm = nn.InstanceNorm1d(out_features, momentum=momentum, affine=True)
        act = _make_act(activation)
        if act is not None:
            self.act = act
        self._folded = _FoldedParams()
        self.weight_init()

    def weight_init(self):
        nn.init.normal_(self.linear.weight, 0, math.sqrt(2. / self.linear.in_features))
        nn.init.zeros_(self.linear.bias)
        if self.normalization in ('batch', 'instance'):
            nn.init.ones_(self.norm.weight)
            nn.init.zeros_(self.norm.bias)

    def folded(self, transpose=False):
        """Eval-mode (w [Cout,Cin] or with transpose [Cin,Cout], shift [Cout]), BN folded in."""
        return self._folded.get(self.linear.weight, self.linear.bias,
                                self.norm if self.normalization == 'batch' else None, transpose)

    def _fast(self, x):
        # instance norm stays PyTorch: on [B, C] the reference's nn.InstanceNorm1d raises
        return (_fast_ok(self, x) and x.dim() == 2
                and self.normalization in KERNEL_NORMALIZATIONS and self.normalization != 'instance'
                and self.activation in KERNEL_ACTIVATIONS)

    def _train_kernels(self, x):
        # instance norm keeps the PyTorch path here too (nn.InstanceNorm1d raises on [B, C])
        return (train_ops.ENABLED and self.training and torch.is_grad_enabled() and x.is_cuda
                and x.dtype == torch.float32 and x.dim() == 2
                and self.normalization in (None, 'batch') and self.activation in KERNEL_ACTIVATIONS)

    def forward(self, x, epoch=None):
        if self._fast(x):
            w, shift = self.folded()
            return ops.linear(x.contiguous(), w, None, shift, self.activation)
        if self._train_kernels(x):
            y = train_ops.LinearStrict.apply(x, self.linear.weight, self.linear.bias)
            norm = self.norm if self.normalization == 'batch' else None
            return train_ops.norm_act_train(y.unsqueeze(2), norm, self.activation, epoch,
                                            size=y.shape).squeeze(2)
        x = self.linear(x)
        if self.normalization == 'batch':
            x = self.norm(x, epoch)
        elif self.normalization is not None:
            x = self.norm(x)
        if self.activation is not None:
            x = self.act(x)
        return x


class _PointwiseConvBase(nn.Module):
    """Shared eval fast path of the 1x1 conv layers: y = act(BN(conv1x1(cat(x0, x1))))."""

    def __init__(self):
        super().__init__()
        self._folded = _FoldedParams()
        self._tc = _Cache()

    def _conv_weight2d(self):
        w = self.conv.weight
        return w.view(w.shape[0], -1)

    def folded(self, transpose=False):
        """Eval-mode (w [Cout,Cin*kh*kw] or its transpose, shift [Cout]), BN folded in."""
        return self._folded.get(self._conv_weight2d(), self.conv.bias,
                                self.norm if self.normalization == 'batch' else None, transpose)

    def _tc_params(self):
        """(blob, inv_scale, shift) of the folded weight for the wgmma kernel, on its device."""
        w, shift = self.folded()

        def build():
            blob, inv = ops.pointwise_tc_pack(w)
            return blob.to(w.device), inv, shift
        return self._tc.get(self._folded.version, build)

    def _fast_eligible(self):
        ks = self.conv.kernel_size
        return (all(k == 1 for k in ks) and all(s == 1 for s in self.conv.stride)
                and all(p == 0 for p in self.conv.padding)
                and _norm_on_kernels(self.normalization, getattr(self, "norm", None))
                and self.activation in KERNEL_ACTIVATIONS)

    def _train_kernels(self, x):
        """train() mode on CUDA fp32 with a kernel norm/activation: the sm_90a train kernels
        (train_ops) instead of the PyTorch composition. Instance norm also needs its affine
        parameters (the reference's layers always have them)."""
        return (train_ops.ENABLED and self.training and torch.is_grad_enabled() and x.is_cuda
                and x.dtype == torch.float32 and self._fast_eligible()
                and (self.normalization != 'instance' or self.norm.affine))

    def _train_norm(self):
        """The norm module train_ops.conv_bn_act_train applies (None: no normalization)."""
        return self.norm if self.normalization in ('batch', 'instance') else None

    def instance_norm(self, z, kcopy=None, group_max=None):
        """This layer's instance norm + activation on its pre-norm output z [B,Cout,P] (in place
        without a reduction; kcopy / group_max as ops.instance_norm)."""
        n = self.norm
        return ops.instance_norm(z, n.weight, n.bias, n.eps, self.activation, kcopy=kcopy,
                                 group_max=group_max,
                                 out=z if kcopy is None and group_max is None else None)

    def forward_points(self, x0, x1=None, addend=None, gidx=None, kcopy=None, group_max=None,
                       route_rows=None):
        """x0 [B,C0,P] (+ x1 [B,C1,P] virtually concatenated on channels) -> [B,Cout,P].
        Dense layers run on wgmma (csrc/pointwise_tc.cu, fp16 hi/lo split); thin ones on the
        exact-fp32 CUDA-core kernel (csrc/pointwise.cu). An instance-norm layer writes the GEMM's
        z (conv bias, no activation) and normalises it with ops.instance_norm, which can also
        reduce the result (kcopy / group_max: instance layers only). route_rows: the row count
        that picks the kernel instead of B*P, for a launch that must take the route of another
        (segmenter.Model.score_points runs each layer on the route of the sampled forward)."""
        inst = self.normalization == 'instance'
        if not inst and (kcopy is not None or group_max is not None):
            raise RuntimeError("forward_points: kcopy / group_max are fused into instance norm only")
        act = None if inst else self.activation
        cin = x0.shape[1] + (0 if x1 is None else x1.shape[1])
        cout = self.conv.out_channels
        rows = x0.shape[0] * x0.shape[2] if route_rows is None else route_rows
        # wgmma eligibility: a dense enough contraction (cin >= 32) over at least two 128-row
        # tiles; thin OUTPUTS (the 128 -> 3 ConvToPC heads) qualify too — the layer is then a
        # streaming read of the activations into the tensor-core kernel instead of the
        # register-tiled fp32 kernel
        if cin >= 32 and rows >= 256 and tc_enabled():
            blob, inv, shift = self._tc_params()
            z = ops.pointwise_layer_tc(x0, blob, inv, shift, cout, act,
                                       x1=x1, addend=addend, gidx=gidx, f16=tc_f16())
        else:
            w, shift = self.folded(transpose=True)
            z = ops.pointwise_layer(x0, w, None, shift, act, x1=x1, addend=addend, gidx=gidx)
        return self.instance_norm(z, kcopy, group_max) if inst else z


class MyConv2d(_PointwiseConvBase):
    """Conv2d + BN2d + act (models/layers.py:169-211); 1x1 kernels run on the point-wise kernel."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, bias=True,
                 activation=None, momentum=0.1, normalization=None, bn_momentum_decay_step=None,
                 bn_momentum_decay=1):
        super().__init__()
        self.activation = activation
        self.normalization = normalization
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride, padding, bias=bias)
        if normalization == 'batch':
            self.norm = MyBatchNorm2d(out_channels, momentum=momentum, affine=True,
                                      momentum_decay_step=bn_momentum_decay_step,
                                      momentum_decay=bn_momentum_decay)
        elif normalization == 'instance':
            self.norm = nn.InstanceNorm2d(out_channels, momentum=momentum, affine=True)
        act = _make_act(activation)
        if act is not None:
            self.act = act
        self.weight_init()

    def weight_init(self):
        c = self.conv
        n = c.kernel_size[0] * c.kernel_size[1] * c.in_channels
        nn.init.normal_(c.weight, 0, math.sqrt(2. / n))
        if c.bias is not None:
            nn.init.zeros_(c.bias)
        if self.normalization in ('batch', 'instance'):
            nn.init.ones_(self.norm.weight)
            nn.init.zeros_(self.norm.bias)

    def _sync_norm(self, x):
        """A train step under data-parallel training (train_ops.EXCHANGE installed) of a layer the
        train kernels do not cover (the decoder's 3x3 convolutions below train_ops.UPCONV_MIN_HW):
        its BatchNorm and activation still run on train_ops.norm_act_train, which synchronises the
        statistics over the ranks. Single-process training keeps the PyTorch composition."""
        return (train_ops.EXCHANGE is not None and self.normalization == 'batch' and self.training
                and torch.is_grad_enabled() and x.is_cuda and x.dtype == torch.float32
                and x.dim() == 4 and self.activation in KERNEL_ACTIVATIONS)

    def forward(self, x, epoch=None, tf32=False):
        """tf32: a cuDNN convolution of a train step may round to TF32 (UpConv's 3x3 convolution
        below train_ops.UPCONV_MIN_HW under SONET_TRAIN_TC=fp16); otherwise it is strict fp32."""
        if _fast_ok(self, x) and x.dim() == 4 and self._fast_eligible():
            B, C, H, W = x.shape
            y = self.forward_points(x.contiguous().view(B, C, H * W))
            return y.view(B, y.shape[1], H, W)
        if x.dim() == 4 and self._train_kernels(x):
            B, C, H, W = x.shape
            y = train_ops.conv_bn_act_train(
                x.contiguous().view(B, C, H * W), self._conv_weight2d(), self.conv.bias,
                self._train_norm(), self.activation, epoch)
            return y.view(B, y.shape[1], H, W)
        # PyTorch/cuDNN path (3x3 decoder convs, training): strict fp32 in the forward and the
        # backward — cuDNN's default TF32 convolution is ~1e-3 relative, outside the 1e-4 parity
        # bar of the reference's fp32 math
        x = train_ops.conv_tf32(self.conv, x) if tf32 else train_ops.conv_strict(self.conv, x)
        if self._sync_norm(x):
            B, C, H, W = x.shape
            y = train_ops.norm_act_train(x.reshape(B, C, H * W), self.norm, self.activation, epoch)
            return y.view(B, C, H, W)
        if self.normalization == 'batch':
            x = self.norm(x, epoch)
        elif self.normalization is not None:
            x = self.norm(x)
        if self.activation is not None:
            x = self.act(x)
        return x


class UpConv(nn.Module):
    """Nearest x2 upsample + 3x3 conv + BN + act (models/layers.py:214-240), the decoder's
    building block. Eval fast path (SURVEY.md §8f-1): four parity GEMMs over the LOW-resolution
    map on wgmma (csrc/upconv.cu, csrc/pointwise_tc.cu) — the up-sampled image is never built
    and the 3x3 taps that coincide after up-sampling are pre-summed (K = 4*Cin, not 9*Cin)."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=0,
                 output_padding=0, bias=True, activation=None, normalization=None):
        super().__init__()
        self.activation = activation
        self.normalization = normalization
        self.up_sample = nn.Upsample(scale_factor=2)
        self.conv = MyConv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1,
                             bias=True, activation=activation, normalization=normalization)
        self._tc = _Cache()
        self._scratch = {}
        self.weight_init()

    def weight_init(self):
        c = self.conv.conv
        n = c.kernel_size[0] * c.kernel_size[1] * c.out_channels
        nn.init.normal_(c.weight, 0, math.sqrt(2. / n))
        if c.bias is not None:
            nn.init.constant_(c.bias, 0.001)

    def _kernel_eligible(self, x):
        """The parity-GEMM kernels apply: a 4-D input, 3x3 / stride 1 / pad 1 / dilation 1, one
        group, Cin >= 16, Cout >= 64, and a norm and activation the kernels have."""
        c = self.conv.conv
        return (x.dim() == 4 and c.kernel_size == (3, 3)
                and c.stride == (1, 1) and c.padding == (1, 1) and c.dilation == (1, 1)
                and c.groups == 1 and c.out_channels >= 64 and c.in_channels >= 16
                and _norm_on_kernels(self.normalization, getattr(self.conv, "norm", None))
                and self.activation in KERNEL_ACTIVATIONS)

    # ---- eval fast path --------------------------------------------------------------------------
    def _fast(self, x):
        return _fast_ok(self, x) and self._kernel_eligible(x) and tc_enabled()

    def _train_kernels(self, x):
        """train() mode on CUDA fp32, input maps of at least train_ops.UPCONV_MIN_HW pixels: the
        parity GEMMs' forward, dgrad and wgrad (train_ops.upconv_train), then the shared norm /
        activation kernels. SONET_TC is ignored."""
        return (train_ops.ENABLED and self.training and torch.is_grad_enabled() and x.is_cuda
                and x.dtype == torch.float32 and self._kernel_eligible(x)
                and x.shape[2] * x.shape[3] >= train_ops.UPCONV_MIN_HW
                and (self.normalization != 'instance' or self.conv.norm.affine))

    def _packed(self):
        """BN-folded, parity-combined weights as wgmma blobs; re-packed when the fold changes.
        Wg[g=(py,px)][co][(a,c)*Cin + ci] = sum of the 3x3 taps (dy,dx) that read low-res
        neighbour (a,c) for output parity (py,px): rows {0}|{1,2} (py=0) or {0,1}|{2} (py=1)."""
        w, shift = self.conv.folded()                                      # [Cout,Cin*9]

        def build():
            Cout, Cin = self.conv.conv.out_channels, self.conv.conv.in_channels
            w4 = w.view(Cout, Cin, 3, 3)
            sets = (((0,), (1, 2)), ((0, 1), (2,)))    # [parity][tap] -> kernel rows
            Wg = torch.zeros(4, Cout, 4, Cin, device=w.device)
            for py in range(2):
                for px in range(2):
                    for a in range(2):
                        for cc in range(2):
                            acc = 0
                            for dy in sets[py][a]:
                                for dx in sets[px][cc]:
                                    acc = acc + w4[:, :, dy, dx]
                            Wg[py * 2 + px, :, a * 2 + cc, :] = acc
            blob4, per4, inv4 = ops.pointwise_tc_pack_groups(Wg.view(4, Cout, 4 * Cin))
            # 1x1 input: only the tap that lands on the single pixel survives -> one dense
            # layer Cin -> 4*Cout (output channel co*4 + py*2 + px)
            W1 = torch.stack([Wg[g, :, (1 - (g >> 1)) * 2 + (1 - (g & 1)), :] for g in range(4)],
                             dim=1).reshape(1, Cout * 4, Cin)
            blob1, per1, inv1 = ops.pointwise_tc_pack_groups(W1)
            return dict(blob4=blob4.to(w.device), per4=per4, inv4=inv4, blob1=blob1.to(w.device),
                        per1=per1, inv1=inv1, shift=shift,
                        shift1=shift.repeat_interleave(4).contiguous())
        return self._tc.get(self.conv._folded.version, build)

    def _scratch_for(self, n, dev):
        buf = self._scratch.get(dev)
        if buf is None or buf.numel() < n:
            buf = self._scratch[dev] = torch.empty(n, dtype=torch.float32, device=dev)
        return buf

    def forward(self, x):
        if not self._fast(x):
            if self._train_kernels(x):
                c = self.conv.conv
                z = train_ops.upconv_train(x, c.weight, c.bias)           # [B, Cout, 2H, 2W]
                B, Cout, H2, W2 = z.shape
                y = train_ops.norm_act_train(z.view(B, Cout, H2 * W2), self.conv._train_norm(),
                                             self.activation)
                return y.view(B, Cout, H2, W2)
            # the decoder's maps below UPCONV_MIN_HW: SONET_TRAIN_TC=fp16 gives up fp32 parity in
            # their cuDNN convolutions too and allows TF32, the reference's default
            tf32 = (train_ops.ENABLED and self.training and torch.is_grad_enabled() and x.is_cuda
                    and train_ops.train_f16())
            return self.conv(self.up_sample(x), tf32=tf32)
        pk = self._packed()
        f16 = tc_f16()
        B, Cin, H, W = x.shape
        Cout = self.conv.conv.out_channels
        # instance norm: the parity GEMMs write z (conv bias, no activation), then each [2H x 2W]
        # map is normalised
        inst = self.normalization == 'instance'
        act = None if inst else self.activation
        x = x.contiguous()
        if H == 1 and W == 1:
            kch = (Cin + 63) // 64
            splits = ops.pick_splits(kch, ((B + 127) // 128) * ((4 * Cout + 255) // 256))
            scratch = self._scratch_for(splits * B * 4 * Cout, x.device) if splits > 1 else None
            y = ops.pointwise_tc_grouped(x.view(B, Cin, 1), pk["blob1"], pk["per1"], pk["inv1"],
                                         pk["shift1"], 4 * Cout, act, groups=1, splits=splits,
                                         scratch=scratch, f16=f16)
            if inst:     # output channel co*4 + py*2 + px: [B, Cout, 4] rows of the 2x2 maps
                y = self.conv.instance_norm(y.view(B, Cout, 4))
            return y.view(B, Cout, 2, 2)
        P = H * W
        kch = (4 * Cin + 63) // 64
        splits = ops.pick_splits(kch, 4 * ((B * P + 127) // 128) * ((Cout + 255) // 256))
        scratch = self._scratch_for(4 * splits * B * Cout * P, x.device) if splits > 1 else None
        # H*W % 64 == 0 and Cin % 64 == 0: no im2col — three horizontally shifted copies, the
        # vertical shifts are point-coordinate offsets inside the GEMM (3x the input instead of 16x)
        conv = ops.upconv_conv_mode(Cin, H, W)
        xin = ops.upconv_hshift(x) if conv else ops.upconv_im2col(x)      # [3B,Cin,HW] | [4B,4Cin,HW]
        y = ops.pointwise_tc_grouped(xin, pk["blob4"], pk["per4"], pk["inv4"], pk["shift"], Cout,
                                     act, groups=4, splits=splits, scat_w=W, scratch=scratch,
                                     conv=conv, f16=f16)
        if inst:
            y = self.conv.instance_norm(y)                                  # [B, Cout, 4HW]
        return y.view(B, Cout, 2 * H, 2 * W)


class EquivariantLayer(_PointwiseConvBase):
    """Conv1d(k=1) + BN1d + act on [B,C,P] (models/layers.py:243-296)."""

    def __init__(self, num_in_channels, num_out_channels, activation='relu', normalization=None,
                 momentum=0.1, bn_momentum_decay_step=None, bn_momentum_decay=1):
        super().__init__()
        self.num_in_channels = num_in_channels
        self.num_out_channels = num_out_channels
        self.activation = activation
        self.normalization = normalization
        self.conv = nn.Conv1d(num_in_channels, num_out_channels, kernel_size=1, stride=1,
                              padding=0)
        if normalization == 'batch':
            self.norm = MyBatchNorm1d(num_out_channels, momentum=momentum, affine=True,
                                      momentum_decay_step=bn_momentum_decay_step,
                                      momentum_decay=bn_momentum_decay)
        elif normalization == 'instance':
            self.norm = nn.InstanceNorm1d(num_out_channels, momentum=momentum, affine=True)
        act = _make_act(activation)
        if act is not None:
            self.act = act
        self.weight_init()

    def weight_init(self):
        nn.init.normal_(self.conv.weight, 0,
                        math.sqrt(2. / (self.conv.kernel_size[0] * self.conv.in_channels)))
        if self.conv.bias is not None:
            nn.init.zeros_(self.conv.bias)
        if self.normalization in ('batch', 'instance'):
            nn.init.ones_(self.norm.weight)
            nn.init.zeros_(self.norm.bias)

    def fast(self, *tensors):
        return _fast_ok(self, *tensors) and self._fast_eligible()

    def forward(self, x, epoch=None, route_rows=None):
        """route_rows: as forward_points (eval fast path only)."""
        if self.fast(x) and x.dim() == 3:
            return self.forward_points(x.contiguous(), route_rows=route_rows)
        if self._train_kernels(x) and x.dim() == 3:
            return train_ops.conv_bn_act_train(
                x, self._conv_weight2d(), self.conv.bias, self._train_norm(), self.activation,
                epoch)
        y = self.conv(x)
        if self.normalization == 'batch':
            y = self.norm(y, epoch)
        elif self.normalization is not None:
            y = self.norm(y)
        if self.activation is not None:
            y = self.act(y)
        return y


class KNNModule(nn.Module):
    """Group K neighbour nodes, decentre, 1x1-conv stack, max over K (models/layers.py:299-367)."""

    def __init__(self, in_channels, out_channels_list, activation, normalization, momentum=0.1,
                 bn_momentum_decay_step=None, bn_momentum_decay=1):
        super().__init__()
        self.layers = nn.ModuleList()
        prev = in_channels
        for c_out in out_channels_list:
            self.layers.append(MyConv2d(prev, c_out, kernel_size=1, stride=1, padding=0, bias=True,
                                        activation=activation, normalization=normalization,
                                        momentum=momentum,
                                        bn_momentum_decay_step=bn_momentum_decay_step,
                                        bn_momentum_decay=bn_momentum_decay))
            prev = c_out
        self._tc = _Cache()

    def _fast(self, coordinate, x, precomputed_knn_I, center_type):
        return (_fast_ok(self, coordinate, x) and center_type in ('avg', 'center')
                and all(l._fast_eligible() for l in self.layers)
                and (precomputed_knn_I is None or precomputed_knn_I.is_cuda))

    # ---- fused wgmma path (csrc/knn_tc.cu) ----------------------------------------------------
    def _tc_fused(self, K, M):
        """Two BN/ReLU or BN/ELU layers 3+C -> 512 -> 512 (the encoder's), 2 <= K <= 16,
        M*K <= 2304."""
        ls = self.layers
        return (tc_enabled() and len(ls) == 2
                and ls[0].conv.in_channels >= 3 + 32
                and all(l.conv.out_channels == 512 for l in ls)
                and all(l.normalization in (None, 'batch') for l in ls)   # folds into the GEMMs
                and ls[0].activation in ('relu', 'elu') and ls[1].activation == ls[0].activation
                and 2 <= K <= 16 and M * K <= 2304)

    def _tc_params(self):
        """Layer 1 split by linearity into the per-node GEMM of its feature columns (a generic
        wgmma blob) and (W1d | shift1) [512,4]; layer 2 as the fused kernel's weight stream.
        Re-packed only when a fold changes."""
        (w1, s1), (w2, s2) = [l.folded() for l in self.layers]

        def build():
            yblob, yinv = ops.pointwise_tc_pack(w1[:, 3:])
            blob2, inv2 = ops.knn_mlp_tc_pack(w2)
            return dict(yblob=yblob.to(w1.device), yinv=yinv,
                        w1=torch.cat((w1[:, :3], s1[:, None]), dim=1).contiguous(),
                        blob2=blob2.to(w1.device), inv2=inv2, shift2=s2)
        return self._tc.get(tuple(l._folded.version for l in self.layers), build)

    def _tc_forward(self, coord, center, knn_I, K, x):
        """x [B,C,M] -> knn_feature [B,512,M]: Y = W1f x once per node, stored node-major so the
        fused kernel gathers each neighbour's channels as contiguous pairs, then one fused launch."""
        pk = self._tc_params()
        f16 = tc_f16()
        y = ops.pointwise_layer_tc(x, pk["yblob"], pk["yinv"], None, 512, False, rows=True, f16=f16)
        return ops.knn_mlp_tc(coord, center, knn_I, K, y.transpose(1, 2), pk["w1"], pk["blob2"],
                              pk["inv2"], pk["shift2"], f16=f16, act=self.layers[0].activation)

    def forward_pooled(self, coordinate, pool, precomputed_knn_I, K, center_type, epoch=None,
                       owner=None):
        """forward() for the fused-pool path: `pool` = (keys [B,C,M] i32, p0 [B,C]) as left by
        ops.pointresnet_tc_pool(finalize=False). Returns (center, feature, masked_max [B,C,M]) or
        None when this module cannot take the fused route (the caller then finalizes the pool)."""
        keys, p0 = pool
        B, C, M = keys.shape
        if not (self._fast(coordinate, p0, precomputed_knn_I, center_type)
                and M <= 256 and M * K <= 2304):
            return None
        coord = coordinate.detach().contiguous()
        if precomputed_knn_I is not None:
            if precomputed_knn_I.size()[2] < K:
                return None      # the unfused forward() raises the reference's assertion
            knn_I = precomputed_knn_I.contiguous()
        else:
            knn_I = ops.node_knn(coord, K)
        if self._tc_fused(K, M):
            center, _, masked_max = ops.knn_assemble_pool(coord, keys, p0, knn_I, K, center_type,
                                                          owner=owner, want_x_aug=False)
            return center, self._tc_forward(coord, center, knn_I, K, masked_max), masked_max
        center, h, masked_max = ops.knn_assemble_pool(coord, keys, p0, knn_I, K, center_type,
                                                      owner=owner)
        return center, self._layers_max(h, B, M, K), masked_max

    def _layers_max(self, h, B, M, K):
        """The 1x1-conv stack on x_aug [B,3+C,M*K] and the max over each node's K neighbours.
        An instance-norm last layer takes the max inside its normalisation pass."""
        last = self.layers[-1]
        for layer in self.layers[:-1]:
            h = layer.forward_points(h)                     # [B, C', M*K]
        if last.normalization == 'instance':
            return last.forward_points(h, group_max=K)
        h = last.forward_points(h)
        return ops.rowmax(h.view(B, h.shape[1], M, K))      # max over K

    def forward(self, coordinate, x, precomputed_knn_I, K, center_type, epoch=None):
        """coordinate [B,3,M], x [B,C,M], precomputed_knn_I [B,M,K'] -> (center [B,3,M],
        feature [B,Cout,M])."""
        if self._fast(coordinate, x, precomputed_knn_I, center_type):
            coord = coordinate.detach().contiguous()
            if precomputed_knn_I is not None:
                assert precomputed_knn_I.size()[2] >= K
                knn_I = precomputed_knn_I.contiguous()  # kernel reads the first K columns
            else:
                knn_I = ops.node_knn(coord, K)
            B, C, M = x.shape
            if self._tc_fused(K, M):
                center, _ = ops.knn_assemble(coord, x.contiguous(), knn_I, K, center_type,
                                             want_x_aug=False)
                return center, self._tc_forward(coord, center, knn_I, K, x.contiguous())
            center, h = ops.knn_assemble(coord, x.contiguous(), knn_I, K, center_type)
            return center, self._layers_max(h, B, M, K)

        coordinate_tensor = coordinate.data
        if precomputed_knn_I is not None:
            assert precomputed_knn_I.size()[2] >= K
            knn_I = precomputed_knn_I[:, :, 0:K]
        else:
            d = torch.sum((coordinate_tensor.unsqueeze(3) - coordinate_tensor.unsqueeze(2)) ** 2,
                          dim=1)
            _, knn_I = torch.topk(d, k=K, dim=2, largest=False, sorted=True)
        neighbors = operations.knn_gather_wrapper(coordinate_tensor, knn_I)  # Bx3xMxK
        if center_type == 'avg':
            neighbors_center = torch.mean(neighbors, dim=3, keepdim=True)
        elif center_type == 'center':
            neighbors_center = coordinate_tensor.unsqueeze(3)
        neighbors_decentered = (neighbors - neighbors_center).detach()
        neighbors_center = neighbors_center.squeeze(3).detach()
        x_neighbors = operations.knn_gather_by_indexing(x, knn_I)
        x_augmented = torch.cat((neighbors_decentered, x_neighbors), dim=1)
        for layer in self.layers:
            x_augmented = layer(x_augmented, epoch)
        feature, _ = torch.max(x_augmented, dim=3, keepdim=False)
        return neighbors_center, feature


def _chain(in_channels, out_channels_list, activation, normalization, momentum,
           bn_momentum_decay_step, bn_momentum_decay, last_extra_in=0):
    layers = nn.ModuleList()
    prev = in_channels
    last = len(out_channels_list) - 1
    for i, c_out in enumerate(out_channels_list):
        if i != last:
            layers.append(EquivariantLayer(prev, c_out, activation, normalization, momentum,
                                           bn_momentum_decay_step, bn_momentum_decay))
        else:
            layers.append(EquivariantLayer(prev + last_extra_in, c_out, None, None))
        prev = c_out
    return layers


class PointNet(nn.Module):
    """Chain of EquivariantLayers, last one bare (models/layers.py:370-387)."""

    def __init__(self, in_channels, out_channels_list, activation, normalization, momentum=0.1,
                 bn_momentum_decay_step=None, bn_momentum_decay=1):
        super().__init__()
        self.layers = _chain(in_channels, out_channels_list, activation, normalization, momentum,
                             bn_momentum_decay_step, bn_momentum_decay)
        self._node_images = ops.NodeImages()

    def forward(self, x, epoch=None):
        for layer in self.layers:
            x = layer(x, epoch)
        return x

    def _node_route(self, x0, x1):
        """The eval fast path runs on ops.nodegemm_pointnet: two layers, both dense enough for
        wgmma (forward_points' rule), BatchNorm + ReLU / ELU then the bare last layer, over at
        most ops.NODEGEMM_MAX_ROWS rows (the encoder's node-level final PointNet)."""
        if len(self.layers) != 2 or x0.dim() != 3 or not tc_enabled():
            return False
        l1, l2 = self.layers
        rows = x0.shape[0] * x0.shape[2]
        return (l1.fast(x0, x1) and l2.fast(x0)
                and l1.normalization == 'batch' and l1.activation in ('relu', 'elu')
                and l2.normalization is None and l2.activation is None
                and x0.shape[1] + x1.shape[1] >= 32 and l1.conv.out_channels >= 32
                and 256 <= rows <= ops.NODEGEMM_MAX_ROWS)

    def forward_pair(self, x0, x1, epoch=None):
        """forward(torch.cat((x0, x1), dim=1)) without materialising the concat in eval mode."""
        first = self.layers[0]
        if self._node_route(x0, x1):
            l1, l2 = self.layers
            return ops.nodegemm_pointnet(x0.contiguous(), x1.contiguous(), l1._tc_params(),
                                         l1.conv.out_channels, l1.activation, l2._tc_params(),
                                         l2.conv.out_channels, f16=tc_f16(),
                                         owner=self._node_images)
        if first.fast(x0, x1):
            x = first.forward_points(x0.contiguous(), x1.contiguous())
            for layer in self.layers[1:]:
                x = layer(x, epoch)
            return x
        return self.forward(torch.cat((x0, x1), dim=1), epoch)


class PointResNet(nn.Module):
    """in -> out[0] -> ... -> out[k-2]; cat(out[0], out[k-2]) -> out[k-1] (models/layers.py:390-432)."""

    def __init__(self, in_channels, out_channels_list, activation, normalization, momentum=0.1,
                 bn_momentum_decay_step=None, bn_momentum_decay=1):
        super().__init__()
        self.out_channels_list = out_channels_list
        self.layers = _chain(in_channels, out_channels_list, activation, normalization, momentum,
                             bn_momentum_decay_step, bn_momentum_decay,
                             last_extra_in=out_channels_list[0])
        self._tc = _Cache()

    # ---- fused wgmma path (csrc/pointmlp_tc.cu): the encoder's first PointResNet -------------
    def _tc_eligible(self, cin, x1):
        if x1 is not None or not tc_enabled():
            return False
        if list(self.out_channels_list) != [64, 128, 256, 384] or cin > 6:
            return False
        ls = self.layers
        return (all(l.normalization == 'batch' for l in ls[:3])
                and ls[0].activation in ('relu', 'elu')
                and all(l.activation == ls[0].activation for l in ls[:3])
                and ls[3].normalization is None and ls[3].activation is None)

    def _tc_params(self):
        """(blob, fparams) on the weights' device, re-packed only when a fold changes."""
        ws, shifts = zip(*[l.folded() for l in self.layers])

        def build():
            blob, fpar = ops.pointresnet_tc_pack(ws, shifts, ws[0].shape[1])
            return blob.to(ws[0].device), fpar.to(ws[0].device)
        return self._tc.get(tuple(l._folded.version for l in self.layers), build)

    def forward(self, x, epoch=None, x1=None, route_rows=None):
        """x [B,C,P]; x1: optional second tensor virtually concatenated to x (eval fast path);
        route_rows: as EquivariantLayer.forward_points (the fused kernel has one route)."""
        n = len(self.out_channels_list)
        first, last = self.layers[0], self.layers[n - 1]
        if first.fast(x) and x.dim() == 3 and all(l.fast(x) for l in self.layers) \
                and self._tc_eligible(x.shape[1], x1):
            blob, fpar = self._tc_params()
            return ops.pointresnet_tc(x.contiguous(), blob, fpar, f16=tc_f16(),
                                      act=self.layers[0].activation)
        if first.fast(x) and x.dim() == 3 and all(l.fast(x) for l in self.layers):
            layer0_out = first.forward_points(x.contiguous(),
                                              None if x1 is None else x1.contiguous(),
                                              route_rows=route_rows)
            x_tmp = layer0_out
            for l in range(1, n - 1):
                x_tmp = self.layers[l].forward_points(x_tmp, route_rows=route_rows)
            # the skip-concat, never materialised
            return last.forward_points(layer0_out, x_tmp, route_rows=route_rows)
        if x1 is not None:
            x = torch.cat((x, x1), dim=1)
        layer0_out = first(x, epoch)
        x_tmp = layer0_out
        for l in range(1, n - 1):
            x_tmp = self.layers[l](x_tmp, epoch)
        return last(torch.cat((layer0_out, x_tmp), dim=1), epoch)
