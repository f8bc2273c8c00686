"""Train-mode building blocks on the sm_90a kernels (SURVEY.md §8f-2, csrc/train.cu): autograd
Functions that the layer classes use in train() mode instead of the PyTorch composition
conv1d -> batch_norm(training=True) -> relu / elu and gather (models/layers.py:22-70, 282-296;
models/networks.py:185).

    ConvTC        y = W x + b, dx = W^T dy AND dW = dy x^T on the generic wgmma layer kernel
                  (weights / activations packed on the device each step; gradients pre-scaled by a
                  power of two before the fp16 hi/lo split)
    BNActTrain    batch-statistics BatchNorm + ReLU / ELU / none, forward and backward, fused elementwise passes
                  and deterministic reductions through per-cloud records, which EXCHANGE
                  (data-parallel training) synchronises over the ranks
    InstanceNormActTrain  instance norm + ReLU / ELU / none: the instance-norm kernel forward, the
                  BatchNorm backward on the [1, B*C, P] view
    UpConvTC      nearest x2 up-sampling + 3x3 conv (pad 1) as four parity GEMMs over the
                  low-resolution map (csrc/upconv.cu): forward, dgrad (one GEMM with K = 16*Cout over
                  the gathered gradient D) and wgrad (one GEMM per parity) on the wgmma layer kernel
    LinearStrict  x W^T + b on cuBLAS with TF32 off in the forward and the backward (MyLinear)
    IndexMaxGather  first_pn_out_masked_max = first_pn_out.gather(2, idx * mask_row_max) with the
                  arg-max kernel in the forward and a deterministic scatter in the backward

norm_act_train is the norm / activation half every train-mode layer shares. ENABLED = False
switches every layer back to the PyTorch composition (the tests compare the two). train_f16()
(SONET_TRAIN_TC=fp16) runs ConvTC's and UpConvTC's GEMMs as one fp16 product per MAC.
"""
import contextlib
import os

import torch
import torch.nn.functional as F
from torch.nn.modules.instancenorm import _InstanceNorm

from . import _C, ops

ENABLED = True


def train_f16():
    """True under SONET_TRAIN_TC=fp16: the train-mode wgmma GEMMs (ConvTC's and UpConvTC's forward,
    dgrad and wgrad) run as one fp16 product per MAC on the `_f16` twins of their entries, each
    operand pre-scaled by a power of two first, and the decoder's cuDNN convolutions below
    UPCONV_MIN_HW run with TF32 allowed. Read when a layer's forward runs, so a change applies from
    the next train step on; its backward keeps the forward's mode. Unset or any other value: the
    fp16 hi/lo split. Eval mode ignores it (SONET_TC is eval's switch)."""
    return os.environ.get("SONET_TRAIN_TC") == "fp16"


def _f16(name, f16):
    """The C-ABI entry `name`, or with f16 its one-product twin (`_f32` becomes `_f16`)."""
    if not f16:
        return name
    return (name[:-4] if name.endswith("_f32") else name) + "_f16"


def _scratch(dev, n, dtype, cache):
    key = (dev, dtype)
    buf = cache.get(key)
    if buf is None or buf.numel() < n:
        buf = cache[key] = torch.empty(max(n, 1), dtype=dtype, device=dev)
    return buf


def scratch_buffers():
    """Every scratch buffer the train ops hold now. A captured CUDA graph keeps these alive: a
    larger step replaces a buffer in its cache, and the graph must not write into freed memory."""
    return [b for c in _WGRAD_CACHE.values() for b in c.values()]


# The BatchNorm exchange of data-parallel training (dist.DataParallelTraining), or None. BNActTrain
# writes the records of the local clouds, gathers them along the cloud axis by exchange.gather(rec)
# -> [Bg, C, k] in global cloud order, then folds them in that order. exchange.global_rows(B) is the
# global batch Bg of a local batch of B clouds. With none installed BNActTrain uses _LOCAL.
EXCHANGE = None


class _LocalExchange:
    """One process's batch is the whole batch."""

    @staticmethod
    def global_rows(B):
        return B

    @staticmethod
    def gather(rec):
        return rec


_LOCAL = _LocalExchange()


def _exchange():
    return _LOCAL if EXCHANGE is None else EXCHANGE


def _bn_backward(dy, x, mean, invstd, gamma, beta, B, C, P, act, ex, dx, dgamma, dbeta):
    """The BatchNorm backward of x [B,C,P] (contiguous, like dy and dx) into dx, dgamma, dbeta: the
    records of the B local clouds, gathered by the exchange ex and folded over its global batch."""
    rec = torch.empty((B, C, _C.CONSTANTS["SONET_BN_REC_BWD"]), dtype=torch.float64, device=x.device)
    ops._call("sonet_bn_cloud_partials_f32", _C.ptr(x), _C.ptr(dy), _C.ptr(mean), _C.ptr(invstd),
              _C.ptr(gamma), _C.ptr(beta), B, C, P, act, 1, _C.ptr(rec), ops._stream(x))
    rec = ex.gather(rec)
    ops._call("sonet_bn_sync_backward_f32", _C.ptr(rec), _C.ptr(dy), _C.ptr(x), _C.ptr(mean),
              _C.ptr(invstd), _C.ptr(gamma), _C.ptr(beta), ex.global_rows(B), B, C, P, act,
              _C.ptr(dx), _C.ptr(dgamma), _C.ptr(dbeta), ops._stream(x), kernels=2)


class BNActTrain(torch.autograd.Function):
    """Batch-statistics BatchNorm + activation of x [B,C,P] through the per-cloud records
    (sonet_bn_cloud_partials_f32, then sonet_bn_sync_forward_f32 / _backward_f32). The backward's
    dy is the gradient of this process's loss, a mean over its B clouds. The exchange works in
    units of the global-batch loss, whose gradient here is dy * B / Bg: dgamma and dbeta come out
    as the global gradients, the same on every rank, and dx goes back to this rank's units.

    cols (device int64 [B+1]): x is a ragged batch's [1,C,L] layer output whose cloud b owns the
    columns cols[b] .. cols[b+1]; the records are per (cloud, channel) over those columns and the
    statistics cover all L columns (sonet_bn_cloud_partials_ragged_f32, sonet_bn_ragged_*_f32).
    Single-process only."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps, act, cols=None):
        x = x.contiguous()
        ctx.cols = cols
        if cols is not None:
            ctx.act = ops.act_code(act)
            rec = ops.bn_cloud_partials_ragged(x, cols)
            y, mean, var, invstd = ops.bn_ragged_forward(rec, cols, x, gamma, beta, eps, ctx.act)
            ctx.save_for_backward(x, mean, invstd, gamma, beta)
            ctx.mark_non_differentiable(mean, var)
            return y, mean, var
        B, C, P = x.shape
        dev = x.device
        ex = ctx.exchange = _exchange()
        ctx.act = ops.act_code(act)
        with torch.cuda.device(dev):
            y = torch.empty_like(x)
            mean = torch.empty(C, dtype=torch.float32, device=dev)
            var = torch.empty(C, dtype=torch.float32, device=dev)
            invstd = torch.empty(C, dtype=torch.float32, device=dev)
            rec = torch.empty((B, C, _C.CONSTANTS["SONET_BN_REC_FWD"]), dtype=torch.float64, device=dev)
            ops._call("sonet_bn_cloud_partials_f32", _C.ptr(x), None, None, None, None, None, B, C, P,
                      ctx.act, 0, _C.ptr(rec), ops._stream(x))
            rec = ex.gather(rec)
            ops._call("sonet_bn_sync_forward_f32", _C.ptr(rec), _C.ptr(x), _C.ptr(gamma), _C.ptr(beta),
                      ex.global_rows(B), B, C, P, float(eps), ctx.act, _C.ptr(y), _C.ptr(mean),
                      _C.ptr(var), _C.ptr(invstd), ops._stream(x), kernels=2)
        ctx.save_for_backward(x, mean, invstd, gamma, beta)
        ctx.mark_non_differentiable(mean, var)
        return y, mean, var

    @staticmethod
    def backward(ctx, dy, _dm, _dv):
        x, mean, invstd, gamma, beta = ctx.saved_tensors
        dy = dy.contiguous()
        if ctx.cols is not None:
            rec = ops.bn_cloud_partials_ragged(x, ctx.cols, ctx.act, dy, mean, invstd, gamma, beta)
            dx, dgamma, dbeta = ops.bn_ragged_backward(rec, ctx.cols, dy, x, mean, invstd, gamma, beta,
                                                       ctx.act)
            return dx, dgamma, dbeta, None, None, None
        B, C, P = x.shape
        dev = x.device
        share = B / ctx.exchange.global_rows(B)
        if share != 1.0:
            dy = dy * share
        with torch.cuda.device(dev):
            dx = torch.empty_like(x)
            dgamma = torch.empty(C, dtype=torch.float32, device=dev)
            dbeta = torch.empty(C, dtype=torch.float32, device=dev)
            _bn_backward(dy, x, mean, invstd, gamma, beta, B, C, P, ctx.act, ctx.exchange, dx, dgamma,
                         dbeta)
        if share != 1.0:
            dx.div_(share)
        return dx, dgamma, dbeta, None, None, None


class InstanceNormActTrain(torch.autograd.Function):
    """Instance norm (affine, no running statistics) + ReLU / ELU / none of z [B,C,P]. Forward:
    the instance-norm kernel, keeping each row's mean and invstd. Backward: the BatchNorm backward
    of one cloud on the [1, B*C, P] view, whose per-channel statistics are exactly the per-row
    ones, with gamma and beta expanded to [B*C]; dgamma and dbeta are then summed over the clouds
    in fp64."""

    @staticmethod
    def forward(ctx, z, gamma, beta, eps, act):
        z = z.contiguous()
        y, mean, invstd = ops.instance_norm(z, gamma.detach(), beta.detach(), eps, act,
                                            save_stats=True)
        ctx.save_for_backward(z, mean, invstd, gamma, beta)
        ctx.act = ops.act_code(act)
        return y

    @staticmethod
    def backward(ctx, dy):
        z, mean, invstd, gamma, beta = ctx.saved_tensors
        dy = dy.contiguous()
        B, C, P = z.shape
        dev = z.device
        # the entries take at most 65535 channels: whole clouds per call
        cb = max(1, 65535 // C)
        with torch.cuda.device(dev):
            dz = torch.empty_like(z)
            g_rows = gamma.detach().repeat(cb).contiguous()
            b_rows = beta.detach().repeat(cb).contiguous()
            dgamma = torch.empty((B, C), dtype=torch.float32, device=dev)
            dbeta = torch.empty((B, C), dtype=torch.float32, device=dev)
            for b0 in range(0, B, cb):
                n = min(cb, B - b0)
                _bn_backward(dy[b0:b0 + n], z[b0:b0 + n], mean[b0:b0 + n], invstd[b0:b0 + n], g_rows,
                             b_rows, 1, n * C, P, ctx.act, _LOCAL, dz[b0:b0 + n], dgamma[b0:b0 + n],
                             dbeta[b0:b0 + n])
        return (dz, dgamma.double().sum(0).float(), dbeta.double().sum(0).float(), None, None)


def _pack_device(W, transpose):
    """W [Cout,Cin] (device) -> (blob, scale2) for the wgmma layer; W^T when transpose."""
    Cout, Cin = W.shape
    n, k = (Cin, Cout) if transpose else (Cout, Cin)
    dev = W.device
    with torch.cuda.device(dev):
        blob = torch.empty(int(_C.lib().sonet_pointwise_tc_blob_bytes(n, k)), dtype=torch.uint8,
                           device=dev)
        scale2 = torch.empty(2, dtype=torch.float32, device=dev)
        bits = torch.empty(1, dtype=torch.int32, device=dev)
        ops._call("sonet_pointwise_tc_pack_device", _C.ptr(W), Cout, Cin, int(transpose),
                  _C.ptr(blob), _C.ptr(scale2), _C.ptr(bits), ops._stream(W), kernels=3)
    return blob, scale2


def _absmax_scale(t):
    """(scale, 1/scale) device tensor: the power of two that puts max|t| into [256,512) — gradients
    are far below fp16's normal range, so they are pre-scaled before the fp16 hi/lo split."""
    dev = t.device
    with torch.cuda.device(dev):
        scale2 = torch.empty(2, dtype=torch.float32, device=dev)
        bits = torch.empty(1, dtype=torch.int32, device=dev)
        ops._call("sonet_absmax_scale_f32", _C.ptr(t), t.numel(), _C.ptr(scale2), _C.ptr(bits),
                  ops._stream(t), kernels=2)
    return scale2


def _forward_scale(x):
    """_absmax_scale of a forward activation, except that an infinite max gives 1 instead of NaN:
    the forward keeps the split's saturation rule (an infinite activation acts as the largest fp16)
    instead of making its outputs NaN."""
    return torch.nan_to_num(_absmax_scale(x), nan=1.0)


def _forward_scales(scale2, x):
    """(inv, act) of an fp16-mode forward with weight scales scale2 = (s_w, 1/s_w): act = s_x of
    _forward_scale(x), inv = 1/(s_w s_x) folded into one fp32 power of two. The fold underflows to
    0 when s_w s_x > 2^149, i.e. max|W| max|x| below about 2^-131 (both pre-scales near their 2^126
    cap): the products, all of them then below fp32's normal range, are lost and y is the bias."""
    s_x = _forward_scale(x)
    return scale2[1:] * s_x[1:], s_x[:1]


def _tc_dev(x, blob, inv, shift, cout, act_scale=None, f16=False):
    """Generic wgmma layer with a device-packed blob: inv (1-element device tensor) = the total
    inverse pre-scale, act_scale (1-element) = activation pre-scale or None; f16: the
    one-product twin."""
    B, C, P = x.shape
    with torch.cuda.device(x.device):
        out = torch.empty((B, cout, P), dtype=torch.float32, device=x.device)
        ops._call(_f16("sonet_pointwise_tc_forward_dev", f16), _C.ptr(x), C, B, P, _C.ptr(blob),
                  _C.ptr(inv), _C.ptr(act_scale), _C.ptr(shift), int(cout), 0, 1, _C.ptr(out), None,
                  ops._stream(x))
    return out


def tc_eligible(cin, cout, rows):
    return cin >= 32 and cout >= 32 and rows >= 256


def wgrad_tc(dy, x, f16=False):
    """dW [Cout,Cin] = sum_{b,p} dy[b,:,p] x[b,:,p]^T on wgmma (csrc/train.cu: sonet_wgrad_tc_f32,
    with f16 its one-product twin sonet_wgrad_tc_f16: same splits and scratch)."""
    B, Cout, P = dy.shape
    Cin = x.shape[1]
    lib = _C.lib()
    base = ((Cout + 127) // 128) * (((Cin + 63) // 64 * 64 + 255) // 256)
    kch = (B * P + 63) // 64
    splits = max(1, min(64, 296 // base, kch))
    if -(-kch // splits) > WGRAD_MAX_KPI:
        splits = min(64, -(-kch // WGRAD_MAX_KPI))
    Kpad = int(lib.sonet_wgrad_kpad(B, P, splits))
    dev = dy.device
    with torch.cuda.device(dev):
        dyT = _scratch(dev, Kpad * Cout, torch.float32, _WGRAD_CACHE.setdefault("dyT", {}))
        blob = _scratch(dev, int(lib.sonet_wgrad_blob_bytes(Cin, Kpad)), torch.uint8,
                        _WGRAD_CACHE.setdefault("blob", {}))
        part = _scratch(dev, splits * Cin * Cout, torch.float32, _WGRAD_CACHE.setdefault("part", {}))
        small = torch.empty(int(lib.sonet_wgrad_small_floats(Cout)), dtype=torch.float32, device=dev)
        dWT = torch.empty((Cin, Cout), dtype=torch.float32, device=dev)
        ops._call(_f16("sonet_wgrad_tc_f32", f16), _C.ptr(dy), _C.ptr(x), B,
                  Cout, Cin, P, splits, _C.ptr(dyT), _C.ptr(blob), _C.ptr(part), _C.ptr(small),
                  _C.ptr(dWT), ops._stream(dy), kernels=8 if splits > 1 else 7)
    return dWT.t()


_WGRAD_CACHE = {}

# Longest K extent, in 64-point chunks, that one wgmma accumulator of the wgrad sums (more splits
# when the CTA count alone would allow longer ones). As with UPCONV_MAX_KPI, the tensor cores' fp32
# accumulation loses precision with the length of one chain: the segmenter's 3356 -> 1024 layer at
# B*P = 24576 had 2 splits of 192 chunks and a dW row error of 6.9e-5 (strict fp32 cuBLAS: 3e-6) on
# one H100 80GB HBM3 (700 W), tests/test_gpu_train_tc_envelope.py.
WGRAD_MAX_KPI = 32


class ConvTC(torch.autograd.Function):
    """x [B,Cin,P], W [Cout,Cin], b [Cout] or None -> W x + b. Forward, dgrad and wgrad all run on
    the generic wgmma layer kernel (fp16 hi/lo split, fp32 accumulation; under train_f16() one fp16
    product per MAC, the forward's x pre-scaled by a power of two like the dgrad's dy)."""

    @staticmethod
    def forward(ctx, x, W, b):
        x = x.contiguous()
        Wc = W.contiguous()
        f16 = train_f16()
        blob, scale2 = _pack_device(Wc, False)
        shift = None if b is None else b.contiguous()
        inv, act = _forward_scales(scale2, x) if f16 else (scale2[1:], None)
        y = _tc_dev(x, blob, inv, shift, Wc.shape[0], act_scale=act, f16=f16)
        ctx.save_for_backward(x, Wc)
        ctx.has_bias = b is not None
        ctx.f16 = f16
        return y

    @staticmethod
    def backward(ctx, dy):
        x, W = ctx.saved_tensors
        dy = dy.contiguous()
        dx = dW = db = None
        if ctx.needs_input_grad[0]:
            blob, scale2 = _pack_device(W, True)                     # dgrad: dx = W^T dy
            s_dy = _absmax_scale(dy)
            inv = scale2[1:] * s_dy[1:]
            dx = _tc_dev(dy, blob, inv, None, W.shape[1], act_scale=s_dy[:1], f16=ctx.f16)
        if ctx.needs_input_grad[1]:
            if W.shape[0] % 64 == 0 and W.shape[1] >= 16 and WGRAD_TC:
                dW = wgrad_tc(dy, x, ctx.f16)
            else:                                                    # thin layers: cuBLAS fp32
                with _cublas_strict_fp32():
                    dW = torch.einsum("bop,bip->oi", dy, x)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.sum(dim=(0, 2))
        return dx, dW, db


WGRAD_TC = True


class IndexMaxGatherRagged(torch.autograd.Function):
    """The per-node max of a ragged batch's stacked copies, differentiable w.r.t. data: data
    [1,C,k*T] (cloud b's columns cols[b] .. cols[b+1], cols = k*offsets), index [k*T] i32
    cloud-local nodes -> [B,C,M] (index_max_ragged's values). Backward: a deterministic scatter of
    each (cloud, channel)'s gradient in ascending node order (sonet_index_max_ragged_backward_f32)."""

    @staticmethod
    def forward(ctx, data, index, offsets, cols, M, k):
        data = data.contiguous()
        idx, val = ops.index_max_ragged(data.detach()[0], index, offsets, M, k)
        ctx.save_for_backward(idx, cols)
        ctx.L = data.shape[2]
        return val

    @staticmethod
    def backward(ctx, g):
        idx, cols = ctx.saved_tensors
        gd = ops.index_max_ragged_backward(g.contiguous(), idx, cols, ctx.L)
        return gd.unsqueeze(0), None, None, None, None, None


class IndexMaxGather(torch.autograd.Function):
    """data [B,C,N], index [B,N] int32, K -> data.gather(2, idx * mask_row_max) [B,C,K]
    (models/networks.py:181-185), differentiable w.r.t. data."""

    @staticmethod
    def forward(ctx, data, index, K):
        data = data.contiguous()
        idx, val = ops.index_max(data.detach(), index, K, with_values=True)
        ctx.save_for_backward(idx)
        ctx.N = data.shape[2]
        return val

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        g = g.contiguous()
        B, C, K = g.shape
        with torch.cuda.device(g.device):
            gd = torch.empty((B, C, ctx.N), dtype=torch.float32, device=g.device)
            ops._call("sonet_index_max_backward_f32", _C.ptr(g), _C.ptr(idx), B, C, ctx.N, K,
                      _C.ptr(gd), ops._stream(g))
        return gd, None, None


def _cudnn_strict_fp32(tf32=False):
    c = torch.backends.cudnn
    return c.flags(enabled=True, benchmark=c.benchmark, deterministic=c.deterministic,
                   allow_tf32=tf32)


def _conv_forward(ctx, tf32, x, weight, bias, stride, padding, dilation, groups):
    ctx.tf32 = tf32
    with _cudnn_strict_fp32(tf32):
        y = torch.ops.aten.convolution(x, weight, bias, stride, padding, dilation, False,
                                       [0] * len(stride), groups)
    ctx.save_for_backward(x, weight)
    ctx.conf = (None if bias is None else [bias.shape[0]], stride, padding, dilation, groups)
    return y


class ConvStrict(torch.autograd.Function):
    """F.conv1d / F.conv2d (zero padding) with cuDNN's TF32 off in the forward AND the backward,
    whatever torch.backends.cudnn.allow_tf32 says. PyTorch's own backward reads the global flag
    when backward() runs, outside any context the forward was called in; TF32 (~5e-4 per product)
    is far outside the 1e-4 parity bar of the reference's fp32 math."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, dilation, groups):
        return _conv_forward(ctx, False, x, weight, bias, stride, padding, dilation, groups)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        bias_sizes, stride, padding, dilation, groups = ctx.conf
        need = ctx.needs_input_grad
        with _cudnn_strict_fp32(ctx.tf32):
            dx, dw, db = torch.ops.aten.convolution_backward(
                dy.contiguous(), x, weight, bias_sizes, stride, padding, dilation, False,
                [0] * len(stride), groups, [need[0], need[1], bias_sizes is not None and need[2]])
        return dx, dw, db, None, None, None, None


class ConvTF32(ConvStrict):
    """ConvStrict with TF32 allowed in the forward and the backward (the reference's default),
    whatever the global flag says when backward() runs: the decoder's cuDNN convolutions under
    train_f16()."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, dilation, groups):
        return _conv_forward(ctx, True, x, weight, bias, stride, padding, dilation, groups)


def conv_strict(conv, x):
    """conv (nn.Conv1d / nn.Conv2d, zero padding) applied to x through ConvStrict."""
    return ConvStrict.apply(x, conv.weight, conv.bias, list(conv.stride), list(conv.padding),
                            list(conv.dilation), conv.groups)


def conv_tf32(conv, x):
    """conv applied to x through ConvTF32."""
    return ConvTF32.apply(x, conv.weight, conv.bias, list(conv.stride), list(conv.padding),
                          list(conv.dilation), conv.groups)


@contextlib.contextmanager
def _cublas_strict_fp32():
    """cuBLAS fp32 GEMMs without TF32 for the duration, whatever the global flag says."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


class LinearStrict(torch.autograd.Function):
    """x [B,Cin] W^T + b on cuBLAS with TF32 off in the forward AND the backward (the global flag
    is read when backward() runs, outside any context the forward was called in)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        with _cublas_strict_fp32():
            y = torch.addmm(bias, x, weight.t()) if bias is not None else x @ weight.t()
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        need = ctx.needs_input_grad
        dx = dW = db = None
        with _cublas_strict_fp32():
            if need[0]:
                dx = dy @ weight
            if need[1]:
                dW = dy.t() @ x
        if ctx.has_bias and need[2]:
            db = dy.sum(0)
        return dx, dW, db


def norm_act_train(y0, norm, act, epoch=None, size=None, cols=None):
    """The norm / activation half of every train-mode layer on its pre-norm output y0 [B,C,P]:
    batch-stat BN (+ running-stat update with the reference's momentum schedule,
    models/layers.py:57-65; like F.batch_norm, num_batches_tracked is left alone) or instance norm
    (affine, no running statistics: nothing to update) or none -> act: the layer's activation
    (None, 'relu' or 'elu'; a bool means ReLU or none). size: the layer output's shape as the
    reference sees it, for the messages of F.batch_norm's and F.instance_norm's ValueErrors.
    cols: the device column offsets of a ragged batch's y0 [1,C,L] (BNActTrain); the statistics
    then cover n = L columns, in the running variance too. Refused with instance norm and with a
    data-parallel exchange installed."""
    B, C, P = y0.shape
    size = y0.size() if size is None else torch.Size(size)
    instance = isinstance(norm, _InstanceNorm)
    if cols is not None and (instance or EXCHANGE is not None):
        raise RuntimeError("norm_act_train: a ragged batch (cols) has no %s" % (
            "per-cloud instance statistics" if instance else "data-parallel BatchNorm exchange"))
    if instance and not (norm.affine and not norm.track_running_stats):
        raise RuntimeError("norm_act_train: instance norm needs affine=True and "
                           "track_running_stats=False")
    if instance and P < 2:   # F.instance_norm's check
        raise ValueError("Expected more than 1 spatial element when training, got input size "
                         "{}".format(size))
    if instance:
        return InstanceNormActTrain.apply(y0, norm.weight, norm.bias, norm.eps, act)
    if norm is None:
        code = ops.act_code(act)
        if code == ops.ACT_ELU:
            return F.elu(y0)
        return torch.relu(y0) if code == ops.ACT_RELU else y0
    # with a BatchNorm exchange installed the statistics are those of the global batch
    n = P if cols is not None else _exchange().global_rows(B) * P
    if n == 1:         # F.batch_norm's check: a batch statistic of one value is undefined
        raise ValueError("Expected more than 1 value per channel when training, got input size "
                         "{}".format(size))
    norm.momentum = norm.momentum_at(epoch)
    y, mean, var = BNActTrain.apply(y0, norm.weight, norm.bias, norm.eps, act, cols)
    with torch.no_grad():
        m = norm.momentum
        norm.running_mean.mul_(1 - m).add_(mean, alpha=m)
        norm.running_var.mul_(1 - m).add_(var * (n / (n - 1)), alpha=m)
    return y


def conv_bn_act_train(x3, weight2d, bias, norm, act, epoch=None, cols=None):
    """Train-mode EquivariantLayer / MyConv2d(1x1) body on [B,Cin,P]: conv (wgmma when dense
    enough, else strict-fp32 cuDNN) -> norm_act_train (cols: a ragged batch's, as there)."""
    B, Cin, P = x3.shape
    Cout = weight2d.shape[0]
    if tc_eligible(Cin, Cout, B * P):
        y0 = ConvTC.apply(x3, weight2d, bias)
    else:
        y0 = ConvStrict.apply(x3, weight2d.unsqueeze(2), bias, [1], [0], [1], 1)
    return norm_act_train(y0, norm, act, epoch, cols=cols)


# ---- the up-convolution (csrc/upconv.cu) -----------------------------------------------------------
def _fold(src, Cout, Cin, adjoint, out, out_dgrad=None):
    ops._call("sonet_upconv_fold_weights_f32", _C.ptr(src), Cout, Cin, int(adjoint), _C.ptr(out),
              _C.ptr(out_dgrad), ops._stream(src), kernels=(out is not None) + (out_dgrad is not None))


def _pack_groups_device(Wg):
    """Wg [G,Cout,Cin] (device) -> (G consecutive blobs, scale2) with one common pre-scale."""
    G, Cout, Cin = Wg.shape
    dev = Wg.device
    per = int(_C.lib().sonet_pointwise_tc_blob_bytes(Cout, Cin))
    with torch.cuda.device(dev):
        blob = torch.empty(per * G, dtype=torch.uint8, device=dev)
        scale2 = torch.empty(2, dtype=torch.float32, device=dev)
        part = torch.empty(_C.CONSTANTS["SONET_ABSMAX_SLOTS"], dtype=torch.float32, device=dev)
        ops._call("sonet_pointwise_tc_pack_groups_device", _C.ptr(Wg), G, Cout, Cin, _C.ptr(blob),
                  _C.ptr(scale2), _C.ptr(part), ops._stream(Wg), kernels=2 + G)
    return blob, per, scale2


# Longest K extent, in 64-channel chunks, that one wgmma accumulator of the up-convolution's forward
# and dgrad GEMMs sums before the fixed-order fp32 split-K reduce takes over. The tensor cores' fp32
# accumulation loses precision with the length of one accumulation chain: the row error of deconv6's
# dx from fp64 grew about linearly with it (one H100 80GB HBM3, 700 W, B = 16: 1.1e-5 at 32 chunks,
# 1.5e-6 at 4; cuDNN strict fp32 4.6e-7). The extra split costs deconv6's forward + backward at
# B = 32 3.31 ms instead of 2.98.
UPCONV_MAX_KPI = 4


def _upconv_splits(kchunks, base_items):
    """K split of an up-convolution GEMM: ops.pick_splits' choice, raised to the smallest divisor of
    kchunks that keeps every accumulator within UPCONV_MAX_KPI chunks."""
    s = ops.pick_splits(kchunks, base_items)
    if kchunks // s <= UPCONV_MAX_KPI:
        return s
    return min(d for d in range(s, kchunks + 1) if kchunks % d == 0 and kchunks // d <= UPCONV_MAX_KPI)


class UpConvTC(torch.autograd.Function):
    """x [B,Cin,H,W] (H*W > 1), W [Cout,Cin,3,3], b [Cout] -> z = conv3x3(upsample2(x)) + b
    [B,Cout,2H,2W] as four parity GEMMs (Wg = the taps that coincide after up-sampling, summed).
      forward  z = grouped parity GEMMs (Wg, x) + b, Wg folded and packed on the device
      dgrad    dx = Wd D: D [B][16*Cout][H*W] = dz gathered at each (parity, tap, co)'s offset
      wgrad    dWg[g] = dz_g xcol_g^T per parity (xcol recomputed from x), dW = adjoint fold
    Under train_f16() all three take the one-product twins, the forward's x pre-scaled by a power
    of two (max|im2col(x)| = max|x|)."""

    @staticmethod
    def forward(ctx, x, W, b):
        x = x.contiguous()
        f16 = train_f16()
        Wc = W.contiguous()
        B, Cin, H, Wd = x.shape
        Cout = Wc.shape[0]
        P = H * Wd
        dev = x.device
        with torch.cuda.device(dev):
            Wg = torch.empty((4, Cout, 4 * Cin), dtype=torch.float32, device=dev)
            _fold(Wc, Cout, Cin, False, Wg)
            blob, per, scale2 = _pack_groups_device(Wg)
            conv = ops.upconv_conv_mode(Cin, H, Wd)
            xin = ops.upconv_hshift(x) if conv else ops.upconv_im2col(x)
            splits = _upconv_splits((4 * Cin + 63) // 64, 4 * ((B * P + 127) // 128) * ((Cout + 255) // 256))
            z = torch.empty((B, Cout, 4 * P), dtype=torch.float32, device=dev)
            scratch = (torch.empty(4 * splits * B * Cout * P, dtype=torch.float32, device=dev)
                       if splits > 1 else None)
            shift = None if b is None else b.contiguous()
            inv, act = _forward_scales(scale2, x) if f16 else (scale2[1:], None)
            scales = (_C.ptr(inv), _C.ptr(act)) if f16 else (_C.ptr(inv),)   # the twin's extra argument
            ops._call(_f16("sonet_pointwise_tc_grouped_forward_dev", f16), _C.ptr(xin), xin.shape[1], B,
                      P, _C.ptr(blob), per, *scales, _C.ptr(shift), Cout, ops.ACT_NONE, 4, splits, Wd,
                      Wd if conv else 0, 4 * P, 0, _C.ptr(z), _C.ptr(scratch), ops._stream(x),
                      kernels=2 if splits > 1 else 1)
        ctx.save_for_backward(x, Wc)
        ctx.has_bias = b is not None
        ctx.f16 = f16
        return z.view(B, Cout, 2 * H, 2 * Wd)

    @staticmethod
    def backward(ctx, dz):
        x, W = ctx.saved_tensors
        dz = dz.contiguous()
        B, Cin, H, Wd = x.shape
        Cout = W.shape[0]
        P = H * Wd
        dev = x.device
        dx = dW = db = None
        with torch.cuda.device(dev):
            if ctx.needs_input_grad[0]:
                Wdg = torch.empty((Cin, 16 * Cout), dtype=torch.float32, device=dev)
                _fold(W, Cout, Cin, False, None, Wdg)
                blob, scale2 = _pack_device(Wdg, False)
                D = torch.empty((B, 16 * Cout, P), dtype=torch.float32, device=dev)
                ops._call("sonet_upconv_dgrad_im2col_f32", _C.ptr(dz), B, Cout, H, Wd, _C.ptr(D),
                          ops._stream(dz))
                s_dz = _absmax_scale(dz)            # max|D| = max|dz|: D holds every dz element
                splits = _upconv_splits((16 * Cout + 63) // 64,
                                        ((B * P + 127) // 128) * (((Cin + 63) // 64 * 64 + 127) // 128))
                dx = torch.empty((B, Cin, P), dtype=torch.float32, device=dev)
                scratch = (torch.empty(splits * B * Cin * P, dtype=torch.float32, device=dev)
                           if splits > 1 else None)
                ops._call(_f16("sonet_pointwise_tc_forward_dev", ctx.f16), _C.ptr(D), 16 * Cout, B, P,
                          _C.ptr(blob),
                          _C.ptr(scale2[1:] * s_dz[1:]), _C.ptr(s_dz[:1]), None, Cin, 0, splits,
                          _C.ptr(dx), _C.ptr(scratch), ops._stream(dz),
                          kernels=2 if splits > 1 else 1)
                dx = dx.view(B, Cin, H, Wd)
            if ctx.needs_input_grad[1]:
                # the four parity planes of dz, copied once: [4][B][Cout][H*W]
                dzg = dz.view(B, Cout, H, 2, Wd, 2).permute(3, 5, 0, 1, 2, 4).reshape(4, B, Cout, P)
                xcol = ops.upconv_im2col(x).view(4, B, 4 * Cin, P)
                if Cout % 64 == 0 and WGRAD_TC:
                    dWT = torch.stack([wgrad_tc(dzg[g], xcol[g], ctx.f16).t() for g in range(4)])
                else:
                    with _cublas_strict_fp32():
                        dWT = torch.einsum("gbkp,gbop->gko", xcol, dzg)
                dW = torch.empty_like(W)
                _fold(dWT.contiguous(), Cout, Cin, True, dW)
            if ctx.has_bias and ctx.needs_input_grad[2]:
                db = dz.sum(dim=(0, 2, 3))
        return dx, dW, db


# Smallest input map (H*W) whose train-mode up-convolution runs on the parity GEMMs; smaller maps
# keep the strict-fp32 cuDNN composition. Measured with tools/ae_train_bench.py on one H100 80GB HBM3
# (700 W power limit), B = 32, forward + backward of each DecoderConv stage: kernels vs cuDNN
# 1.33/1.12 ms (1x1 input), 1.67/0.79 (2x2), 1.47/0.74 (4x4), 1.29/0.70 (8x8), 1.57/1.44 and
# 1.45/1.58 in two runs (16x16), 3.31/8.00 (32x32): below 32x32 the fixed cost of the per-step fold,
# packs and four wgrad calls (tools/ae_train_bench.py breaks it down) outweighs the GEMMs.
UPCONV_MIN_HW = 1024


def upconv_train(x, weight, bias):
    """Train-mode nearest x2 up-sampling + 3x3 conv (pad 1) of x [B,Cin,H,W] -> [B,Cout,2H,2W],
    before the norm. A 1x1 input is the dense layer Cin -> 4*Cout whose weight holds, per output
    parity, the sum of the taps that land on the single pixel (rows / columns {1,2} for parity 0,
    {0,1} for parity 1); larger maps run UpConvTC."""
    B, Cin, H, Wd = x.shape
    Cout = weight.shape[0]
    if H * Wd > 1:
        return UpConvTC.apply(x, weight, bias)
    taps = ((1, 2), (0, 1))
    W1 = torch.stack([weight[:, :, taps[py][0]:taps[py][1] + 1, taps[px][0]:taps[px][1] + 1].sum((2, 3))
                      for py in range(2) for px in range(2)], dim=1).reshape(4 * Cout, Cin)
    b1 = None if bias is None else bias.repeat_interleave(4)
    x3 = x.reshape(B, Cin, 1)
    if tc_eligible(Cin, 4 * Cout, B):
        y0 = ConvTC.apply(x3, W1, b1)
    else:
        y0 = ConvStrict.apply(x3, W1.unsqueeze(2), b1, [1], [0], [1], 1)
    return y0.view(B, Cout, 2, 2)      # output channel co*4 + py*2 + px
