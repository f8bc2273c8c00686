"""Shared test helpers: golden loading, model construction with the seeded synthetic weights."""
import os

import numpy as np
import torch

from sonet_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

# parity tolerance for floating-point tensors (BASELINE.json north_star: fp32 within 1e-4 rel):
#   |a - b| <= TOL * max(|b|, 1)
TOL = 1e-4


# ---- error bars of the fp16 hi/lo tensor-core GEMMs (csrc/tc_common.cuh) ------------------------
# The 3-product split x*w ~= hi(x)hi(w) + lo(x)hi(w) + hi(x)lo(w) carries about 22 significant
# bits per operand, then the products are summed in fp32. Below |x| ~ 2^-3 the lo half of an
# activation is an fp16 subnormal, so every activation carries an ABSOLUTE error of up to 2^-25
# however small it is; the same holds for a weight after its matrix's power-of-two pre-scale s_w
# (2^-25 / s_w unscaled). So per output element of y = W x (+ shift, + addend):
#
#     |got - y| <= TC_R * m + TC_F * (sum_k |W[o,k]| + sum_k |x[k]| / s_w)
#
# with m = |W| |x| + |shift| + |addend| in fp64: TC_R bounds the split's relative error, TC_F is
# the subnormal-lo floor. Measured on one H100 80GB HBM3 (400 W power limit) over
# tests/test_gpu_tc_envelope.py: max |got - y| / m was 1.2e-6 for the generic layer at input scale
# 2^8 (K = 1024, floor negligible; strict-fp32 cuBLAS on the same operands: 3.2e-7) and 1.6e-6 with
# per-channel input scales from 2^-14 to 2^14; at input scale 2^-14, where the floor rules, the
# error was 0.1 of the floor term below. TC_R is 2.5x the largest measurement, TC_F = 2 * 2^-25.
TC_R = 4e-6
TC_F = 2.0 ** -24
# how much worse than strict fp32 (in units of the bar) the tensor-core path may be; below
# TC_FP32_FLOOR units the comparison is noise
TC_FP32_FACTOR = 8.0
TC_FP32_FLOOR = 0.125

# Error bar of one opt-in fp16-mode GEMM output (SONET_TC=fp16: one fp16 product per MAC) against
# the fp64 GEMM of its rounded operands:
#     |got - y16| <= F16_C * (sum_k |W16[o,k] x16[k]| / s + |shift| + |addend|)
# F16_C covers the fp32 accumulation inside the tensor cores, the fp32 epilogue and, with split-K,
# the fp32 partial sums. Measured on one H100 80GB HBM3 (700 W power limit) over the kernel cases
# of tests/test_gpu_fp16_mode.py: max err / m = 6.0e-7 (the saturated-input case; 1.2e-7 .. 5.3e-7
# elsewhere). F16_C is 2.5x that, as TC_R is 2.5x its measurement. A leftover lo product would
# show as ~2^-11 = 4.9e-4.
F16_C = 1.5e-6


def tc_reference(W, x, shift=None, addend=None, w_scale=None, parts=False):
    """fp64 y = W x (+ shift[o]) (+ addend, already gathered to [B,Cout,P]) and the error bar of
    the tensor-core layer (see TC_R / TC_F), both on x's device (cuBLAS fp64).
    W [Cout,Cin]; x [B,Cin,P]; w_scale = the weights' power-of-two pre-scale (1 / inv_scale).
    parts=True returns (y, m, floor) instead of (y, bar)."""
    dev = x.device
    W64, x64 = W.to(dev, torch.float64), x.to(torch.float64)
    y = torch.einsum("ok,bkp->bop", W64, x64)
    m = torch.einsum("ok,bkp->bop", W64.abs(), x64.abs())
    if shift is not None:
        s64 = shift.to(dev, torch.float64)[None, :, None]
        y = y + s64
        m = m + s64.abs()
    if addend is not None:
        a64 = addend.to(dev, torch.float64)
        y = y + a64
        m = m + a64.abs()
    floor = W64.abs().sum(1)[None, :, None].expand_as(m)
    if w_scale is not None:
        floor = floor + x64.abs().sum(1, keepdim=True) / float(w_scale)
    if parts:
        return y, m, floor
    return y, TC_R * m + TC_F * floor


def fp32_gemm(W, x, shift=None, addend=None):
    """The same layer as a strict-fp32 cuBLAS GEMM (TF32 off) on x's device: the yardstick the
    tensor-core path is held to."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        y = torch.matmul(W.to(x.device, torch.float32), x.float())
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    if shift is not None:
        y = y + shift.to(x.device, torch.float32)[None, :, None]
    if addend is not None:
        y = y + addend.float()
    return y


def bar_units(got, y, bar, relu=False):
    """max |got - y| / bar (y, bar from tc_reference; relu applied to y here)."""
    if relu:
        y = y.clamp(min=0)
    return float(((got.to(y.device, torch.float64) - y).abs() / bar).max())


def assert_in_tc_envelope(got, y, bar, what, relu=False, fp32=None):
    """got within the tensor-core error bar, and no more than TC_FP32_FACTOR times worse than the
    strict-fp32 result `fp32` of the same operands (both in units of the bar)."""
    u = bar_units(got, y, bar, relu)
    assert u <= 1.0, "%s: error is %.3g x the tensor-core error bar" % (what, u)
    if fp32 is not None:
        u32 = bar_units(fp32.clamp(min=0) if relu else fp32, y, bar, relu)
        assert u <= TC_FP32_FACTOR * max(u32, TC_FP32_FLOOR), \
            "%s: %.3g bar units, strict fp32 %.3g" % (what, u, u32)
    return u


def row_rel_err(a, b):
    """Per-row relative error of a gradient matrix [R, C] (or anything viewed so):
    max_c |a - b| / max_c |b| for every row; a row whose reference is all zero must be all zero."""
    a = torch.as_tensor(a).detach().to(torch.float64).reshape(a.shape[0], -1)
    b = torch.as_tensor(b).detach().to(a.device, torch.float64).reshape(b.shape[0], -1)
    num = (a - b).abs().amax(1)
    den = b.abs().amax(1)
    return torch.where(den > 0, num / den.clamp(min=1e-300), torch.where(num > 0, torch.inf, 0.0))


def assert_rows_close(a, b, what, tol):
    e = row_rel_err(a, b)
    worst = int(e.argmax())
    assert float(e[worst]) <= tol, "%s: row %d has relative error %.3e > %.1e" % (
        what, worst, float(e[worst]), tol)
    return float(e.max())


def golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)


def rel_err(a, b):
    a = torch.as_tensor(a, dtype=torch.float32).cpu()
    b = torch.as_tensor(b, dtype=torch.float32).cpu()
    return float(((a - b).abs() / b.abs().clamp(min=1.0)).max())


def assert_close(a, b, what, tol=TOL):
    e = rel_err(a, b)
    assert e <= tol, "%s: max |a-b|/max(|b|,1) = %.3e > %.1e" % (what, e, tol)


def sampled(g, name, t):
    """Compare-ready view of tensor t at the positions a golden strided sample was taken."""
    stride = int(g[name + "__stride"])
    assert tuple(g[name + "__shape"]) == tuple(t.shape), (name, tuple(g[name + "__shape"]), tuple(t.shape))
    return t.detach().cpu().contiguous().view(-1)[::stride]


def assert_golden(g, name, t, tol=TOL):
    assert_close(sampled(g, name, t), torch.from_numpy(g[name]), "golden " + name, tol)


def build_states(task, opt, seed, make=synth.synth_state_dict):
    """State dicts (CPU tensors) for encoder and head, keyed like the reference's."""
    from sonet_b200 import networks
    cpu_opt = synth.make_opt(task, **{k: v for k, v in vars(opt).items()
                                      if k not in ("device",)})
    cpu_opt.device = torch.device("cpu")
    enc = networks.Encoder(cpu_opt)
    st = dict(encoder=make(enc, seed=seed))
    if task == "classifier":
        st["head"] = make(networks.Classifier(cpu_opt), seed=seed + 1)
    elif task == "segmenter":
        st["head"] = make(networks.Segmenter(cpu_opt), seed=seed + 1)
    elif task == "autoencoder":
        st["head"] = make(networks.Decoder(cpu_opt), seed=seed + 1)
    return st


def trained_like_state_dict(module_or_state, seed=0):
    """synth_state_dict with BatchNorm statistics as spread out as a trained network's:
    running_var log-uniform on [1e-6, 1e2], gamma log-uniform on [1e-3, 3] with a few exact zeros,
    running_mean ~ N(0, 3) in units of the channel's standard deviation. As in a trained network
    the statistics describe the data the BN sees: the rows (and bias) of the layer in front of
    each BN are scaled by sqrt(running_var). (Statistics drawn independently of the weights instead
    push every layer's output up to 3e3 times its input, and activations past fp16's range within
    a few layers: 1e5 after the first PointResNet, 1e11 at the final PointNet.)"""
    st = synth.synth_state_dict(module_or_state, seed=seed)
    rs = np.random.RandomState(seed + 4242)
    for name, t in list(st.items()):
        if not name.endswith("norm.running_var"):
            continue
        pre = name[:-len("norm.running_var")]
        n = t.numel()
        var = 10.0 ** rs.uniform(-6, 2, n)
        gamma = 10.0 ** rs.uniform(-3, np.log10(3.0), n)
        gamma[rs.randint(0, n, size=max(1, n // 50))] = 0.0
        sd = np.sqrt(var)
        st[name] = torch.from_numpy(var.astype(np.float32))
        st[pre + "norm.weight"] = torch.from_numpy(gamma.astype(np.float32))
        st[pre + "norm.running_mean"] = torch.from_numpy((rs.normal(0, 3, n) * sd).astype(np.float32))
        for k in st:
            if k.startswith(pre) and "norm" not in k[len(pre):] and k.endswith((".weight", ".bias")) \
                    and st[k].shape[0] == n:
                s = torch.from_numpy(sd.astype(np.float32)).view(-1, *[1] * (st[k].dim() - 1))
                st[k] = st[k] * s
    return st


def golden_options(g):
    """The non-default options a fixture was generated with (oracle/make_golden.py stores each
    one as opt_<name>)."""
    return {key[4:]: g[key].item() for key in g.files if key.startswith("opt_")}


def golden_case(g, task, **over):
    B, N, seed = int(g["B"]), int(g["N"]), int(g["seed"])
    som_k = int(g["som_k"])
    kw = dict(batch_size=B, input_pc_num=N, som_k=som_k)
    kw.update(golden_options(g))
    kw.update(over)
    opt = synth.make_opt(task, **kw)
    inp = synth.synth_inputs(B, N, opt.node_num, max(som_k, 1), seed=seed,
                             node_mode=str(g["node_mode"]))
    return opt, inp, seed


def check_encoder_against_golden(g, enc, opt):
    """Every cached encoder attribute of a CUDA run against a reference fixture: k-sets and mask
    statistics exact, node-level tensors and (in the reference's slot order) first_pn_out within
    TOL."""
    from oracle import oracle
    assert np.array_equal(oracle.canon_sets(enc.min_idx.cpu(), opt.k).numpy(), g["knn_sets"])
    mask = enc.mask
    assert mask.dtype == torch.int32
    assert np.array_equal(torch.max(mask, dim=1)[0].cpu().numpy(), g["mask_row_max"])
    assert np.array_equal(torch.sum(mask, dim=1).cpu().numpy(), g["mask_row_sum"])
    for n in ("som_node", "first_pn_out_masked_max", "final_pn_out", "feature"):
        assert_golden(g, n, getattr(enc, n))
    assert_golden(g, "first_pn_out", to_ref_slot_order(enc.first_pn_out, enc.min_idx, g, opt.k))
    if opt.som_k >= 2:
        assert_golden(g, "knn_center_1", enc.knn_center_1)
        assert_golden(g, "knn_feature_1", enc.knn_feature_1)


def to_ref_slot_order(t, our_min_idx, g, k):
    return to_slot_order(t, our_min_idx, torch.from_numpy(g["min_idx_ref"].astype(np.int64)), k)


def to_slot_order(t, our_min_idx, ref, k):
    """Reorder the k stacked copies of a [B,C,kN] tensor from OUR slot order (ascending distance)
    to the slot order the reference run used (its topk(sorted=False) order is implementation
    defined; parity for the assignment is per-point set equality — SURVEY.md Appendix C)."""
    ref = ref.detach().cpu().long()                                     # [B,kN]
    ours = our_min_idx.detach().cpu().long()
    B, kN = ours.shape
    N = kN // k
    ours_k = ours.view(B, k, N)
    ref_k = ref.view(B, k, N)
    # src_slot[b, s, n] = our slot holding the node the reference has in slot s
    match = ref_k.unsqueeze(2) == ours_k.unsqueeze(1)                   # [B, k_ref, k_ours, N]
    assert bool(match.any(dim=2).all()), "assignment sets differ"
    src_slot = match.float().argmax(dim=2)                              # [B,k,N]
    src = (src_slot * N + torch.arange(N).view(1, 1, N)).view(B, kN)
    tc = t.detach().cpu()
    return torch.gather(tc, 2, src.unsqueeze(1).expand(B, tc.shape[1], kN))
