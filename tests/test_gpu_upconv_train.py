"""-m gpu: the auto-encoder's decoder in train() mode on the sm_90a kernels (train_ops.UpConvTC,
the shared norm / activation half, MyLinear's strict-fp32 GEMM):

  A. every DecoderConv stage shape against the same module in fp64, held to 8x the error of the
     strict-fp32 PyTorch composition (the bar of test_gpu_train_parity's layer test), over the
     activations, normalizations and both operand forms of the parity GEMMs;
  B. the dgrad GEMM and wgrad at gradients of 1e-7 against fp64; the device-packed grouped blob;
  C. the route (ops.PROFILE, conv_strict only for ineligible stages), ENABLED = False, determinism
     and the running statistics;
  D. the whole Decoder, MyLinear, and one autoencoder.Model.optimize() step.
"""
import contextlib
import copy

import pytest
import torch
import torch.nn.functional as F

from helpers import build_states, row_rel_err, trained_like_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def kernels_at_every_map_size(monkeypatch):
    """The parity GEMMs at every stage shape, below train_ops.UPCONV_MIN_HW too (the map-size rule
    itself: test_map_size_rule)."""
    from sonet_b200 import train_ops
    monkeypatch.setattr(train_ops, "UPCONV_MIN_HW", 1)


@contextlib.contextmanager
def flags(kernels, cudnn_tf32=False):
    from sonet_b200 import train_ops
    prev = (train_ops.ENABLED, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    train_ops.ENABLED = kernels
    torch.backends.cudnn.allow_tf32 = cudnn_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        train_ops.ENABLED, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _run(mod, inputs, dtype, w):
    """One train-mode forward + backward of a copy of mod in dtype: {name: tensor}."""
    mod = copy.deepcopy(mod).to(DEV, dtype).train()
    x = inputs.to(DEV, dtype).requires_grad_(True)
    y = mod(x)
    y.backward(w.to(DEV, dtype))
    out = {"y": y.detach(), "dx": x.grad.detach()}
    out.update({"d " + n: p.grad.detach() for n, p in mod.named_parameters() if p.grad is not None})
    return out


def _rows(name, t):
    if name in ("y", "dx"):
        return t.transpose(0, 1).reshape(t.shape[1], -1)
    return t.reshape(1, -1) if t.dim() == 1 else t.reshape(t.shape[0], -1)


def _before_norm(grads, n):
    """A layer's bias in front of its normalization (a per-channel constant the norm removes): its
    gradient is analytically zero, and what any arithmetic returns is rounding noise."""
    return (n.endswith(".bias") and not n.endswith(".norm.bias")
            and n.rsplit(".", 2)[0] + ".norm.weight" in grads)


# a ReLU pre-activation within this fraction of its channel's largest magnitude may take either gate
GATE_TOL = 1e-4


class _GatedReLU(torch.nn.Module):
    """The fp64 reference's ReLU for one fp32 run: z > 0, except where |z| is within GATE_TOL of its
    channel's largest |z|, where it takes that run's gate (y > 0). There the fp32 pre-activation is
    within rounding of zero and either gate is right; a flipped gate moves a whole gradient value, so
    without this the error would count gates, not arithmetic. A gate flipped anywhere else moves y by
    more than GATE_TOL of its channel, which the y comparison catches."""

    def __init__(self, gate):
        super().__init__()
        self.gate = gate

    def forward(self, z):
        dims = [d for d in range(z.dim()) if d != 1]
        amb = z.abs() <= GATE_TOL * z.abs().amax(dim=dims, keepdim=True)
        return z * torch.where(amb, self.gate.to(z.device), z > 0).to(z.dtype)


def _fp64_ref(mod, x, w, y32):
    """mod in fp64; ReLU gates near zero follow the fp32 output y32."""
    m = copy.deepcopy(mod)
    for parent in [m] + list(m.modules()):
        if isinstance(getattr(parent, "act", None), torch.nn.ReLU):
            parent.act = _GatedReLU(y32 > 0)
    return _run(m, x, torch.float64, w)


def _vs_fp64(case, mod, x):
    """kernels on (cuDNN TF32 allowed: PyTorch's default) vs fp64, bar max(8 x strict fp32, 1e-5);
    each fp32 run against an fp64 reference whose ambiguous ReLU gates follow that run."""
    mod.load_state_dict(trained_like_state_dict(mod, seed=len(case)))
    with torch.no_grad(), flags(False):
        shape = copy.deepcopy(mod).to(DEV).train()(x.to(DEV)).shape
    w = torch.randn(shape, generator=torch.Generator().manual_seed(5))
    with flags(True, cudnn_tf32=True):
        got = _run(mod, x, torch.float32, w)
    with flags(False):
        strict = _run(mod, x, torch.float32, w)
    ref = _fp64_ref(mod, x, w, got["y"])
    ref32 = _fp64_ref(mod, x, w, strict["y"])
    assert set(got) == set(ref) == set(strict)
    worst = {}
    for n, r64 in ref.items():
        if _before_norm(ref, n):
            assert float(got[n].abs().max()) < 1e-3 * float(ref[n[:-4] + "weight"].abs().max()), n
            continue
        e32 = row_rel_err(_rows(n, strict[n]), _rows(n, ref32[n]))
        e = row_rel_err(_rows(n, got[n]), _rows(n, r64))
        lim = torch.clamp(8 * e32, min=1e-5)
        worst[n] = (float((e / lim).max()), float(e.max()), float(e32.max()))
        bad = e > lim
        assert not bool(bad.any()), "%s %s: row %d has relative error %.3e; strict fp32 %.3e" % (
            case, n, int(bad.nonzero()[0]), float(e[bad][0]), float(e32[bad][0]))
    n_w = max(worst, key=lambda k: worst[k][0])
    print("\n[upconv-train] %s: worst ratio %.3f (%s %.2e, fp32 %.2e)" % ((case, worst[n_w][0], n_w)
                                                                      + worst[n_w][1:]))


STAGES = [  # name, Cin, Cout, H, B
    ("deconv1_1x1", 1024, 1024, 1, 4),
    ("deconv2_2x2", 1024, 512, 2, 4),
    ("deconv3_4x4", 512, 256, 4, 4),
    ("deconv4_8x8", 256, 128, 8, 4),
    ("deconv5_16x16", 128, 128, 16, 4),
    ("deconv6_32x32", 128, 128, 32, 2),
    ("deconv6_32x32_b32", 128, 128, 32, 32),
    ("enabled_64x64", 128, 128, 64, 2),
    ("f512_deconv3_4x4", 256, 128, 4, 4),
]
CASES = [(s, "relu", "batch") for s in STAGES]
# DecoderConv at feature_num 1024 (B = 4; deconv6 also at the training batch, B = 32), one stage at
# 512, and a 64x64 input
CASES += [(STAGES[i], "elu", "instance") for i in (0, 2, 4)]
CASES += [(STAGES[i], None, None) for i in (1, 3)]
CASES += [(STAGES[i], "relu", "instance") for i in (3,)]
CASES += [(STAGES[i], "elu", "batch") for i in (5,)]


@pytest.mark.parametrize("stage,act,norm", CASES,
                         ids=["%s-%s-%s" % (s[0], a, n) for s, a, n in CASES])
def test_decoder_stage_vs_fp64(stage, act, norm):
    from sonet_b200 import layers
    name, Cin, Cout, H, B = stage
    torch.manual_seed(0)
    mod = layers.UpConv(Cin, Cout, activation=act, normalization=norm)
    x = torch.randn(B, Cin, H, H, generator=torch.Generator().manual_seed(Cin + H))
    _vs_fp64("%s-%s-%s" % (name, act, norm), mod, x)


@pytest.mark.parametrize("name", ["deconv4_8x8", "deconv5_16x16"])
def test_decoder_stage_im2col_form_vs_fp64(name, monkeypatch):
    """SONET_UPCONV_IM2COL=1: the stages that read the horizontal shifts take the 16x im2col."""
    from sonet_b200 import layers
    monkeypatch.setenv("SONET_UPCONV_IM2COL", "1")
    _, Cin, Cout, H, B = dict((s[0], s) for s in STAGES)[name]
    torch.manual_seed(0)
    mod = layers.UpConv(Cin, Cout, activation="relu", normalization="batch")
    x = torch.randn(B, Cin, H, H, generator=torch.Generator().manual_seed(Cin + H))
    _vs_fp64(name + "-im2col", mod, x)


def _conv_grads64(x, W, b, dz):
    x64, W64, b64 = (t.double().requires_grad_(True) for t in (x, W, b))
    z = F.conv2d(F.interpolate(x64, scale_factor=2, mode="nearest"), W64, b64, padding=1)
    z.backward(dz.double())
    return z.detach(), x64.grad, W64.grad


@pytest.mark.parametrize("Cin,Cout,H,B", [(256, 128, 8, 8), (128, 96, 16, 4), (64, 64, 3, 5),
                                          (128, 128, 32, 16), (64, 16, 32, 16)])
def test_dgrad_and_wgrad_at_small_gradients_vs_fp64(Cin, Cout, H, B):
    """UpConvTC alone, gradients scaled to 1e-7 (far below fp16's normal range: the power-of-two
    pre-scales must carry them): dx of the K = 16*Cout GEMM and dW of the per-parity wgrad (cuBLAS
    fp32 at Cout % 64 != 0) against fp64, 8x the strict-fp32 error or 1e-5. Split-K and unsplit
    launches: deconv6 at B = 16 is split only to keep each accumulator within UPCONV_MAX_KPI chunks,
    and the Cout = 16 case runs its dgrad unsplit over all 4 chunks."""
    from sonet_b200 import train_ops
    g = torch.Generator(device=DEV).manual_seed(Cin + Cout + H)
    x = torch.randn(B, Cin, H, H, device=DEV, generator=g)
    W = torch.randn(Cout, Cin, 3, 3, device=DEV, generator=g) * (2.0 / (9 * Cin)) ** 0.5
    b = torch.randn(Cout, device=DEV, generator=g)
    dz = torch.randn(B, Cout, 2 * H, 2 * H, device=DEV, generator=g) * 1e-7
    _, dx64, dW64 = _conv_grads64(x, W, b, dz)
    xs, Ws, bs = (t.clone().requires_grad_(True) for t in (x, W, b))
    with flags(False):
        train_ops.ConvStrict.apply(F.interpolate(xs, scale_factor=2), Ws, bs, [1, 1], [1, 1], [1, 1],
                                   1).backward(dz)
    xk, Wk, bk = (t.clone().requires_grad_(True) for t in (x, W, b))
    train_ops.UpConvTC.apply(xk, Wk, bk).backward(dz)
    for n, got, s32, r64 in (("dx", xk.grad, xs.grad, dx64), ("dW", Wk.grad, Ws.grad, dW64)):
        rows = (lambda t: t.transpose(0, 1).reshape(t.shape[1], -1)) if n == "dx" else \
            (lambda t: t.reshape(t.shape[0], -1))
        e = row_rel_err(rows(got), rows(r64))
        e32 = row_rel_err(rows(s32), rows(r64))
        print("\n[upconv-grad] Cin %d Cout %d %dx%d: %s %.2e (fp32 %.2e)" % (Cin, Cout, H, H, n,
                                                                       float(e.max()), float(e32.max())))
        assert bool((e <= torch.clamp(8 * e32, min=1e-5)).all()), n


def test_device_packed_groups_match_the_host_pack():
    from sonet_b200 import ops, train_ops
    g = torch.Generator(device=DEV).manual_seed(7)
    Wg = torch.randn(4, 128, 4 * 96, device=DEV, generator=g) * 0.03
    Wg[2, 5, 7] = 3.0                                       # the common scale comes from one group
    blob_h, per_h, inv_h = ops.pointwise_tc_pack_groups(Wg)
    blob_d, per_d, scale2 = train_ops._pack_groups_device(Wg)
    assert per_h == per_d
    assert torch.equal(blob_d.cpu(), blob_h)
    assert float(scale2[1]) == inv_h
    x = torch.randn(4 * 2, 4 * 96, 64, device=DEV, generator=g)
    y_h = ops.pointwise_tc_grouped(x, blob_h.to(DEV), per_h, inv_h, None, 128, None, groups=4)
    y_d = torch.empty_like(y_h)
    ops._call("sonet_pointwise_tc_grouped_forward_dev", x.data_ptr(), 4 * 96, 2, 64, blob_d.data_ptr(),
              per_d, scale2[1:].data_ptr(), None, 128, 0, 4, 1, 0, 0, 64, 2 * 128 * 64, y_d.data_ptr(),
              None, ops._stream(x))
    assert torch.equal(y_d, y_h)


def _stage_step(mod, x, w):
    mod.zero_grad()
    xg = x.clone().requires_grad_(True)
    y = mod(xg)
    y.backward(w)
    return [y.detach().clone(), xg.grad.clone()] + [p.grad.clone() for p in mod.parameters()]


def test_route_profile_ineligible_stages_and_determinism(monkeypatch):
    from sonet_b200 import layers, ops, train_ops
    calls = []
    real = train_ops.conv_strict
    monkeypatch.setattr(train_ops, "conv_strict", lambda c, x: calls.append(1) or real(c, x))
    torch.manual_seed(0)
    mod = layers.UpConv(128, 128, activation="relu", normalization="batch").to(DEV).train()
    x = torch.randn(4, 128, 16, 16, device=DEV)
    w = torch.randn(4, 128, 32, 32, device=DEV)
    ops.PROFILE = []
    try:
        a = _stage_step(mod, x, w)
        names = {p[0] for p in ops.PROFILE}
    finally:
        ops.PROFILE = None
    for n in ("sonet_upconv_fold_weights_f32", "sonet_pointwise_tc_pack_groups_device",
              "sonet_pointwise_tc_grouped_forward_dev", "sonet_upconv_dgrad_im2col_f32",
              "sonet_pointwise_tc_forward_dev", "sonet_wgrad_tc_f32"):
        assert n in names, n
    assert not calls, "an eligible stage went through conv_strict"
    b = _stage_step(mod, x, w)
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), "output %d is not bit-identical between two passes" % i
    # ineligible (Cout < 64): the strict-fp32 cuDNN path, as before
    small = layers.UpConv(64, 32, activation="relu", normalization="batch").to(DEV).train()
    _stage_step(small, torch.randn(4, 64, 8, 8, device=DEV), torch.randn(4, 32, 16, 16, device=DEV))
    assert len(calls) == 1


def test_map_size_rule(monkeypatch):
    """At the default UPCONV_MIN_HW, a 16x16 input keeps the strict-fp32 cuDNN path and a 32x32
    input (deconv6) takes the parity GEMMs."""
    from sonet_b200 import layers, train_ops
    monkeypatch.undo()
    assert train_ops.UPCONV_MIN_HW == 1024
    calls = []
    real = train_ops.conv_strict
    monkeypatch.setattr(train_ops, "conv_strict", lambda c, x: calls.append(x.shape[2]) or real(c, x))
    mod = layers.UpConv(128, 128, activation="relu", normalization="batch").to(DEV).train()
    for h in (16, 32):
        _stage_step(mod, torch.randn(2, 128, h, h, device=DEV), torch.randn(2, 128, 2 * h, 2 * h, device=DEV))
    assert calls == [32]                     # the up-sampled 16x16 input, once


def test_enabled_false_restores_the_composition(monkeypatch):
    """ENABLED = False: no new entry runs, the stage is up_sample -> MyConv2d (strict-fp32 cuDNN,
    F.batch_norm, ELU), and its results are bit for bit those of that composition called directly
    (cuDNN in its deterministic mode, so that its weight gradient is reproducible at all)."""
    from sonet_b200 import layers, ops, train_ops
    calls = []
    real = train_ops.conv_strict
    monkeypatch.setattr(train_ops, "conv_strict", lambda c, x: calls.append(1) or real(c, x))
    torch.manual_seed(0)
    mod = layers.UpConv(128, 128, activation="elu", normalization="batch").to(DEV).train()
    ref = copy.deepcopy(mod)
    x = torch.randn(4, 128, 8, 8, device=DEV)
    w = torch.randn(4, 128, 16, 16, device=DEV)
    ops.PROFILE = []
    try:
        with flags(False), torch.backends.cudnn.flags(deterministic=True):
            a = _stage_step(mod, x, w)
        assert not ops.PROFILE, sorted({p[0] for p in ops.PROFILE})
    finally:
        ops.PROFILE = None
    assert len(calls) == 1
    with flags(False), torch.backends.cudnn.flags(deterministic=True):
        xg = x.clone().requires_grad_(True)
        y = ref.conv(ref.up_sample(xg))
        y.backward(w)
    b = [y.detach(), xg.grad] + [p.grad for p in ref.parameters()]
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    assert torch.equal(mod.conv.norm.running_mean, ref.conv.norm.running_mean)


def test_running_statistics_follow_f_batch_norm():
    """Several steps, kernels on vs off: the running statistics the BN kernels' batch moments feed
    match F.batch_norm's to the conv outputs' precision (the conv arithmetic differs)."""
    from sonet_b200 import layers
    torch.manual_seed(0)
    mod = layers.UpConv(128, 128, activation="relu", normalization="batch").to(DEV).train()
    mod.conv.norm.momentum = 0.3
    ref = copy.deepcopy(mod)
    gen = torch.Generator(device=DEV).manual_seed(2)
    for _ in range(4):
        x = torch.randn(4, 128, 8, 8, device=DEV, generator=gen) * 3 + 1
        with flags(True):
            mod(x.requires_grad_(True))
        with flags(False):
            ref(x)
    for n in ("running_mean", "running_var"):
        a, b = getattr(mod.conv.norm, n), getattr(ref.conv.norm, n)
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-5 * float(b.abs().max())), n
    assert mod.conv.norm.momentum == ref.conv.norm.momentum
    assert int(mod.conv.norm.num_batches_tracked) == int(ref.conv.norm.num_batches_tracked)


@pytest.mark.parametrize("B", [16, 32])
def test_whole_decoder_vs_fp64(B):
    """Decoder (feature_num 1024, the FC and conv branches) in train mode with every UpConv stage on
    the parity GEMMs, MyLinear on LinearStrict + the BN kernels and the ConvToPC heads on the 1x1
    train kernels: a fixed linear functional of all its outputs (no nearest-neighbour switching)
    and its gradients, kernels on vs fp64, 8x the strict-fp32 error or 1e-5 per row.
    ELU: the gradient of every stage is then continuous in its input. With ReLU, pre-activations
    within rounding of zero take either gate depending on the arithmetic, and each flipped gate moves
    whole gradient values: through the six-stage chain that difference from fp64 depends on how many
    gates a run flips, not on how well it computes the gradient it chose."""
    from sonet_b200 import networks, synth
    opt = synth.make_opt("autoencoder")
    opt.activation = "elu"
    torch.manual_seed(0)
    dec = networks.Decoder(opt)
    dec.load_state_dict(trained_like_state_dict(dec, seed=3))
    x = torch.randn(B, opt.feature_num, generator=torch.Generator().manual_seed(1))

    def run(dtype, kernels):
        m = copy.deepcopy(dec).to(DEV, dtype).train()
        xg = x.to(DEV, dtype).requires_grad_(True)
        with flags(kernels):
            out = m(xg)
            outs = [out, m.conv_pc4, m.conv_pc5, m.conv_pc6]
            gen = torch.Generator().manual_seed(9)
            loss = sum((o * torch.randn(o.shape, generator=gen).to(DEV, dtype)).sum() for o in outs)
            loss.backward()
        g = {"dx": xg.grad.detach()}
        g.update({n: p.grad.detach() for n, p in m.named_parameters() if p.grad is not None})
        g.update({"out%d" % i: o.detach() for i, o in enumerate(outs)})
        return g
    got, strict, ref = run(torch.float32, True), run(torch.float32, False), run(torch.float64, False)
    worst = (0.0, "")
    for n, r in ref.items():
        if _before_norm(ref, n):
            continue
        rows = lambda t: t.reshape(t.shape[0], -1) if t.dim() > 1 else t.reshape(1, -1)  # noqa: E731
        e = row_rel_err(rows(got[n]), rows(r))
        lim = torch.clamp(8 * row_rel_err(rows(strict[n]), rows(r)), min=1e-5)
        worst = max(worst, (float((e / lim).max()), n))
        assert bool((e <= lim).all()), "%s: relative error %.3e" % (n, float(e.max()))
    print("\n[upconv-train] whole decoder B=%d: worst ratio %.3f (%s)" % ((B,) + worst))


def test_mylinear_train_vs_fp64_and_batch_of_one():
    from sonet_b200 import layers
    torch.manual_seed(0)
    for act, norm in (("relu", "batch"), ("elu", None), (None, None)):
        mod = layers.MyLinear(256, 512, activation=act, normalization=norm)
        _vs_fp64("mylinear-%s-%s" % (act, norm), mod, torch.randn(32, 256))
    mod = layers.MyLinear(16, 8, activation="relu", normalization="batch").to(DEV).train()
    with pytest.raises(ValueError) as got:
        mod(torch.randn(1, 16, device=DEV, requires_grad=True))
    with pytest.raises(ValueError) as want:
        F.batch_norm(torch.randn(1, 8), None, None, training=True)
    assert str(got.value) == str(want.value)


@pytest.mark.parametrize("conv_pc", [1024, 4096])
def test_autoencoder_optimize_step_loss_kernels_on_vs_off(conv_pc):
    """One autoencoder.Model.optimize() with every UpConv stage on the parity GEMMs (the autouse
    fixture; with output_conv_pc_num = 4096 deconv6's backward runs too): the loss within 1e-4
    relative of the kernels-off step."""
    from sonet_b200 import autoencoder, synth
    B, N = 4, 512
    opt = synth.make_opt("autoencoder", batch_size=B, input_pc_num=N, device=DEV,
                         output_conv_pc_num=conv_pc)
    opt.device = torch.device(DEV)
    st = build_states("autoencoder", opt, seed=29)
    inp = synth.synth_inputs(B, N, seed=29)
    losses = []
    for on in (True, False):
        with flags(on):
            m = autoencoder.Model(opt)
            m.encoder.load_state_dict(st["encoder"])
            m.decoder.load_state_dict(st["head"])
            m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
            torch.manual_seed(0)
            m.optimize(epoch=2)
            losses.append(float(m.loss))
    print("\n[upconv-train] optimize() loss kernels on %.7g off %.7g" % tuple(losses))
    assert abs(losses[0] - losses[1]) <= 1e-4 * abs(losses[1])
