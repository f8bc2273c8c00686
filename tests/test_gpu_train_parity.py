"""-m gpu: the train-mode path against fp64 and against the reference's bookkeeping.

  A. the batch-statistics BatchNorm kernels (csrc/train.cu through train_ops.BNActTrain) against
     fp64 statistics and F.batch_norm + ReLU in fp64, over channels whose |mean|/std spans 0..1e4,
     near-constant and constant channels, variances around eps, gamma = 0 and dead ReLUs, at the
     training shapes and at every branch of the per-cloud record kernels;
  B. every train-mode layer kind (kernels on, PyTorch's default precision flags) against the same
     module in fp64, held to 8x the error of a strict-fp32 run of the PyTorch composition; and the
     whole training step with cuDNN's TF32 flag on and off;
  C. running statistics, momentum and num_batches_tracked against F.batch_norm over several
     epochs, and the whole state_dict after one optimize() step of every wrapper, kernels on / off.
"""
import contextlib
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import build_states, row_rel_err, trained_like_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
EPS = float(np.float32(1e-5))      # the fp32 eps the kernel widens; the fp64 reference uses it too

# Backward error bar of the BatchNorm kernels, in the form of helpers.TC_R: BN_BWD_R times the fp64
# sum of the absolute terms (see _bwd_bars). Measured on one H100 80GB HBM3 (700 W power limit)
# over test_bn_train_vs_fp64 (the run prints "[bn-train] ..."): the largest error was 0.364 x
# 8*2^-24 of the sum (dx, on a channel with var ~ eps); BN_BWD_R is 2.7x that. The forward used
# up to 0.37 of its bar, the statistics 0.12.
BN_BWD_R = 8 * U


@contextlib.contextmanager
def precision_flags(cudnn_tf32, matmul_tf32=False):
    """Set cuDNN's and cuBLAS's TF32 flags (PyTorch's defaults: True, False), restore afterwards."""
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = cudnn_tf32
    torch.backends.cuda.matmul.allow_tf32 = matmul_tf32
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


@contextlib.contextmanager
def train_kernels(on):
    from sonet_b200 import train_ops
    prev = train_ops.ENABLED
    train_ops.ENABLED = on
    try:
        yield
    finally:
        train_ops.ENABLED = prev


# ---- A. batch-statistics BatchNorm against fp64 ------------------------------------------------------
# channel kinds: rs -> (mean, std, gamma, beta); the hardest first (C = 1 takes the first)
def _kind_ratio(r):
    def make(rs):
        s = 10.0 ** rs.uniform(-1, 1)
        return rs.choice((-1.0, 1.0)) * r * s, s, None, None
    return "mean/std=%g" % r, make


KINDS = [
    _kind_ratio(1e4),
    ("near-constant, var >> eps", lambda rs: (rs.choice((-1, 1)) * 1e4 * 10 ** rs.uniform(0, 1), None,
                                              None, None)),
    _kind_ratio(1e3),
    ("constant", lambda rs: (float(rs.normal(0, 30)), 0.0, None, None)),
    _kind_ratio(1e2),
    ("near-constant, var << eps", lambda rs: (rs.choice((-1, 1)) * 10 ** rs.uniform(-1, 2), None,
                                              None, None)),
    _kind_ratio(10),
    ("var ~ eps", lambda rs: (float(rs.normal(0, 0.01)), (EPS * 10 ** rs.uniform(-1, 1)) ** 0.5,
                              None, None)),
    _kind_ratio(0),
    ("gamma = 0", lambda rs: (float(rs.normal(0, 3)), 1.0, 0.0, None)),
    ("beta << 0 (dead ReLU)", lambda rs: (float(rs.normal(0, 3)), 1.0, None, -1e3)),
]


def _bn_case(B, C, P, seed):
    rs = np.random.RandomState(seed)
    kinds = [KINDS[i % len(KINDS)] for i in range(C)]
    kinds = [kinds[i] for i in (rs.permutation(C) if C > 1 else [0])]
    mean, std, gamma, beta = (np.zeros(C) for _ in range(4))
    for c, (_, make) in enumerate(kinds):
        m, s, g, b = make(rs)
        mean[c] = m
        std[c] = 1e-6 * abs(m) if s is None else s
        gamma[c] = rs.choice((-1, 1)) * rs.uniform(0.5, 1.5) if g is None else g
        beta[c] = rs.normal(0, 0.5) if b is None else b
    gen = torch.Generator(device=DEV).manual_seed(seed)
    z = torch.randn(B, C, P, device=DEV, generator=gen, dtype=torch.float64)
    t = lambda a: torch.from_numpy(a).to(DEV)
    x = (t(mean)[None, :, None] + t(std)[None, :, None] * z).float()
    w = torch.randn(B, C, P, device=DEV, generator=gen)
    return x, t(gamma).float(), t(beta).float(), w, [k[0] for k in kinds]


def _per_channel(t):
    """[B,C,P] -> [C, B*P]"""
    return t.transpose(0, 1).reshape(t.shape[1], -1)


def _worst(units, names):
    """(max units, kind of the channel it is in) of a [C, ...] tensor of error / bar."""
    u = units.reshape(units.shape[0], -1).amax(1)
    c = int(u.argmax())
    return float(u[c]), names[c]


def _bwd_bars(x64, mu, invstd, gamma, gref):
    """Absolute-term sums of the backward (BN_BWD_R times them is the bar), all fp64 [B,C,P] / [C]:
    g = dy gated, xh = (x - mean) invstd, r = |mean| invstd (mean is rounded to fp32 before the
    kernel forms xh: an error of up to r 2^-24 in every xh of the channel).
        dbeta  = sum g                       -> S0 = sum |g|
        dgamma = sum g xh                    -> S1 + r S0,  S1 = sum |g xh|
        dx = gamma invstd (g - dbeta/n - xh dgamma/n)
               -> |gamma| invstd (|g| + S0/n + |xh| (S1 + r S0)/n + r S1/n)"""
    n = x64.shape[0] * x64.shape[2]
    is_ = invstd[None, :, None]
    xh = ((x64 - mu[None, :, None]) * is_).abs()
    r = (mu.abs() * invstd)
    G = gref.abs()
    S0 = G.sum((0, 2))
    S1 = (G * xh).sum((0, 2))
    bar_db = S0
    bar_dg = S1 + r * S0
    bar_dx = gamma.abs()[None, :, None] * is_ * (G + (S0 / n)[None, :, None]
                                                 + xh * (bar_dg / n)[None, :, None]
                                                 + (r * S1 / n)[None, :, None])
    return bar_dx, bar_dg, bar_db


def _units(err, bar):
    """err / bar with 0/0 = 0 (an exactly-zero bar demands an exactly-zero error)."""
    return torch.where(bar > 0, err / bar.clamp(min=1e-300), torch.where(err > 0, torch.inf, 0.0))


BN_SHAPES = [
    # name, B, C, P, relu: the training shapes (first PointResNet at N = 5000, KNN module),
    # B = 1 with a long odd row, C = 1, and each branch of the record kernels: a thread per record
    # (P = 1, also at B = 2), a warp (1 < P <= 1024) and a 256-thread CTA (P > 1024), with both
    # sides of the warp / CTA edge
    ("first_pointresnet_n5000", 64, 64, 15000, True),
    ("knn_module", 64, 512, 576, True),
    ("b1_p100003", 1, 16, 100003, False),
    ("p1_b50", 50, 24, 1, True),
    ("c1_split_cap", 70, 1, 999, True),
    ("c600_one_split", 3, 600, 257, False),
    ("b4_split_b", 4, 40, 3000, True),
    ("b4_split_b_linear", 4, 40, 3000, False),
    ("p1_b2", 2, 64, 1, True),
    ("p1_b2_linear", 2, 64, 1, False),
    ("p1024_warp_edge", 5, 48, 1024, True),
    ("p1025_cta_edge", 5, 48, 1025, False),
]


@pytest.mark.parametrize("name,B,C,P,relu", BN_SHAPES, ids=[s[0] for s in BN_SHAPES])
def test_bn_train_vs_fp64(name, B, C, P, relu):
    from sonet_b200 import train_ops
    x, gamma, beta, w, kinds = _bn_case(B, C, P, seed=B * 7 + C * 13 + P)
    runs = []
    for _ in range(2):                                   # the second run: bit-reproducibility
        xg, gg, bg = (t.clone().requires_grad_(True) for t in (x, gamma, beta))
        y, mean, var = train_ops.BNActTrain.apply(xg, gg, bg, EPS, relu)
        invstd = y.grad_fn.saved_tensors[2]
        y.backward(w)
        runs.append([t.detach().clone() for t in (y, mean, var, invstd, xg.grad, gg.grad, bg.grad)])
    for a, b, n in zip(runs[0], runs[1], ("y", "mean", "var", "invstd", "dx", "dgamma", "dbeta")):
        assert torch.equal(a, b), "%s is not bit-reproducible" % n
    y, mean, var, invstd, dx, dgamma, dbeta = runs[0]

    # fp64 reference
    x64 = x.double().requires_grad_(True)
    g64 = gamma.double().requires_grad_(True)
    b64 = beta.double().requires_grad_(True)
    with torch.no_grad():
        var64, mu64 = torch.var_mean(x64, dim=(0, 2), unbiased=False)
        is64 = 1.0 / torch.sqrt(var64 + EPS)
    z64 = F.batch_norm(x64, None, None, g64, b64, True, 0.0, EPS)
    with torch.no_grad():
        xd = x64.detach()
        bar_y = 8 * U * (gamma.double().abs()[None, :, None] * is64[None, :, None]
                         * ((xd - mu64[None, :, None]).abs() + mu64.abs()[None, :, None])
                         + beta.double().abs()[None, :, None])
        y64 = z64.clamp(min=0) if relu else z64
        # the ReLU gate: where the pre-activation is within the forward bar of 0 either side is
        # right, and the reference takes the kernel's (y > 0 iff its pre-activation is > 0)
        gate = torch.where(z64.abs() <= bar_y, y > 0, z64 > 0) if relu else torch.ones_like(y, dtype=torch.bool)
        gref = w.double() * gate
    z64.backward(gref)

    # statistics
    u_var = _units((var.double() - var64).abs(), 8 * U * (var64 + EPS))
    u_is = _units((invstd.double() - is64).abs(), 8 * U * is64)
    u_mu = _units((mean.double() - mu64).abs(), 8 * U * (mu64.abs() + var64.sqrt()))
    const = torch.tensor([k == "constant" for k in kinds], device=DEV)
    fp32_is_eps = float(np.float32(1.0 / np.sqrt(np.float64(EPS))))
    # forward / backward
    u_y = _units((y.double() - y64).abs(), bar_y)
    bdx, bdg, bdb = _bwd_bars(xd, mu64, is64, gamma.double(), gref)
    u_dx = _units((dx.double() - x64.grad).abs(), bdx)
    u_dg = _units((dgamma.double() - g64.grad).abs(), bdg)
    u_db = _units((dbeta.double() - b64.grad).abs(), bdb)
    report = {k: _worst(v, kinds) for k, v in (
        ("var", u_var), ("invstd", u_is), ("mean", u_mu), ("y", u_y.transpose(0, 1)),
        ("dx", u_dx.transpose(0, 1) / (8 * U)), ("dgamma", u_dg / (8 * U)),
        ("dbeta", u_db / (8 * U)))}
    print("\n[bn-train] %s: worst error in units of 8*2^-24 (bwd units: of the abs-term sum x 8*2^-24) "
          % name + ", ".join("%s %.3g (%s)" % (k, u, c) for k, (u, c) in report.items()))
    for k, (u, c) in report.items():
        lim = 1.0 if k in ("var", "invstd", "mean", "y") else BN_BWD_R / (8 * U)
        assert u <= lim, "%s: %.3g x the bar on a '%s' channel" % (k, u / lim, c)
    if bool(const.any()):
        assert bool((var[const] == 0).all()), "constant channels must have var == 0 exactly"
        assert bool((invstd[const] == fp32_is_eps).all()), "constant channels: invstd != 1/sqrt(eps)"


# ---- B. every train-mode layer kind against fp64, under PyTorch's default precision flags ---------
def _layer_cases():
    from sonet_b200 import layers, networks, synth
    opt = synth.make_opt("autoencoder")
    g = torch.Generator().manual_seed(11)
    r = lambda *s: torch.randn(*s, generator=g)

    def equi(cin, cout, B, P):
        return (lambda: layers.EquivariantLayer(cin, cout, 'relu', 'batch'),
                lambda: (r(B, cin, P),))

    def knn_inputs():
        B, M, K, C = 4, 64, 9, 61
        coord = r(B, 3, M)
        d = ((coord[:, :, :, None] - coord[:, :, None, :]) ** 2).sum(1)
        knn_I = torch.argsort(d, dim=2)[:, :, :K]
        return coord, r(B, C, M), knn_I, K, 'avg'

    return {
        "equivariant_6_64_thin": equi(6, 64, 8, 1000),
        "equivariant_64_128_wgmma": equi(64, 128, 8, 1000),
        "equivariant_64_128_200rows": equi(64, 128, 2, 100),
        "myconv2d_1x1_knn": (lambda: layers.MyConv2d(387, 512, 1, activation='relu',
                                                     normalization='batch'),
                             lambda: (r(4, 387, 64, 9),)),
        "convtopc_128_3": (lambda: networks.ConvToPC(128, opt), lambda: (r(4, 128, 16, 16),)),
        "upconv_3x3": (lambda: layers.UpConv(64, 32, activation='relu', normalization='batch'),
                       lambda: (r(4, 64, 8, 8),)),
        "pointresnet": (lambda: layers.PointResNet(6, [64, 128, 256, 384], 'relu', 'batch'),
                        lambda: (r(4, 6, 1000),)),
        "knn_module": (lambda: layers.KNNModule(64, (128, 128), 'relu', 'batch'), knn_inputs),
    }


LAYER_CASES = list(_layer_cases())


def _first(out):
    return out[1] if isinstance(out, tuple) else out      # KNNModule returns (center, feature)


def _layer_run(mod, inputs, dtype, w):
    """One forward + backward of mod (train mode, on DEV, in dtype); returns {name: tensor}."""
    mod = copy.deepcopy(mod).to(DEV, dtype).train()
    args = [a.to(DEV, dtype) if torch.is_tensor(a) and a.is_floating_point() else
            (a.to(DEV) if torch.is_tensor(a) else a) for a in inputs]
    x = args[1] if len(args) > 1 else args[0]
    x.requires_grad_(True)
    y = _first(mod(*args))
    y.backward(w.to(dtype))
    out = {"y": y.detach(), "dx": x.grad.detach()}
    out.update({"d " + n: p.grad.detach() for n, p in mod.named_parameters() if p.grad is not None})
    return out


def _analytically_zero(grads, name):
    """A bias in front of a batch-statistics BN (a per-channel constant the BN removes) has an
    analytically zero gradient: what both arithmetics return is rounding noise."""
    w = name[:-4] + "weight"
    return (name.endswith(".bias") and w in grads
            and float(grads[name].abs().max()) < 1e-3 * float(grads[w].abs().max()))


def _rows(name, t):
    """Compare-ready rows: activations by channel, parameters by output channel."""
    if name in ("y", "dx"):
        return _per_channel(t.reshape(t.shape[0], t.shape[1], -1))
    return t.reshape(1, -1) if t.dim() == 1 else t.reshape(t.shape[0], -1)


@pytest.mark.parametrize("case", LAYER_CASES)
def test_train_layer_vs_fp64_under_default_flags(case):
    make, inputs = _layer_cases()[case]
    torch.manual_seed(0)
    mod = make()
    mod.load_state_dict(trained_like_state_dict(mod, seed=len(case)))
    inp = inputs()
    with torch.no_grad():
        y_shape = _first(copy.deepcopy(mod).to(DEV).train()(*[a.to(DEV) if torch.is_tensor(a) else a
                                                              for a in inp])).shape
    w = torch.randn(y_shape, generator=torch.Generator().manual_seed(5)).to(DEV)
    with precision_flags(cudnn_tf32=True, matmul_tf32=False), train_kernels(True):
        got = _layer_run(mod, inp, torch.float32, w)
    with precision_flags(cudnn_tf32=False, matmul_tf32=False), train_kernels(False):
        strict = _layer_run(mod, inp, torch.float32, w)
    ref = _layer_run(mod, inp, torch.float64, w)
    assert set(got) == set(ref) == set(strict)
    worst = {}
    for n, r64 in ref.items():
        e32 = row_rel_err(_rows(n, strict[n]), _rows(n, r64))
        e = row_rel_err(_rows(n, got[n]), _rows(n, r64))
        if _analytically_zero(ref, n):
            assert float(got[n].abs().max()) < 1e-3 * float(ref[n[:-4] + "weight"].abs().max()), n
            continue
        lim = torch.clamp(8 * e32, min=1e-5)
        worst[n] = (float(e.max()), float(e32.max()))
        bad = e > lim
        assert not bool(bad.any()), "%s %s: row %d has relative error %.3e; strict fp32 %.3e" % (
            case, n, int(bad.nonzero()[0]), float(e[bad][0]), float(e32[bad][0]))
    print("\n[train-layer] %s: " % case + ", ".join("%s %.2e (fp32 %.2e)" % (n, a, b)
                                                    for n, (a, b) in worst.items()))


# ---- the whole classifier step with cuDNN's TF32 flag on and off -------------------------------------
# Largest row error between two runs with the same flags: 2.3e-6; between TF32 on and off: 2.3e-6
# (one H100 80GB HBM3, 700 W power limit). TF32 in a layer shows as 2e-4 to 5e-4.
STEP_TF32_TOL = 1e-5


def _classifier_grads(cudnn_tf32, enabled=True, seed=81):
    from sonet_b200 import classifier, synth
    opt = synth.make_opt("classifier", batch_size=8, input_pc_num=512, device=DEV)
    opt.device = torch.device(DEV)
    st = build_states("classifier", opt, seed=seed)
    inp = synth.synth_inputs(8, 512, seed=seed)
    with precision_flags(cudnn_tf32), train_kernels(enabled):
        m = classifier.Model(opt)
        m.encoder.load_state_dict(st["encoder"])
        m.classifier.load_state_dict(st["head"])
        m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
        m.encoder.train()
        m.classifier.train()
        torch.manual_seed(0)
        m.forward(is_train=True, epoch=3)
        loss = m.softmax_criteria(m.score, m.label)
        m.encoder.zero_grad()
        m.classifier.zero_grad()
        loss.backward()
    grads = {n: p.grad.detach().clone() for mod in (m.encoder, m.classifier)
             for n, p in mod.named_parameters() if p.grad is not None}
    grads["loss"] = loss.detach().reshape(1)
    return grads


def _max_row_err(a, b):
    out = {}
    for n in b:
        if _analytically_zero(b, n):
            continue
        out[n] = float(row_rel_err(_rows("p", a[n]), _rows("p", b[n])).max())
    return out


def test_training_step_independent_of_tf32_flags():
    """Kernels on: the step's gradients with cudnn.allow_tf32 on (PyTorch's default) match those
    with it off to within the run-to-run spread (the gather's scatter_add backward is not
    bit-deterministic), far below TF32's ~1e-3."""
    on = _classifier_grads(True)
    off = _classifier_grads(False)
    again = _classifier_grads(True)
    spread = _max_row_err(again, on)
    diff = _max_row_err(on, off)
    n_sp, n_df = max(spread, key=spread.get), max(diff, key=diff.get)
    print("\n[train-step] run-to-run max row error %.2e (%s); TF32 on vs off %.2e (%s)" % (
        spread[n_sp], n_sp, diff[n_df], n_df))
    assert diff[n_df] <= STEP_TF32_TOL, "%s: TF32 on vs off differ by %.3e" % (n_df, diff[n_df])


# ---- C. running-statistics bookkeeping -----------------------------------------------------------------
def test_running_stats_momentum_and_counter_match_f_batch_norm():
    """conv_bn_act_train (identity conv, so both arms normalise the same tensor) against the
    reference's MyBatchNorm1d.forward (F.batch_norm) over 3 steps at epochs 0, 1, 25 and 60 with
    the momentum decaying to its 0.01 floor."""
    from sonet_b200 import layers, train_ops
    C = 16
    norm_k = layers.MyBatchNorm1d(C, momentum=0.1, momentum_decay_step=10, momentum_decay=0.6).to(DEV)
    norm_r = copy.deepcopy(norm_k)
    eye = torch.eye(C, device=DEV)
    rs = np.random.RandomState(3)
    offs = torch.from_numpy(rs.normal(0, 3, C) * 10 ** rs.uniform(-2, 2, C)).float().to(DEV)
    scale = torch.from_numpy(10 ** rs.uniform(-2, 2, C)).float().to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(3)
    seen = []
    for epoch in (0, 1, 25, 60):
        for step in range(3):
            x = torch.randn(4, C, 777, device=DEV, generator=gen) * scale[None, :, None] + offs[None, :, None]
            x.requires_grad_(True)
            train_ops.conv_bn_act_train(x, eye, None, norm_k, True, epoch)
            norm_r(x, epoch)
            for n in ("running_mean", "running_var"):
                a, b = getattr(norm_k, n), getattr(norm_r, n)
                err = float(((a - b).abs() / b.abs().clamp(min=1e-30)).max())
                assert err <= 1e-6, "epoch %d step %d %s: relative error %.3e" % (epoch, step, n, err)
            assert norm_k.momentum == norm_r.momentum, (epoch, norm_k.momentum, norm_r.momentum)
            assert int(norm_k.num_batches_tracked) == int(norm_r.num_batches_tracked), \
                "num_batches_tracked %d, F.batch_norm leaves %d" % (
                    int(norm_k.num_batches_tracked), int(norm_r.num_batches_tracked))
        seen.append(norm_k.momentum)
    assert seen[0] == seen[1] == 0.1 and seen[-1] == 0.01 and 0.01 < seen[2] < 0.1, seen


@pytest.mark.parametrize("layer", ["equivariant", "myconv2d"])
def test_one_value_per_channel_raises_like_f_batch_norm(layer):
    from sonet_b200 import layers
    if layer == "equivariant":
        mod, x = layers.EquivariantLayer(64, 128, 'relu', 'batch'), torch.randn(1, 64, 1)
    else:
        mod, x = layers.MyConv2d(64, 128, 1, activation='relu', normalization='batch'), torch.randn(1, 64, 1, 1)
    mod = mod.to(DEV).train()
    x = x.to(DEV)
    with train_kernels(False), pytest.raises(ValueError) as want:
        mod(x)
    rm = mod.norm.running_mean.clone()
    with train_kernels(True), pytest.raises(ValueError) as got:
        mod(x)
    msg = "Expected more than 1 value per channel when training"
    assert str(want.value).startswith(msg) and str(got.value).startswith(msg), (want.value, got.value)
    if layer == "equivariant":
        assert str(got.value) == str(want.value)
    assert torch.equal(mod.norm.running_mean, rm)


def _wrapper_step(task, enabled):
    from sonet_b200 import autoencoder, classifier, segmenter, synth
    B, N = 4, 512
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, device=DEV)
    opt.device = torch.device(DEV)
    st = build_states(task, opt, seed=29)
    inp = synth.synth_inputs(B, N, seed=29)
    mod = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}[task]
    head = {"classifier": "classifier", "segmenter": "segmenter", "autoencoder": "decoder"}[task]
    with train_kernels(enabled), precision_flags(cudnn_tf32=enabled):
        m = mod.Model(opt)
        m.encoder.load_state_dict(st["encoder"])
        getattr(m, head).load_state_dict(st["head"])
        if task == "segmenter":
            seg = torch.from_numpy(np.random.RandomState(29).randint(0, 50, size=(B, N)))
            m.set_input(inp["pc"], inp["sn"], inp["label"], seg, inp["node"], inp["node_knn_I"])
        else:
            m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
        torch.manual_seed(0)
        m.optimize(epoch=2)
    mods = (m.encoder, getattr(m, head))
    state = {"%d.%s" % (i, k): v.detach().clone() for i, mm in enumerate(mods)
             for k, v in mm.state_dict().items()}
    grads = {"%d.%s" % (i, k): p.grad.detach().clone() for i, mm in enumerate(mods)
             for k, p in mm.named_parameters() if p.grad is not None}
    before = {"%d.%s" % (i, k): v for i, sd in enumerate((st["encoder"], st["head"]))
              for k, v in sd.items()}
    return state, grads, before, opt.lr


def _adam_first_step_dir(g):
    """Adam's first step is -lr * g / (|g| + 1e-8) (bias-corrected moments m = g, v = g^2)."""
    return g / (g.abs() + 1e-8)


# gradient tolerance of one step, kernels on vs the strict-fp32 PyTorch composition, in units of
# each tensor's largest gradient (test_gpu_train.py: CLASSIFIER_STEP_GRAD_TOL)
STEP_GRAD_TOL = 1e-4


@pytest.mark.parametrize("task", ["classifier", "segmenter", "autoencoder"])
def test_optimize_step_state_dict_kernels_on_vs_off(task):
    """After one optimize(): every buffer (running statistics within 1e-4 of each tensor's scale,
    num_batches_tracked exactly) and every parameter after Adam. A parameter element may differ by
    what Adam makes of a gradient within STEP_GRAD_TOL of its tensor's scale of the reference's; the
    conv biases in front of a batch-statistics BN (gradient analytically zero) by any Adam step.
    The auto-encoder's parameters are held only to the one-Adam-step envelope: its chamfer loss
    picks each point's nearest neighbour, and near-ties switch between the arms (measured: ~80
    elements of the last FC layer take opposite steps, different ones from run to run)."""
    on, g_on, before, lr = _wrapper_step(task, True)
    off, g_off, _, _ = _wrapper_step(task, False)
    assert set(on) == set(off)
    for k, ref in off.items():
        got = on[k]
        if k.endswith("num_batches_tracked"):
            assert torch.equal(got, ref), "%s: %s vs %s" % (k, got, ref)
        elif k.endswith(("running_mean", "running_var")):
            err = float((got - ref).abs().max() / ref.abs().max().clamp(min=1e-30))
            assert err <= 1e-4, "%s: %.3e" % (k, err)
        else:
            if k not in g_off:                          # no gradient: Adam leaves it alone
                assert torch.equal(got, ref), k
                continue
            g = g_off[k].double()
            if _analytically_zero(g_off, k):
                slack = 2 * lr * torch.ones_like(g)
            else:
                eps_g = STEP_GRAD_TOL * g.abs().max()
                d0 = _adam_first_step_dir(g)
                slack = lr * torch.maximum((_adam_first_step_dir(g + eps_g) - d0).abs(),
                                           (_adam_first_step_dir(g - eps_g) - d0).abs())
            p0 = before[k].to(DEV).double()
            bar = 1e-6 * p0.abs().max() + slack
            diff = (got.double() - ref.double()).abs()
            assert bool((diff <= 1e-6 * p0.abs().max() + 2 * lr).all()), k
            if task == "autoencoder":
                continue
            # below 1% of the tensor's largest gradient the sign of an element's first Adam step is
            # not settled by the parity of the two arms; and a max-pool whose arg-max switches
            # between two near-equal points routes a gradient elsewhere (measured: up to 4 elements
            # of a 512x512 weight take opposite steps). Everything else must follow the reference.
            firm = g.abs() >= 1e-2 * g.abs().max()
            bad = firm & (diff > bar)
            assert int(bad.sum()) <= max(4, 1e-4 * g.numel()), "%s: %.3e over the bar (%d elements)" % (
                k, float((diff - bar)[bad].max()), int(bad.sum()))
