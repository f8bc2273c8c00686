"""The derived-weight caches of the eval fast path: the BatchNorm fold of every layer and the wgmma
packings built from it (generic layer, UpConv, KNN module, first PointResNet, segmenter layer 1).

Host tests (packing runs on the CPU): a pack is built once, rebuilt exactly once per in-place
edit of any tensor it derives from, and then equals byte for byte the pack of a fresh module
loaded with the edited state; writes through `.data` take effect after layers.invalidate().
GPU tests: SONET_TC is honoured at call time by the segmenter, and end to end a model whose
weights were edited in place computes what a freshly loaded one does."""
import pytest
import torch

from sonet_b200 import layers, networks, ops, synth

PACKERS = ("pointwise_tc_pack", "pointwise_tc_pack_groups", "knn_mlp_tc_pack",
           "pointresnet_tc_pack")

# cache owner -> (constructor, sub-module whose tensors the pack derives from, the pack,
#                 packer calls per build)
OWNERS = {
    "EquivariantLayer": (lambda: layers.EquivariantLayer(64, 128, 'relu', 'batch'),
                         lambda m: m, lambda m: m._tc_params(), 1),
    "EquivariantLayer-nobn": (lambda: layers.EquivariantLayer(64, 48, None, None),
                              lambda m: m, lambda m: m._tc_params(), 1),
    "MyConv2d": (lambda: layers.MyConv2d(64, 128, 1, activation='relu', normalization='batch'),
                 lambda m: m, lambda m: m._tc_params(), 1),
    "UpConv": (lambda: layers.UpConv(32, 64, activation='relu', normalization='batch'),
               lambda m: m, lambda m: m._packed(), 2),
    "KNNModule": (lambda: layers.KNNModule(3 + 384, (512, 512), 'relu', 'batch'),
                  lambda m: m, lambda m: m._tc_params(), 2),
    "PointResNet": (lambda: layers.PointResNet(6, [64, 128, 256, 384], 'relu', 'batch'),
                    lambda m: m, lambda m: m._tc_params(), 1),
    "Segmenter": (lambda: networks.Segmenter(synth.make_opt("segmenter")),
                  lambda m: m.layer1, lambda m: m._pack_layer1(12, 16, 384, 1920), 2),
}


@pytest.fixture
def packs(lib_built, monkeypatch):
    """Names of the packer calls made while the test runs."""
    calls = []
    for name in PACKERS:
        def counted(*a, _fn=getattr(ops, name), _name=name, **k):
            calls.append(_name)
            return _fn(*a, **k)
        monkeypatch.setattr(ops, name, counted)
    return calls


def _build(owner, state=None):
    m = OWNERS[owner][0]()
    m.load_state_dict(synth.synth_state_dict(m, seed=1) if state is None else state)
    return m.eval()


def _sources(m, scope):
    """The tensors a module's fold(s) read: weights, biases, BN affine and running statistics."""
    return [(n, t) for n, t in scope(m).state_dict(keep_vars=True).items()
            if not n.endswith("num_batches_tracked")]


def _assert_same(a, b, where="pack"):
    """Equal structure, and tensors equal byte for byte (dtype, shape and device included)."""
    assert type(a) is type(b), where
    if isinstance(a, torch.Tensor):
        assert (a.dtype, a.shape, a.device) == (b.dtype, b.shape, b.device), where
        assert torch.equal(a.contiguous().reshape(-1).view(torch.uint8),
                           b.contiguous().reshape(-1).view(torch.uint8)), where
    elif isinstance(a, dict):
        assert a.keys() == b.keys(), where
        for k in a:
            _assert_same(a[k], b[k], "%s[%r]" % (where, k))
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, "%s[%d]" % (where, i))
    else:
        assert a == b, where


@pytest.mark.parametrize("owner", sorted(OWNERS))
def test_pack_is_built_once(owner, packs):
    _, _, pack, per_build = OWNERS[owner]
    m = _build(owner)
    first = pack(m)
    assert len(packs) == per_build
    assert pack(m) is first
    assert len(packs) == per_build


@pytest.mark.parametrize("owner", sorted(OWNERS))
def test_pack_rebuilds_once_per_in_place_edit(owner, packs):
    _, scope, pack, per_build = OWNERS[owner]
    m = _build(owner)
    pack(m)
    for name, t in _sources(m, scope):
        del packs[:]
        with torch.no_grad():
            t.add_(0.25)
        got = pack(m)
        assert len(packs) == per_build, name
        assert pack(m) is got and len(packs) == per_build, name
        _assert_same(got, pack(_build(owner, m.state_dict())), name)


@pytest.mark.parametrize("owner", sorted(OWNERS))
def test_data_writes_take_effect_after_invalidate(owner, packs):
    _, scope, pack, per_build = OWNERS[owner]
    m = _build(owner)
    stale = pack(m)
    for _, t in _sources(m, scope):
        t.data.add_(0.25)          # `.data` does not bump the tensor's version counter
    assert pack(m) is stale and len(packs) == per_build
    layers.invalidate(m)
    got = pack(m)
    assert len(packs) == 2 * per_build
    _assert_same(got, pack(_build(owner, m.state_dict())))


@pytest.mark.parametrize("make", [lambda: layers.MyLinear(40, 24, 'relu', 'batch'),
                                  lambda: layers.EquivariantLayer(40, 24, 'relu', 'batch'),
                                  lambda: layers.MyConv2d(40, 24, 1, activation='relu',
                                                          normalization='batch'),
                                  lambda: layers.MyLinear(40, 24, None, None)])
def test_fold_refolds_once_per_change(make):
    def fresh(state):
        f = make()
        f.load_state_dict(state)
        return f.eval()

    m = fresh(synth.synth_state_dict(make(), seed=2))
    w, shift = m.folded()
    v = m._folded.version
    wt, _ = m.folded(transpose=True)
    assert torch.equal(wt, w.t())
    assert m.folded()[0] is w and m.folded(transpose=True)[0] is wt and m._folded.version == v
    for name, t in m.state_dict(keep_vars=True).items():
        if name.endswith("num_batches_tracked"):
            continue
        with torch.no_grad():
            t.mul_(1.5)
        got = m.folded()
        assert m._folded.version != v, name
        v = m._folded.version
        assert m.folded()[0] is got[0] and m._folded.version == v, name
        ref = fresh(m.state_dict())
        _assert_same(got, ref.folded(), name)
        _assert_same(m.folded(transpose=True), ref.folded(transpose=True), name)
    next(m.parameters()).data.mul_(2.0)      # `.data` does not bump the version counter
    assert m.folded()[0] is got[0] and m._folded.version == v
    layers.invalidate(m)
    _assert_same(m.folded(), fresh(m.state_dict()).folded())
    assert m._folded.version != v


@pytest.mark.parametrize("normalization", ['batch', None])
def test_upconv_blobs_equal_those_of_the_4d_fold(normalization, lib_built):
    """UpConv folds through its inner MyConv2d's [Cout, Cin*9] fold; the blobs must equal those of
    the fold on the [Cout, Cin, 3, 3] weight restated here."""
    m = layers.UpConv(32, 64, activation='relu', normalization=normalization)
    m.load_state_dict(synth.synth_state_dict(m, seed=4))
    m.eval()
    c = m.conv.conv
    with torch.no_grad():
        w = c.weight.detach().float()
        shift = c.bias.detach().float()
        if normalization == 'batch':
            n = m.conv.norm
            sc = n.weight / torch.sqrt(n.running_var + n.eps)
            shift = (shift - n.running_mean) * sc + n.bias
            w = w * sc[:, None, None, None]
        sets = (((0,), (1, 2)), ((0, 1), (2,)))
        Cout, Cin = w.shape[0], w.shape[1]
        Wg = torch.zeros(4, Cout, 4, Cin)
        for py in range(2):
            for px in range(2):
                for a in range(2):
                    for cc in range(2):
                        acc = 0
                        for dy in sets[py][a]:
                            for dx in sets[px][cc]:
                                acc = acc + w[:, :, dy, dx]
                        Wg[py * 2 + px, :, a * 2 + cc, :] = acc
        blob4, per4, inv4 = ops.pointwise_tc_pack_groups(Wg.view(4, Cout, 4 * Cin))
        W1 = torch.stack([Wg[g, :, (1 - (g >> 1)) * 2 + (1 - (g & 1)), :] for g in range(4)],
                         dim=1).reshape(1, Cout * 4, Cin)
        blob1, per1, inv1 = ops.pointwise_tc_pack_groups(W1)
    want = dict(blob4=blob4, per4=per4, inv4=inv4, blob1=blob1, per1=per1, inv1=inv1,
                shift=shift.contiguous(), shift1=shift.repeat_interleave(4).contiguous())
    _assert_same(m._packed(), want)


# ---- on the GPU --------------------------------------------------------------------------------
DEV = "cuda:0"
HEAD = {"classifier": "classifier", "segmenter": "segmenter", "autoencoder": "decoder"}
OUT = {"classifier": "score", "segmenter": "score_segmenter", "autoencoder": "predicted_pc"}


def _model(task, opt, st):
    from sonet_b200 import autoencoder, classifier, segmenter
    mod = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}[task]
    m = mod.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    getattr(m, HEAD[task]).load_state_dict(st["head"])
    return m


def _case(task, seed=3):
    from helpers import build_states
    opt = synth.make_opt(task, batch_size=2, input_pc_num=512, device=DEV)
    return opt, build_states(task, opt, seed=seed), synth.synth_inputs(2, 512, seed=seed)


def _forward(m, task, inp):
    """set_input + test_model(); returns (output, names of the C-ABI calls made)."""
    keys = ["pc", "sn", "label", "node", "node_knn_I"]
    args = [inp[k] for k in keys]
    if task == "segmenter":
        args.insert(3, torch.zeros(2, 512, dtype=torch.int64))
    m.set_input(*args)
    ops.PROFILE = []
    try:
        m.test_model()
        torch.cuda.synchronize()
        names = [name for name, _, _, _ in ops.PROFILE]
    finally:
        ops.PROFILE = None
    return getattr(m, OUT[task]).clone(), names


@pytest.mark.gpu
def test_segmenter_follows_sonet_tc_at_call_time(monkeypatch):
    opt, st, inp = _case("segmenter")
    m = _model("segmenter", opt, st)
    layer1 = "sonet_pointwise_tc_grouped_forward"    # the node-level GEMM of the split layer 1
    monkeypatch.setenv("SONET_TC", "1")
    _, names = _forward(m, "segmenter", inp)
    assert layer1 in names
    monkeypatch.setenv("SONET_TC", "0")
    exact, names = _forward(m, "segmenter", inp)
    assert not [n for n in names if "_tc_" in n], names
    want, _ = _forward(_model("segmenter", opt, st), "segmenter", inp)
    assert torch.equal(exact, want)
    monkeypatch.setenv("SONET_TC", "1")
    _, names = _forward(m, "segmenter", inp)
    assert layer1 in names


@pytest.mark.gpu
@pytest.mark.parametrize("task", ["classifier", "segmenter", "autoencoder"])
def test_in_place_edits_reach_every_cached_pack(task, monkeypatch):
    """Edit one fold source of every BN-folded layer in place (cycling through weight, bias, BN
    gamma, beta, running mean and var) between two eval forwards: the second forward equals that
    of a model freshly loaded with the edited state."""
    monkeypatch.setenv("SONET_TC", "1")
    opt, st, inp = _case(task)
    m = _model(task, opt, st)
    before, _ = _forward(m, task, inp)
    head = getattr(m, HEAD[task])
    i = 0
    for part in (m.encoder, head):
        for mod in part.modules():
            if isinstance(getattr(mod, "_folded", None), layers._FoldedParams):
                srcs = [t for n, t in mod.state_dict(keep_vars=True).items()
                        if not n.endswith("num_batches_tracked")]
                with torch.no_grad():
                    srcs[i % len(srcs)].mul_(1.03)
                i += 1
    after, _ = _forward(m, task, inp)
    assert not torch.equal(after, before)
    fresh = _model(task, opt, dict(encoder=m.encoder.state_dict(), head=head.state_dict()))
    _forward(fresh, task, inp)
    want, _ = _forward(fresh, task, inp)
    assert torch.equal(after, want)
