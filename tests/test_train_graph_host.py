"""Host side of GraphedModel.enable_train_graph (no GPU): which steps take the graph path, what
changes the re-capture key and what leaves it alone, the optimizers' capturable conversion, and
the BatchNorm momentum the key reads."""
import pytest
import torch

from sonet_b200 import classifier, layers, synth, train_ops


def _model(**over):
    opt = synth.make_opt("classifier", batch_size=2, input_pc_num=64, device="cpu", **over)
    m = classifier.Model(opt)
    m._optim = m._make_optimizers()
    return m


def test_cpu_model_never_takes_the_graph_path():
    m = _model()
    m.enable_train_graph(True)
    assert not m._use_train_graph and not m._train_graph_applies()


def test_eager_cases():
    m = _model()
    m._use_train_graph = True            # as enable_train_graph sets it on a CUDA device
    assert m._train_graph_applies()
    m.opt.random_pc_dropout_lower_limit = 0.5
    assert not m._train_graph_applies()
    m.opt.random_pc_dropout_lower_limit = 1
    prev, train_ops.EXCHANGE = train_ops.EXCHANGE, object()
    try:
        assert not m._train_graph_applies()
    finally:
        train_ops.EXCHANGE = prev
    assert m._train_graph_applies()
    m.enable_train_graph(False)
    assert not m._train_graph_applies()


def test_key_changes(monkeypatch):
    m = _model(bn_momentum_decay_step=2)
    s = m._sets[m._cur]
    base = m._train_key(s, 1)
    assert m._train_key(s, 1) == base
    assert m._train_key(s, None) == base          # no decay before epoch 1: the current momentum
    assert m._train_key(s, 2) != base             # a decay-step epoch crossed
    assert m._train_key(s, 3) == m._train_key(s, 2)

    def changed(edit, undo):
        edit()
        try:
            return m._train_key(s, 1) != base
        finally:
            undo()
            assert m._train_key(s, 1) == base

    g = m._optim[0].param_groups[0]
    assert changed(lambda: g.update(lr=2e-3), lambda: g.update(lr=1e-3))
    assert changed(lambda: g.update(betas=(0.8, 0.999)), lambda: g.update(betas=(0.9, 0.999)))
    assert changed(lambda: g.update(eps=1e-7), lambda: g.update(eps=1e-8))
    assert changed(lambda: g.update(weight_decay=1e-4), lambda: g.update(weight_decay=0))
    assert changed(lambda: setattr(m.opt, "dropout", 0.0), lambda: setattr(m.opt, "dropout", 0.7))
    fc = m.classifier.fc1
    assert changed(lambda: setattr(fc, "activation", "elu"), lambda: setattr(fc, "activation", "relu"))
    w = fc.linear.weight
    assert changed(lambda: w.requires_grad_(False), lambda: w.requires_grad_(True))
    assert changed(lambda: setattr(train_ops, "ENABLED", False), lambda: setattr(train_ops, "ENABLED", True))
    bn = fc.norm
    assert m._train_key(s, 1) == base
    bn.momentum = 0.05                   # a decay-step epoch sets it, whatever it was before
    assert m._train_key(s, 1) == base and m._train_key(s, None) != m._train_key(s, 1)
    bn.momentum = 0.1
    old = w.data
    assert changed(lambda: setattr(w, "data", old.clone()), lambda: setattr(w, "data", old))
    st = m._optim[1].state
    assert changed(lambda: setattr(m._optim[1], "state", type(st)()),
                   lambda: setattr(m._optim[1], "state", st))
    monkeypatch.setenv("SONET_TRAIN_TC", "fp16")
    assert m._train_key(s, 1) != base
    monkeypatch.setenv("SONET_TRAIN_TC", "1")       # any other value is the default mode
    assert m._train_key(s, 1) == base
    monkeypatch.delenv("SONET_TRAIN_TC")
    # the input shapes
    m.set_input(torch.zeros(3, 3, 64), torch.zeros(3, 3, 64), torch.zeros(3, dtype=torch.int64),
                torch.zeros(3, 3, 64), torch.zeros(3, 64, 9, dtype=torch.int64))
    assert m._train_key(m._sets[m._cur], 1) != m._train_key(m._sets[m._cur ^ 1], 1)
    # tensor versions are not part of the key
    with torch.no_grad():
        w.add_(1.0)
    assert m._train_key(s, 1) == base


def test_make_capturable_carries_adam_state_over():
    m = _model()
    p = next(m.encoder.parameters())
    st = m._optim[0].state[p]
    st["step"] = torch.tensor(5.0)
    st["exp_avg"] = torch.full_like(p, 0.25)
    st["exp_avg_sq"] = torch.full_like(p, 0.5)
    moments = (st["exp_avg"], st["exp_avg_sq"])
    m._make_capturable()
    for o in m._optim:
        assert o.defaults["capturable"] and all(g["capturable"] for g in o.param_groups)
    assert st["step"].dtype == torch.float32 and float(st["step"]) == 5.0
    assert st["step"].device == p.device
    assert st["exp_avg"] is moments[0] and st["exp_avg_sq"] is moments[1]
    m._make_capturable()                     # already capturable: left as it is
    assert float(st["step"]) == 5.0
    m.enable_train_graph(False)              # ordinary Adams again, `step` a host scalar
    for o in m._optim:
        assert not o.defaults["capturable"] and not any(g["capturable"] for g in o.param_groups)
    assert st["step"].device.type == "cpu" and st["step"].dtype == torch.float32
    assert float(st["step"]) == 5.0 and st["exp_avg"] is moments[0]


@pytest.mark.parametrize("step,decay,epochs", [(None, 0.6, (None, 0, 5)), (2, 0.6, (None, 0, 1, 2, 7, 40)),
                                               (0, 0.6, (3,)), (3, 0.5, (1, 3, 6, 30))])
def test_momentum_at_is_what_a_forward_sets(step, decay, epochs):
    bn = layers.MyBatchNorm1d(4, momentum=0.1, momentum_decay_step=step, momentum_decay=decay)
    bn.train()
    for e in epochs:
        want = bn.momentum_at(e)
        bn(torch.randn(3, 4), e)
        assert bn.momentum == want
        if e is not None and e >= 1 and step:
            assert want == max(0.1 * decay ** (e // step), 0.01)


def test_train_graph_off_by_default():
    m = _model()
    assert not m._use_train_graph and m._train_graphs == {}
