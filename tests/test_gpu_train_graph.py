"""-m gpu: optimize() replayed as one CUDA graph (GraphedModel.enable_train_graph).

Equivalence: a graphed model and an eager one (both with capturable Adam) start each step from the
same state. Whether two eager steps from one state are bit-identical is found out first: if they
are, every step's loss, gradients, running statistics, parameters and Adam state must be equal;
if not (torch.gather's backward adds with atomics), the loss and gradients must be within
test_gpu_train.py's bar (1e-4 of each tensor's max; biases whose gradient is analytically zero
stay below 1e-3 of their weight's) or within 4x the spread of two eager steps from one state,
whichever is larger, and the optimizer half must be exact: an eager capturable Adam step on the
replay's own gradients, from the pre-step state, gives the replay's parameters and Adam state bit
for bit. The spread matters under SONET_TRAIN_TC=fp16: one fp16 rounding flipped by a last-bit
difference upstream moved the first layers' weight gradients by up to 8e-4 of their max between
two eager steps on one H100 80GB HBM3 (700 W)."""
import copy

import numpy as np
import pytest
import torch

from helpers import build_states

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4
SHAPES = {"classifier": (4, 512), "segmenter": (4, 256), "autoencoder": (4, 512)}


def _mod(task):
    from sonet_b200 import autoencoder, classifier, segmenter
    return {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}[task]


def _inputs(task, B, N, seed):
    from sonet_b200 import synth
    inp = synth.synth_inputs(B, N, seed=seed)
    args = [inp["pc"], inp["sn"], inp["label"]]
    if task == "segmenter":
        args.append(torch.from_numpy(np.random.RandomState(seed).randint(0, 50, size=(B, N))))
    return args + [inp["node"], inp["node_knn_I"]]


def _make(task, st, B=None, N=None, seed=0, graph=False, capturable=True, **over):
    from sonet_b200 import synth
    B0, N0 = SHAPES[task]
    B, N = B or B0, N or N0
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, device=DEV, **over)
    m = _mod(task).Model(opt)
    enc, head = m._state_modules()
    enc.load_state_dict(st["encoder"])
    head.load_state_dict(st["head"])
    m.set_input(*_inputs(task, B, N, seed))
    m._optim = m._make_optimizers()
    if capturable:
        m._make_capturable()
    if graph:
        m.enable_train_graph(True)
    return m


def _states(task, seed, **over):
    from sonet_b200 import synth
    B, N = SHAPES[task]
    return build_states(task, synth.make_opt(task, batch_size=B, input_pc_num=N, **over), seed=seed)


def _loss(m):
    return m.loss_segmenter if hasattr(m, "segmenter") else m.loss


def _params(m):
    return [(n, p) for sm in m._state_modules() for n, p in sm.named_parameters()]


def _running(m):
    return [(n, b) for sm in m._state_modules() for n, b in sm.named_buffers()
            if n.endswith(("running_mean", "running_var"))]


def _adam(m):
    return [(i, j, k, v) for i, o in enumerate(m._optim) for j, (p, st) in enumerate(o.state.items())
            for k, v in sorted(st.items())]


def _copy_state(dst, src):
    """dst takes src's parameters, buffers and Adam state (copies, not aliases)."""
    with torch.no_grad():
        for a, b in zip(dst._state_modules(), src._state_modules()):
            for x, y in zip(list(a.parameters()) + list(a.buffers()),
                            list(b.parameters()) + list(b.buffers())):
                x.copy_(y)
    for a, b in zip(dst._optim, src._optim):
        a.load_state_dict(copy.deepcopy(b.state_dict()))


def _grads(m):
    return {n: p.grad.detach().clone() for n, p in _params(m) if p.grad is not None}


def _close(a, b, what, tol=TOL):
    scale = float(b.abs().max().clamp(min=1e-12))
    err = float((a.double() - b.double()).abs().max()) / scale
    assert err <= tol, "%s: max|a-b|/max|b| = %.3e > %.1e" % (what, err, tol)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max()) / float(b.abs().max().clamp(min=1e-12))


def _check_grads(got, want, exact, spread=None):
    assert set(got) == set(want) and len(want) > 20
    spread = spread or {}
    for n, gref in want.items():
        g = got[n]
        if exact:
            assert torch.equal(g, gref), n
            continue
        wname = n.rsplit(".", 1)[0] + ".weight"
        if n.endswith(".bias") and wname in want:
            wscale = float(want[wname].abs().max())
            if float(gref.abs().max()) < 1e-3 * wscale:
                assert float(g.abs().max()) < 1e-3 * wscale, n
                continue
        _close(g, gref, "grad " + n, max(TOL, 4 * spread.get(n, 0.0)))


def _step_record(m, epoch):
    m.optimize(epoch)
    torch.cuda.synchronize()
    return dict(loss=_loss(m).detach().clone(), grads=_grads(m),
                running=[b.clone() for _, b in _running(m)])


def _spread(task, st):
    """(bit-identical, {tensor: relative difference}) of two eager steps from one state: the loss,
    the gradients and the parameters after Adam."""
    rec = []
    for _ in range(2):
        m = _make(task, st, dropout=0.0)
        r = _step_record(m, 1)
        r["params"] = [p.detach().clone() for _, p in _params(m)]
        rec.append(r)
    a, b = rec
    exact = (torch.equal(a["loss"], b["loss"]) and all(torch.equal(a["grads"][n], b["grads"][n]) for n in a["grads"])
             and all(torch.equal(x, y) for x, y in zip(a["params"], b["params"])))
    spread = {n: _rel(a["grads"][n], b["grads"][n]) for n in a["grads"]}
    spread["loss"] = _rel(a["loss"], b["loss"])
    return exact, spread


def _shadow_adam_check(m, pre_params, pre_optim):
    """An eager capturable Adam step on m's gradients from the pre-step state gives m's parameters
    and Adam state bit for bit."""
    for o, sd in zip(m._optim, pre_optim):
        params = [p for g in o.param_groups for p in g["params"]]
        shadow = [p.detach().clone() for p in params]
        for sp, p, pre in zip(shadow, params, [pre_params[id(p)] for p in params]):
            sp.copy_(pre)
            sp.grad = None if p.grad is None else p.grad.detach().clone()
        so = torch.optim.Adam(shadow, **{k: v for k, v in o.defaults.items()
                                          if k in ("lr", "betas", "eps", "weight_decay", "amsgrad",
                                                   "capturable")})
        so.load_state_dict(copy.deepcopy(sd))
        so.step()
        for sp, p in zip(shadow, params):
            assert torch.equal(sp, p.detach()), "parameter after the optimizer step"
        for sp, p in zip(shadow, params):
            if p in o.state:
                for k, v in o.state[p].items():
                    assert torch.equal(so.state[sp][k], v), "Adam state " + k


@pytest.mark.parametrize("mode", ["default", "fp16"])
@pytest.mark.parametrize("task", ["classifier", "segmenter", "autoencoder"])
def test_graph_step_matches_eager_step(task, mode, monkeypatch):
    if mode == "fp16":
        monkeypatch.setenv("SONET_TRAIN_TC", "fp16")
    else:
        monkeypatch.delenv("SONET_TRAIN_TC", raising=False)
    st = _states(task, 7, dropout=0.0)
    exact, spread = _spread(task, st)
    eager = _make(task, st, dropout=0.0)
    graphed = _make(task, st, dropout=0.0, graph=True)
    worst = max((v, n) for n, v in spread.items())
    print("\n[train-graph] %s %s: eager steps bit-reproducible: %s, largest spread %.2e (%s)"
          % (task, mode, exact, worst[0], worst[1]))
    for step in range(3):
        if step:
            _copy_state(eager, graphed)      # both arms start the step from the same state
        pre_params = {id(p): p.detach().clone() for _, p in _params(graphed)}
        pre_optim = [copy.deepcopy(o.state_dict()) for o in graphed._optim]
        want = _step_record(eager, 1)
        got = _step_record(graphed, 1)
        g = graphed._train_graphs[graphed._cur]
        assert (g["graph"] is None) == (step == 0), step      # eager warm step, then capture + replay
        if exact:
            assert torch.equal(got["loss"], want["loss"])
        else:
            _close(got["loss"], want["loss"], "loss", max(TOL, 4 * spread["loss"]))
        _check_grads(got["grads"], want["grads"], exact, spread)
        for (n, _), a, b in zip(_running(graphed), got["running"], want["running"]):
            if exact:
                assert torch.equal(a, b), n
            else:
                _close(a, b, n, 1e-5)
        if exact:
            for (n, a), (_, b) in zip(_params(graphed), _params(eager)):
                assert torch.equal(a, b), n
            for a, b in zip(_adam(graphed), _adam(eager)):
                assert a[:3] == b[:3] and torch.equal(a[3], b[3]), a[:3]
        _shadow_adam_check(graphed, pre_params, pre_optim)
    for o in graphed._optim:
        steps = {float(s["step"]) for s in o.state.values()}
        assert steps == {3.0}, steps                 # N calls, N updates


def test_grads_after_replay_are_the_graphs_static_tensors():
    st = _states("classifier", 11, dropout=0.0)
    m = _make("classifier", st, dropout=0.0, graph=True)
    for _ in range(3):
        m.optimize(1)
    g = m._train_graphs[m._cur]
    graph, static = g["graph"], dict(g["grads"])
    checked = [p for p, gr in static.items() if gr is not None]
    assert len(checked) > 20 and all(p.grad is static[p] for p in checked)

    def replay():
        m.optimize(1)
        torch.cuda.synchronize()
        assert m._train_graphs[m._cur]["graph"] is graph           # a replay, no new key
        assert all(p.grad is static[p] for p in checked)
        assert all(torch.isfinite(p.grad).all() for p in checked)

    for sm in m._state_modules():
        sm.zero_grad()
    assert all(p.grad is None for p in checked)
    replay()
    # an eager step in between (a random point dropout keeps the step eager and the graph alive)
    m.opt.random_pc_dropout_lower_limit = 0.5
    m.optimize(1)
    assert all(p.grad is not static[p] for p in checked)
    m.opt.random_pc_dropout_lower_limit = 1
    replay()
    # graph off: ordinary Adams again, `step` carried over as a host scalar
    m.enable_train_graph(False)
    for o in m._optim:
        assert not any(grp["capturable"] for grp in o.param_groups)
        assert {(s["step"].device.type, float(s["step"])) for s in o.state.values()} == {("cpu", 6.0)}
    m.optimize(1)
    for o in m._optim:
        assert {(s["step"].device.type, float(s["step"])) for s in o.state.values()} == {("cpu", 7.0)}


def _recapture_step(m, ref, epoch=1, msg=""):
    """One graphed call that must be an eager warm step of a new key, then one that captures; the
    captured step matches the eager arm from the same state."""
    old = m._train_graphs.get(m._cur, {}).get("graph")
    m.optimize(epoch)
    g = m._train_graphs[m._cur]
    assert g["graph"] is None, msg + ": no new key"
    _copy_state(ref, m)
    want = _step_record(ref, epoch)
    got = _step_record(m, epoch)
    g = m._train_graphs[m._cur]
    assert g["graph"] is not None and g["graph"] is not old, msg
    _close(got["loss"], want["loss"], msg + " loss")
    _check_grads(got["grads"], want["grads"], False)
    graph = g["graph"]
    m.optimize(epoch)
    assert m._train_graphs[m._cur]["graph"] is graph, msg + ": re-captured without a change"


def test_recapture_on_each_key_change(monkeypatch):
    monkeypatch.delenv("SONET_TRAIN_TC", raising=False)
    st = _states("classifier", 13, dropout=0.0, bn_momentum_decay_step=2)
    over = dict(dropout=0.0, bn_momentum_decay_step=2)
    m = _make("classifier", st, graph=True, **over)
    ref = _make("classifier", st, **over)
    m.optimize(1)
    m.optimize(1)
    graph = m._train_graphs[m._cur]["graph"]
    assert graph is not None
    m.optimize(1)
    assert m._train_graphs[m._cur]["graph"] is graph
    for o in m._optim + ref._optim:
        for grp in o.param_groups:
            grp["lr"] = 5e-4
    _recapture_step(m, ref, 1, "lr")
    _recapture_step(m, ref, 2, "bn_momentum_decay_step crossed")
    m.optimize(3)                                        # same momentum: no new key
    assert m._train_graphs[m._cur]["graph"] is not None
    monkeypatch.setenv("SONET_TRAIN_TC", "fp16")
    _recapture_step(m, ref, 3, "SONET_TRAIN_TC=fp16")
    monkeypatch.delenv("SONET_TRAIN_TC")
    _recapture_step(m, ref, 3, "SONET_TRAIN_TC unset")
    for B, N in ((3, 512), (3, 384)):
        for x in (m, ref):
            for _ in range(2):                           # the same input set, resized
                x.set_input(*_inputs("classifier", B, N, 5))
        _recapture_step(m, ref, 3, "B=%d N=%d" % (B, N))


def test_two_input_sets_two_graphs():
    st = _states("classifier", 17, dropout=0.0)
    m = _make("classifier", st, dropout=0.0, graph=True)
    ref = _make("classifier", st, dropout=0.0)
    inp = [_inputs("classifier", 4, 512, s) for s in (1, 2)]
    for rep in range(3):
        for i in (0, 1):
            m.set_input(*inp[i])
            ref.set_input(*inp[i])
            _copy_state(ref, m)
            want = _step_record(ref, 1)
            got = _step_record(m, 1)
            _close(got["loss"], want["loss"], "loss set %d rep %d" % (i, rep))
            _check_grads(got["grads"], want["grads"], False)
    g0, g1 = m._train_graphs[0]["graph"], m._train_graphs[1]["graph"]
    assert g0 is not None and g1 is not None and g0 is not g1


def _eval_equal_fresh(task, m, inp, what):
    """m.test_model() (in m's current eval mode, graph or eager) gives the outputs of a fresh
    wrapper given load_state_dict(m's state), bit for bit."""
    fresh = _mod(task).Model(m.opt)
    for a, b in zip(fresh._state_modules(), m._state_modules()):
        a.load_state_dict(b.state_dict())
    outs = []
    for x in (fresh, m):
        x.set_input(*inp)
        x.test_model()
        outs.append([t.clone() for t in (x.feature, x.score if task == "classifier" else x.predicted_pc)])
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a, b), what


@pytest.mark.parametrize("task", ["classifier", "autoencoder"])
def test_eval_after_graphed_training_sees_the_new_weights(task):
    st = _states(task, 19)
    m = _make(task, st, graph=True)
    train_inp = _inputs(task, *SHAPES[task], 3)
    eval_inp = _inputs(task, *SHAPES[task], 21)
    m.enable_cuda_graph(True)
    _eval_equal_fresh(task, m, eval_inp, "eval graph, start weights")
    for rnd in range(2):
        for _ in range(3):                                 # warm, capture + replay, replay
            m.set_input(*train_inp)
            m.optimize(1)
        # the eval graph captured before these steps, then the eager eval path and its folds;
        # the other way round in round 1
        if rnd == 0:
            _eval_equal_fresh(task, m, eval_inp, "after replays: the earlier eval graph")
            m.enable_cuda_graph(False)
            _eval_equal_fresh(task, m, eval_inp, "after replays: eager eval")
        else:
            m.enable_cuda_graph(False)
            _eval_equal_fresh(task, m, eval_inp, "after replays: eager eval first")
        m.enable_cuda_graph(True)
        _eval_equal_fresh(task, m, eval_inp, "after replays: a new eval graph")
        m.enable_train_graph(False)
        m.set_input(*train_inp)
        m.optimize(1)                                      # an eager step in between
        m.enable_train_graph(True)
        _eval_equal_fresh(task, m, eval_inp, "after an eager step, round %d" % rnd)


def _eval_matches_fresh(task, m, inp, what):
    """m.test_model() on its current input set (no set_input: the train graph's set stays bound)
    gives the outputs of a fresh wrapper given load_state_dict(m's state), bit for bit."""
    fresh = _mod(task).Model(m.opt)
    for a, b in zip(fresh._state_modules(), m._state_modules()):
        a.load_state_dict(b.state_dict())
    fresh.set_input(*inp)
    outs = []
    for x in (fresh, m):
        x.test_model()
        outs.append([t.clone() for t in (x.feature, x.score if task == "classifier" else x.predicted_pc)])
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a, b), what


@pytest.mark.parametrize("task", ["classifier", "autoencoder"])
def test_eval_between_replays_only_sees_the_new_weights(task):
    """Eval, then replays only (no eager warm step, no capture, one input set), then eval again in
    both eval modes: only the replay's version bump tells the BatchNorm folds, the packs and the
    eval graph's key that the weights moved."""
    st = _states(task, 43)
    m = _make(task, st, graph=True)
    inp = _inputs(task, *SHAPES[task], 0)                 # what _make bound
    m.optimize(1)
    m.optimize(1)                                          # warm step, then capture + replay
    cur, graph = m._cur, m._train_graphs[m._cur]["graph"]
    assert graph is not None
    _eval_matches_fresh(task, m, inp, "eager eval after the capture")
    m.enable_cuda_graph(True)
    _eval_matches_fresh(task, m, inp, "eval graph after the capture")

    def replays():
        for _ in range(2):
            m.optimize(1)
        assert m._cur == cur and m._train_graphs[cur]["graph"] is graph

    for rnd in range(2):
        replays()
        _eval_matches_fresh(task, m, inp, "eval graph captured before the replays, round %d" % rnd)
        replays()
        m.enable_cuda_graph(False)
        _eval_matches_fresh(task, m, inp, "eager eval, folds built before the replays, round %d" % rnd)
        m.enable_cuda_graph(True)
        _eval_matches_fresh(task, m, inp, "a new eval graph, round %d" % rnd)


def test_dropout_masks_change_per_replay_and_follow_the_seed():
    st = _states("classifier", 23)
    losses = []
    for run in range(2):
        m = _make("classifier", st, graph=True, lr=0.0)   # lr 0: only the masks move the loss
        torch.manual_seed(5)
        m.optimize(1)
        m.optimize(1)
        seq = []
        for seed in (9, 9):
            torch.manual_seed(seed)
            for _ in range(2):
                m.optimize(1)
                torch.cuda.synchronize()
                seq.append(m.loss.detach().clone())
        assert not torch.equal(seq[0], seq[1]), "two replays drew the same masks"
        assert torch.equal(seq[0], seq[2]) and torch.equal(seq[1], seq[3]), "re-seeding"
        losses.append(seq)
    assert all(torch.equal(a, b) for a, b in zip(*losses)), "two graphed runs"


def _fallback_run(task, st, graph, **over):
    m = _make(task, st, graph=graph, capturable=False, dropout=0.0, **over)
    out = []
    for _ in range(3):
        out.append(_step_record(m, 1))
    assert m._train_graphs == {}
    assert not any(g.get("capturable") for o in m._optim for g in o.param_groups)
    return m, out


def _same_first_step(a, b, exact, spread):
    """Step 1 of two runs from one state (later steps compound the spread through Adam)."""
    x, y = a[0], b[0]
    if exact:
        assert torch.equal(x["loss"], y["loss"])
    _close(x["loss"], y["loss"], "loss", max(TOL, 4 * spread["loss"]))
    _check_grads(x["grads"], y["grads"], exact, spread)


def test_random_point_dropout_stays_eager():
    st = _states("classifier", 29, dropout=0.0)
    exact, spread = _spread("classifier", st)
    _, a = _fallback_run("classifier", st, True, random_pc_dropout_lower_limit=0.5)
    _, b = _fallback_run("classifier", st, False, random_pc_dropout_lower_limit=0.5)
    _same_first_step(a, b, exact, spread)


def test_data_parallel_training_stays_eager(tmp_path):
    import torch.distributed as dist
    from sonet_b200 import dist as sdist
    st = _states("classifier", 31, dropout=0.0)
    exact, spread = _spread("classifier", st)
    dist.init_process_group("gloo", init_method="file://" + str(tmp_path / "store"), rank=0,
                            world_size=1)
    try:
        res = []
        for graph in (True, False):
            m = _make("classifier", st, graph=graph, capturable=False, dropout=0.0)
            with sdist.DataParallelTraining(m, SHAPES["classifier"][0]):
                out = [_step_record(m, 1) for _ in range(3)]
            assert m._train_graphs == {}
            assert not any(g.get("capturable") for o in m._optim for g in o.param_groups)
            res.append(out)
    finally:
        dist.destroy_process_group()
    _same_first_step(*res, exact, spread)


def test_graph_off_launches_what_it_launched_before():
    """enable_train_graph(False) is the eager step: the same C-ABI calls and kernels as a model
    that never enabled it."""
    from sonet_b200 import ops
    st = _states("classifier", 37, dropout=0.0)
    counts = []
    for toggle in (False, True):
        m = _make("classifier", st, dropout=0.0, capturable=False)
        if toggle:
            m.enable_train_graph(True)
            m.enable_train_graph(False)
        m.optimize(1)
        k0, c0 = ops.KERNEL_LAUNCHES, ops.LAUNCHES
        m.optimize(1)
        counts.append((ops.KERNEL_LAUNCHES - k0, ops.LAUNCHES - c0))
    assert counts[0] == counts[1] and counts[0][1] > 50


def test_replay_counts_the_captured_launches():
    from sonet_b200 import ops
    st = _states("classifier", 41, dropout=0.0)
    m = _make("classifier", st, dropout=0.0, graph=True)
    eager = _make("classifier", st, dropout=0.0)
    eager.optimize(1)
    k0, c0 = ops.KERNEL_LAUNCHES, ops.LAUNCHES
    eager.optimize(1)
    want = (ops.KERNEL_LAUNCHES - k0, ops.LAUNCHES - c0)
    for _ in range(3):
        k0, c0 = ops.KERNEL_LAUNCHES, ops.LAUNCHES
        m.optimize(1)
        assert (ops.KERNEL_LAUNCHES - k0, ops.LAUNCHES - c0) == want
