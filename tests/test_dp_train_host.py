"""Data-parallel training without a GPU: the synchronised-BatchNorm entries are exported, declared
and bound from the header, and reject bad arguments before any CUDA call; DataParallelTraining
refuses models whose BatchNorm would not be synchronised; and a world-2 gloo run of its gradient
reduction on a toy module, over a ragged global batch of 5, gives both ranks the same gradient,
the gradient of the full-batch mean loss."""
import ctypes
import os
import re
import socket

import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("sonet_bn_cloud_partials_f32", "sonet_bn_sync_forward_f32", "sonet_bn_sync_backward_f32")
P_ = ctypes.c_void_p(16)      # a non-null pointer the checks never dereference


def _partials(lib, B=2, C=8, P=16, act=1, backward=1, x=P_, dy=P_, mean=P_, invstd=P_, rec=P_):
    return lib.sonet_bn_cloud_partials_f32(x, dy, mean, invstd, None, None, B, C, P, act, backward,
                                           rec, None)


def _sync_fwd(lib, Bg=4, B=2, C=8, P=16, act=1, rec=P_, x=P_, y=P_, mean=P_, var=P_, invstd=P_):
    return lib.sonet_bn_sync_forward_f32(rec, x, None, None, Bg, B, C, P, 1e-5, act, y, mean, var,
                                         invstd, None)


def _sync_bwd(lib, Bg=4, B=2, C=8, P=16, act=1, rec=P_, dy=P_, x=P_, mean=P_, invstd=P_, dx=P_,
              dgamma=P_, dbeta=P_):
    return lib.sonet_bn_sync_backward_f32(rec, dy, x, mean, invstd, None, None, Bg, B, C, P, act, dx,
                                          dgamma, dbeta, None)


CALLS = {"sonet_bn_cloud_partials_f32": _partials, "sonet_bn_sync_forward_f32": _sync_fwd,
         "sonet_bn_sync_backward_f32": _sync_bwd}


def test_sync_bn_entries_exported_declared_and_bound(lib_built):
    from sonet_b200 import _C
    h = ctypes.CDLL(lib_built)
    text = open(os.path.join(ROOT, "include", "sonet_b200.h")).read()
    for name in ENTRIES:
        assert hasattr(h, name), name
        assert re.search(r"\b%s\s*\(" % name, text), name
        assert name in _C.EXPORTED_SYMBOLS and name in _C._SIGNATURES
    assert _C._SIGNATURES["sonet_bn_cloud_partials_f32"][-2] is ctypes.c_void_p     # double* rec
    assert _C.CONSTANTS["SONET_BN_REC_FWD"] == 3 and _C.CONSTANTS["SONET_BN_REC_BWD"] == 2


@pytest.mark.parametrize("name", ENTRIES)
@pytest.mark.parametrize("dim,val", [("B", 0), ("B", 65536), ("C", 0), ("C", 65536), ("P", 0)])
def test_rejects_dims_outside_envelope(lib_built, name, dim, val):
    from sonet_b200 import _C
    kw = {dim: val}
    if name != "sonet_bn_cloud_partials_f32" and dim == "B":
        kw["Bg"] = max(val, 1)
    assert CALLS[name](_C.lib(), **kw) == _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    assert "bad dims" in _C.last_error()


@pytest.mark.parametrize("name", ENTRIES[1:])
@pytest.mark.parametrize("Bg,B", [(0, 1), (65536, 2), (3, 4)])
def test_rejects_global_batch_outside_envelope(lib_built, name, Bg, B):
    from sonet_b200 import _C
    assert CALLS[name](_C.lib(), Bg=Bg, B=B) == _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    assert "bad dims" in _C.last_error()


@pytest.mark.parametrize("name", ENTRIES)
@pytest.mark.parametrize("act", [3, -1, 7])
def test_rejects_unknown_activation(lib_built, name, act):
    from sonet_b200 import _C
    assert CALLS[name](_C.lib(), act=act) == _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    assert "activation code %d" % act in _C.last_error()


NULLS = {"sonet_bn_cloud_partials_f32": ("x", "rec", "dy", "mean", "invstd"),
         "sonet_bn_sync_forward_f32": ("rec", "x", "y", "mean", "var", "invstd"),
         "sonet_bn_sync_backward_f32": ("rec", "dy", "x", "mean", "invstd", "dx", "dgamma", "dbeta")}


@pytest.mark.parametrize("name,arg", [(n, a) for n, args in NULLS.items() for a in args])
def test_rejects_null_pointers(lib_built, name, arg):
    from sonet_b200 import _C
    assert CALLS[name](_C.lib(), **{arg: None}) == _C.CONSTANTS["SONET_ERR_BAD_ARG"]
    assert "null pointer" in _C.last_error()


# ---- DataParallelTraining refuses BatchNorms off the train kernels ---------------------------------
def _classifier(**over):
    from sonet_b200 import classifier, synth
    opt = synth.make_opt("classifier", batch_size=2, input_pc_num=64, **over)
    return classifier.Model(opt)


@pytest.mark.parametrize("activation", ["swish", "leakyrelu"])
def test_refuses_activation_off_the_kernels(lib_built, activation):
    from sonet_b200 import dist as sdist, train_ops
    with pytest.raises(RuntimeError, match="does not run on the train kernels"):
        sdist.DataParallelTraining(_classifier(activation=activation), 2)
    assert train_ops.EXCHANGE is None


def test_refuses_disabled_train_kernels(lib_built, monkeypatch):
    from sonet_b200 import dist as sdist, train_ops
    monkeypatch.setattr(train_ops, "ENABLED", False)
    with pytest.raises(RuntimeError, match="train_ops.ENABLED"):
        sdist.DataParallelTraining(_classifier(), 2)
    assert train_ops.EXCHANGE is None


def test_refuses_a_plain_batchnorm(lib_built):
    from sonet_b200 import dist as sdist
    m = torch.nn.Sequential(torch.nn.Linear(4, 4), torch.nn.BatchNorm1d(4))
    with pytest.raises(RuntimeError, match="BatchNorm 1 "):
        sdist.DataParallelTraining(m, 2)


def test_accepts_instance_norm_and_installs_once(lib_built):
    from sonet_b200 import dist as sdist, train_ops
    for norm in ("instance", "batch"):
        m = _classifier(normalization=norm, activation="elu")
        with sdist.DataParallelTraining(m, 2) as dp:
            assert train_ops.EXCHANGE is dp.exchange
            assert dp.exchange.global_rows(2) == 2
            with pytest.raises(RuntimeError, match="shard of the global batch"):
                dp.exchange.global_rows(3)
            with pytest.raises(RuntimeError, match="another instance"):
                sdist.DataParallelTraining(m, 2)
        assert train_ops.EXCHANGE is None


def test_pytorch_batchnorm_refuses_a_train_step_while_installed(lib_built):
    from sonet_b200 import dist as sdist, layers
    bn = layers.MyBatchNorm1d(4).train()
    x = torch.randn(3, 4)
    with sdist.DataParallelTraining(torch.nn.Linear(4, 4), 3):
        with pytest.raises(RuntimeError, match="outside the train kernels"):
            bn(x)
        bn.eval()(x)                       # eval mode normalises by running statistics: no exchange
    bn.train()(x)


# ---- gloo world 2: the gradient reduction ------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _toy(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(5, 7), torch.nn.Tanh(), torch.nn.Linear(7, 3)).double()


def _data(total):
    g = torch.Generator().manual_seed(1)
    return torch.randn(total, 5, generator=g, dtype=torch.float64), \
        torch.randint(0, 3, (total,), generator=g)


def _worker(rank, world, port, total, q):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))
    from sonet_b200 import dist as sdist
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sdist.init_from_env(backend="gloo")
    model = _toy(seed=rank)                  # different on purpose: the broadcast makes them equal
    opt = torch.optim.SGD(model.parameters(), lr=0.0)
    dp = sdist.DataParallelTraining(model, total)
    lo, hi = dp.shard()
    x, y = _data(total)
    loss = torch.nn.functional.cross_entropy(model(x[lo:hi]), y[lo:hi])
    opt.zero_grad()
    loss.backward()
    opt.step()                               # lr 0: the step pre-hook reduced the gradients in place
    grads = [p.grad.numpy().copy() for p in model.parameters()]
    params = [p.detach().numpy().copy() for p in model.parameters()]
    dp.close()
    q.put((rank, hi - lo, grads, params))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


def test_gloo_world2_ragged_gradients_equal_full_batch():
    total = 5
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, total, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict((r[0], r[1:]) for r in (q.get(timeout=180), q.get(timeout=180)))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert (res[0][0], res[1][0]) == (3, 2)
    for a, b in zip(res[0][1] + res[0][2], res[1][1] + res[1][2]):
        assert (a == b).all()                # identical bits on both ranks
    model = _toy(seed=0)                     # rank 0's initialisation, which was broadcast
    x, y = _data(total)
    torch.nn.functional.cross_entropy(model(x), y).backward()
    for p, g in zip(model.parameters(), res[0][1]):
        assert torch.allclose(torch.from_numpy(g), p.grad, rtol=1e-12, atol=1e-15)
