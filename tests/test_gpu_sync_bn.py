"""-m gpu: the train-mode BatchNorm's records synchronised as data-parallel training does
(csrc/train.cu: sonet_bn_cloud_partials_f32, sonet_bn_sync_forward_f32 / _backward_f32), in one
process. Its accuracy against fp64 is test_gpu_train_parity.test_bn_train_vs_fp64.

  * shard invariance: the records of every shard of a batch, concatenated in cloud order and folded
    by each shard's sync forward / backward, give torch.equal y, mean, var, invstd, dx, dgamma and
    dbeta to the unsplit call, at every shape, activation and split;
  * reproducibility: two identical calls give identical bits."""
import pytest
import torch

from sonet_b200 import _C, ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ACTS = {"none": 0, "relu": 1, "elu": 2}


def _records(x, act, dy=None, mean=None, invstd=None, gamma=None, beta=None):
    B, C, P = x.shape
    k = _C.CONSTANTS["SONET_BN_REC_BWD" if dy is not None else "SONET_BN_REC_FWD"]
    rec = torch.empty((B, C, k), dtype=torch.float64, device=x.device)
    ops._call("sonet_bn_cloud_partials_f32", _C.ptr(x), _C.ptr(dy), _C.ptr(mean), _C.ptr(invstd),
              _C.ptr(gamma), _C.ptr(beta), B, C, P, act, int(dy is not None), _C.ptr(rec),
              ops._stream(x))
    return rec


def _sync_forward(rec, x, gamma, beta, act, eps=1e-5):
    B, C, P = x.shape
    y = torch.empty_like(x)
    mean, var, invstd = (torch.empty(C, device=x.device) for _ in range(3))
    ops._call("sonet_bn_sync_forward_f32", _C.ptr(rec), _C.ptr(x), _C.ptr(gamma), _C.ptr(beta),
              rec.shape[0], B, C, P, eps, act, _C.ptr(y), _C.ptr(mean), _C.ptr(var), _C.ptr(invstd),
              ops._stream(x))
    return y, mean, var, invstd


def _sync_backward(rec, dy, x, mean, invstd, gamma, beta, act):
    B, C, P = x.shape
    dx = torch.empty_like(x)
    dgamma, dbeta = (torch.empty(C, device=x.device) for _ in range(2))
    ops._call("sonet_bn_sync_backward_f32", _C.ptr(rec), _C.ptr(dy), _C.ptr(x), _C.ptr(mean),
              _C.ptr(invstd), _C.ptr(gamma), _C.ptr(beta), rec.shape[0], B, C, P, act, _C.ptr(dx),
              _C.ptr(dgamma), _C.ptr(dbeta), ops._stream(x))
    return dx, dgamma, dbeta


def _sharded(x, dy, gamma, beta, act, split):
    """Forward and backward as ranks holding `split` consecutive clouds each would run them, the
    gathers being concatenations. Every shard's statistics and parameter gradients must agree."""
    assert sum(split) == x.shape[0]
    bounds = [(sum(split[:i]), sum(split[:i + 1])) for i in range(len(split))]
    shards = [(x[lo:hi].contiguous(), dy[lo:hi].contiguous()) for lo, hi in bounds]
    rec = torch.cat([_records(xs, act) for xs, _ in shards])
    fwd = [_sync_forward(rec, xs, gamma, beta, act) for xs, _ in shards]
    for f in fwd[1:]:
        for a, b in zip(f[1:], fwd[0][1:]):
            assert torch.equal(a, b), "the shards' statistics differ"
    _, mean, var, invstd = fwd[0]
    rec_b = torch.cat([_records(xs, act, ds, mean, invstd, gamma, beta) for xs, ds in shards])
    bwd = [_sync_backward(rec_b, ds, xs, mean, invstd, gamma, beta, act) for xs, ds in shards]
    for b in bwd[1:]:
        assert torch.equal(b[1], bwd[0][1]) and torch.equal(b[2], bwd[0][2]), \
            "the shards' dgamma / dbeta differ"
    y = torch.cat([f[0] for f in fwd])
    dx = torch.cat([b[0] for b in bwd])
    return dict(y=y, mean=mean, var=var, invstd=invstd, dx=dx, dgamma=bwd[0][1], dbeta=bwd[0][2])


def _case(B, C, P, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    off = torch.randn(C, device=DEV, generator=g)[None, :, None] * 10
    scale = torch.rand(C, device=DEV, generator=g)[None, :, None] * 3 + 0.1
    x = off + scale * torch.randn(B, C, P, device=DEV, generator=g)
    dy = torch.randn(B, C, P, device=DEV, generator=g)
    gamma = torch.rand(C, device=DEV, generator=g) + 0.5
    beta = torch.randn(C, device=DEV, generator=g) * 0.5
    return x, dy, gamma, beta


SHAPES = [((8, 64, 15000), [(1, 7), (4, 4), (1, 1, 1, 2, 3)]),
          ((5, 384, 3072), [(1, 4), (2, 3), (1, 1, 1, 2)]),
          ((64, 1024, 1), [(4,) * 16, (1, 63), (31, 33)]),
          ((4, 512, 576), [(1, 3), (2, 2), (1, 1, 1, 1)])]


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("shape,splits", SHAPES, ids=["x".join(map(str, s[0])) for s in SHAPES])
def test_shard_invariance(shape, splits, act):
    x, dy, gamma, beta = _case(*shape, seed=sum(shape))
    whole = _sharded(x, dy, gamma, beta, ACTS[act], (shape[0],))
    again = _sharded(x, dy, gamma, beta, ACTS[act], (shape[0],))
    for k in whole:
        assert torch.equal(whole[k], again[k]), "%s is not bit-reproducible" % k
    for split in splits:
        got = _sharded(x, dy, gamma, beta, ACTS[act], split)
        for k in whole:
            assert torch.equal(got[k], whole[k]), "%s differs at split %s" % (k, split)


@pytest.mark.parametrize("act", list(ACTS))
def test_partial_records_depend_on_their_cloud_only(act):
    """A cloud's records are the same bits in any batch it is part of, and changing one cloud
    leaves the other clouds' records alone."""
    for P in (1, 7, 1024, 1025, 5000):
        x, dy, gamma, beta = _case(6, 32, P, seed=P)
        mean = x.mean((0, 2))
        invstd = 1.0 / (x.var((0, 2), unbiased=False) + 1e-5).sqrt()
        a = _records(x, ACTS[act])
        b = _records(x[2:5].contiguous(), ACTS[act])
        assert torch.equal(a[2:5], b)
        ga = _records(x, ACTS[act], dy, mean, invstd, gamma, beta)
        gb = _records(x[2:5].contiguous(), ACTS[act], dy[2:5].contiguous(), mean, invstd, gamma, beta)
        assert torch.equal(ga[2:5], gb)
        x2 = x.clone()
        x2[3] += 1.0
        c = _records(x2, ACTS[act])
        assert torch.equal(c[:3], a[:3]) and torch.equal(c[4:], a[4:])
        assert not torch.equal(c[3], a[3])


# ---- one route: a single process computes what data-parallel training at world 1 computes ----------
def _one_process_and_world1(run, model, B):
    """run() with no exchange installed, then under DataParallelTraining(model, B) without a process
    group: every tensor it returns must be the same bits."""
    from sonet_b200 import dist as sdist, train_ops
    assert train_ops.EXCHANGE is None
    alone = run()
    with sdist.DataParallelTraining(model, B):
        world1 = run()
    assert train_ops.EXCHANGE is None
    for k in alone:
        assert torch.equal(alone[k], world1[k]), \
            "%s differs between one process and data-parallel training at world 1" % k


def test_layer_step_is_the_same_alone_and_at_world1():
    """A train-mode EquivariantLayer on ConvTC (a wgmma shape: deterministic) with BatchNorm + ReLU:
    forward, backward and running-statistics update."""
    import copy
    from sonet_b200 import layers, ops
    torch.manual_seed(0)
    base = layers.EquivariantLayer(64, 128, 'relu', 'batch').to(DEV).train()
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(8, 64, 1000, device=DEV, generator=g)
    dy = torch.randn(8, 128, 1000, device=DEV, generator=g)
    layer = copy.deepcopy(base)

    def run():
        layer.load_state_dict(base.state_dict())
        layer.zero_grad(set_to_none=True)
        xg = x.clone().requires_grad_(True)
        ops.PROFILE = []
        try:
            y = layer(xg)
            y.backward(dy)
            names = {n for n, _, _, _ in ops.PROFILE}
        finally:
            ops.PROFILE = None
        # the wgmma convolution and the BatchNorm kernels ran
        assert "sonet_wgrad_tc_f32" in names and any(n.startswith("sonet_bn_") for n in names), names
        out = dict(y=y.detach(), dx=xg.grad,
                   running_mean=layer.norm.running_mean.clone(),
                   running_var=layer.norm.running_var.clone())
        out.update({"grad " + k: p.grad.clone() for k, p in layer.named_parameters()})
        return out

    _one_process_and_world1(run, layer, x.shape[0])


BN_ROUTE_CASES = [("relu", (32, 64, 15000)), ("elu", (32, 512, 576)), ("none", (32, 1024, 1))]


@pytest.mark.parametrize("act,shape", BN_ROUTE_CASES, ids=[c[0] for c in BN_ROUTE_CASES])
def test_bn_is_the_same_alone_and_at_world1(act, shape):
    from sonet_b200 import train_ops
    x, dy, gamma, beta = _case(*shape, seed=sum(shape))

    def run():
        xg, gg, bg = (t.clone().requires_grad_(True) for t in (x, gamma, beta))
        y, mean, var = train_ops.BNActTrain.apply(xg, gg, bg, 1e-5, None if act == "none" else act)
        y.backward(dy)
        return dict(y=y.detach(), mean=mean, var=var, dx=xg.grad, dgamma=gg.grad, dbeta=bg.grad)

    _one_process_and_world1(run, torch.nn.Module(), shape[0])
