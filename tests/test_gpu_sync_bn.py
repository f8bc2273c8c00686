"""-m gpu: the synchronised BatchNorm of data-parallel training (csrc/train.cu:
sonet_bn_cloud_partials_f32, sonet_bn_sync_forward_f32 / _backward_f32) in one process.

  * shard invariance: the records of every shard of a batch, concatenated in cloud order and folded
    by each shard's sync forward / backward, give torch.equal y, mean, var, invstd, dx, dgamma and
    dbeta to the unsplit call, at every shape, activation and split;
  * accuracy: BNActTrain on the per-cloud route (a one-process exchange installed) against fp64
    F.batch_norm with the error bars of the existing BatchNorm test (test_gpu_train_parity.py),
    which includes channels at mean/std = 1e3 and 1e4 and constant channels; plus P = 1 at B = 2;
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


# ---- accuracy: the per-cloud route through BNActTrain against fp64 ------------------------------------
@pytest.fixture
def per_cloud_route():
    """Install a one-process exchange (the identity, as DataParallelTraining installs without a
    process group) whose global batch follows each call's B."""
    from sonet_b200 import train_ops

    class _Identity:
        def global_rows(self, B):
            return B

        def gather(self, rec):
            return rec

    prev = train_ops.EXCHANGE
    train_ops.EXCHANGE = _Identity()
    yield
    train_ops.EXCHANGE = prev


import test_gpu_train_parity as parity  # noqa: E402  (the existing BatchNorm test's bars)

ACC_SHAPES = parity.BN_SHAPES + [("p1_b2", 2, 64, 1, True), ("p1_b2_linear", 2, 64, 1, False)]


@pytest.mark.parametrize("name,B,C,P,relu", ACC_SHAPES, ids=[s[0] for s in ACC_SHAPES])
def test_per_cloud_route_vs_fp64(per_cloud_route, name, B, C, P, relu):
    """test_gpu_train_parity.test_bn_train_vs_fp64 (fp64 reference, its bars, bit-reproducibility,
    var == 0 and invstd == 1/sqrt(eps) on constant channels) with BNActTrain on the per-cloud route."""
    from sonet_b200 import train_ops
    assert train_ops.EXCHANGE is not None
    parity.test_bn_train_vs_fp64(name, B, C, P, relu)
