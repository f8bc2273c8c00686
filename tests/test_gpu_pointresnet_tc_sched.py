"""Tile schedule of the fused first PointResNet (csrc/pointmlp_tc.cu): the per-node max of the pool
variant against the plain variant followed by index_max at every tile remainder, re-runs over
several tiles per SM, and the debug timeline's slot layout and phase order."""
import pytest
import torch

from test_gpu_tc_envelope import DEV, _acts, _gen, _resnet

pytestmark = pytest.mark.gpu

TILE = 128
TL_PHASES = 10   # tile start, act0, layer 1, layer 2, then (MMA retired, epilogue) x 3 chunks
TL_TILES = 6
TL_WAIT = 60


def _case(B, P, M, seed):
    """Seeded network, node-sorted rows and their node ids. Copy 0 is row 0, the point index_max
    falls back to for empty nodes."""
    net = _resnet(6, seed).to(DEV)
    g = _gen(seed)
    x = _acts(B, 6, P, g).to(DEV)
    node = torch.sort(torch.randint(0, M, (B, P), generator=g), dim=1)[0].int().to(DEV)
    pos0 = torch.zeros(B, dtype=torch.int32, device=DEV)
    blob, fpar = net._tc_params()
    return x, node, pos0, blob, fpar


@pytest.mark.parametrize("M", [1, 64, 256])
@pytest.mark.parametrize("P", [129, 280, 255, 384], ids=lambda p: "P%%128=%d" % (p % TILE))
def test_pool_equals_plain_then_index_max(P, M):
    from sonet_b200 import ops
    B = 2
    x, node, pos0, blob, fpar = _case(B, P, M, seed=P * 7 + M)
    got = ops.pointresnet_tc_pool(x, blob, fpar, node, pos0, M)
    full = ops.pointresnet_tc(x, blob, fpar)
    _, want = ops.index_max(full, node, M, with_values=True)
    assert torch.equal(got, want)


def test_rerun_deterministic_over_several_tiles_per_sm():
    from sonet_b200 import ops
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    P, M = 15000, 64
    B = -(-3 * sm // -(-P // TILE)) + 1
    assert B * -(-P // TILE) >= 3 * sm
    x, node, pos0, blob, fpar = _case(B, P, M, seed=3)
    a = ops.pointresnet_tc_pool(x, blob, fpar, node, pos0, M)
    b = ops.pointresnet_tc_pool(x, blob, fpar, node, pos0, M)
    assert torch.equal(a, b)


def test_debug_timeline_layout_and_phase_order():
    """The clock64 entry point computes what the forward computes, and CTA 0 stamps every phase
    of its first tiles in order, per consumer warpgroup."""
    from sonet_b200 import _C, ops
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    B, P, M = 2, 128 * sm * 2 - 50, 64      # 4 tiles per CTA, a partial one at each cloud's end
    x, node, pos0, blob, fpar = _case(B, P, M, seed=9)
    keys_w, p0_w = ops.pointresnet_tc_pool(x, blob, fpar, node, pos0, M, finalize=False)
    want = (keys_w.clone(), p0_w.clone())
    ops.pool_finalize(keys_w, p0_w)
    keys = torch.empty(B, 384, M, dtype=torch.int32, device=DEV)
    _C.check(_C.lib().sonet_pool_keys_init(keys.data_ptr(), keys.numel(), None), "init")
    p0 = torch.empty(B, 384, device=DEV)
    tl = torch.zeros(128, dtype=torch.int64, device=DEV)
    _C.check(_C.lib().sonet_debug_pointresnet_tc_pool_timeline(
        x.data_ptr(), 6, B, P, blob.data_ptr(), fpar.data_ptr(), node.data_ptr(), pos0.data_ptr(), M,
        keys.data_ptr(), p0.data_ptr(), tl.data_ptr(), None), "timeline")
    torch.cuda.synchronize()
    assert torch.equal(keys, want[0]) and torch.equal(p0, want[1])
    t = tl.cpu().tolist()
    tiles = B * -(-P // TILE)
    ntiles = min(-(-tiles // min(tiles, sm)), TL_TILES)
    assert ntiles == 4
    for wg in range(2):
        s = [t[64 * wg + TL_PHASES * i + p] for i in range(ntiles) for p in range(TL_PHASES)]
        assert t[126] < s[0], wg
        assert all(a <= b for a, b in zip(s, s[1:])), (wg, s)
        assert s[-1] < t[127], wg
        assert all(v == 0 for v in t[64 * wg + TL_PHASES * ntiles: 64 * wg + TL_WAIT]), wg
        assert 0 <= t[64 * wg + TL_WAIT] < t[127] - t[126], wg
