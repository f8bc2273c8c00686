"""Work distribution and Y layouts of the fused KNN kernel (csrc/knn_tc.cu): (tile, pass) work items
below, at and above the grid, single and cloud-straddling node blocks, both Y layouts bit for bit,
and the point-major store of the generic wgmma layer that produces the node-major Y."""
import pytest
import torch

from test_gpu_knn_tc import DEV, _check, _inputs, _module, _reference

pytestmark = pytest.mark.gpu


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _items(B, M, K):
    """Work items of one launch: (tile of two floor(64/K)-node blocks, pass over 256 outputs)."""
    npb = 64 // K
    nblocks = (B * M + npb - 1) // npb
    return 2 * ((nblocks + 1) // 2)


def _run(mod, coord, knn_I, K, y_cm, node_major):
    from sonet_b200 import ops
    pk = mod._tc_params()
    y = y_cm.transpose(1, 2).contiguous().transpose(1, 2) if node_major else y_cm
    assert y.stride(1) == (1 if node_major else y.shape[2])
    return ops.knn_mlp_tc(coord, coord, knn_I, K, y, pk["w1"], pk["blob2"], pk["inv2"], pk["shift2"])


def _check_both_layouts(B, M, K, seed):
    mod = _module(seed)
    coord, _, knn_I = _inputs(B, M, K, seed=seed)
    y = (torch.randn(B, 512, M, device=DEV, generator=torch.Generator(DEV).manual_seed(seed)) * 3)
    out_cm = _run(mod, coord, knn_I, K, y, False)
    out_nm = _run(mod, coord, knn_I, K, y, True)
    assert torch.equal(out_cm, out_nm), "node-major and channel-major Y differ"
    assert torch.equal(out_nm, _run(mod, coord, knn_I, K, y, True)), "re-run differs"
    _, f_ref, f_bar = _reference(mod, coord, None, knn_I, K, "center", y_exact=y)
    _check(out_nm, f_ref, f_bar, "knn_mlp_tc B=%d M=%d K=%d" % (B, M, K))


@pytest.mark.parametrize("K", [2, 9, 16])
@pytest.mark.parametrize("M", [16, 64, 121, 256])
def test_layouts_agree_and_match_fp64(M, K):
    _check_both_layouts(3, M, K, seed=M * 17 + K)


@pytest.mark.parametrize("where", ["below", "equal", "above"])
def test_item_count_against_grid(where):
    """Fewer items than SMs, exactly one round, and >= 3 rounds with a ragged last one. M = 64 at
    K = 9 (7-node blocks) also makes blocks straddle two clouds."""
    sm, M, K = _sm_count(), 64, 9
    if where == "below":
        B = 2
        assert _items(B, M, K) < sm
    else:
        cands = [(B, m) for B in range(2, 200) for m in range(16, 257) if m % 7]
        if where == "equal":
            hit = [(B, m) for B, m in cands if _items(B, m, K) == sm - (sm & 1)]
        else:
            hit = [(B, m) for B, m in cands
                   if _items(B, m, K) >= 3 * sm + 2 and _items(B, m, K) % sm != 0]
        assert hit, "no shape gives the wanted item count on %d SMs" % sm
        B, M = hit[0]
    _check_both_layouts(B, M, K, seed=B * 7 + M)


@pytest.mark.parametrize("M,K", [(16, 2), (16, 16), (9, 9)])
def test_single_cloud_few_blocks(M, K):
    """One cloud: a single node block at K = 2, an idle second warpgroup, a partial last block."""
    _check_both_layouts(1, M, K, seed=M + K)


def test_debug_timeline_matches_forward():
    """The clock64 entry point computes the same result and stamps its phases in order."""
    from sonet_b200 import _C, ops
    B, M, K = 4, 64, 9
    mod = _module(5)
    coord, _, knn_I = _inputs(B, M, K, seed=5)
    pk = mod._tc_params()
    y = (torch.randn(B, M, 512, device=DEV) * 3).contiguous()
    want = ops.knn_mlp_tc(coord, coord, knn_I, K, y.transpose(1, 2), pk["w1"], pk["blob2"],
                          pk["inv2"], pk["shift2"])
    out = torch.empty_like(want)
    tl = torch.zeros(128, dtype=torch.int64, device=DEV)
    _C.check(_C.lib().sonet_debug_knn_mlp_tc_timeline(
        coord.data_ptr(), coord.data_ptr(), knn_I.data_ptr(), B, M, K, knn_I.shape[2], y.data_ptr(),
        1, 512, pk["w1"].data_ptr(), pk["blob2"].data_ptr(), pk["inv2"], pk["shift2"].data_ptr(),
        out.data_ptr(), tl.data_ptr(), None), "timeline")
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    t = tl.cpu().tolist()
    assert t[126] < t[0] <= t[1] <= t[2] <= t[3] < t[127]          # CTA 0 runs item 0
    assert t[64] <= t[65] <= t[66] <= t[67] < t[127]


@pytest.mark.parametrize("P", [1, 37, 129, 300])
@pytest.mark.parametrize("Cout,relu,shift", [(512, False, False), (100, True, True),
                                             (130, True, False), (33, False, True)])
def test_pointwise_rows_store_is_the_transpose(P, Cout, relu, shift):
    """pointwise_layer_tc(rows=True) == the channel-major output transposed, bit for bit, at
    ragged point counts and out widths (odd Cout takes the scalar store)."""
    from sonet_b200 import ops
    g = torch.Generator().manual_seed(P * 1000 + Cout)
    B, Cin = 2, 70
    W = torch.randn(Cout, Cin, generator=g)
    x = (torch.randn(B, Cin, P, generator=g) * 2).to(DEV)
    sh = torch.randn(Cout, generator=g).to(DEV) if shift else None
    blob, inv = ops.pointwise_tc_pack(W)
    blob = blob.to(DEV)
    cm = ops.pointwise_layer_tc(x, blob, inv, sh, Cout, relu)
    rows = ops.pointwise_layer_tc(x, blob, inv, sh, Cout, relu, rows=True)
    assert rows.shape == (B, P, Cout)
    assert torch.equal(rows, cm.transpose(1, 2))
    assert torch.equal(rows, ops.pointwise_layer_tc(x, blob, inv, sh, Cout, relu, rows=True))
