"""-m gpu: pins the wgmma encodings the point-MLP kernels rely on — K-major no-swizzle
shared-memory descriptors (LBO/SBO roles) with the A operand in shared memory, and the A-operand
register fragment — with a single-tile GEMM probe against an exact bf16 reference."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _probe(A, Bm, mode, layout, swap):
    from sonet_b200 import _C
    N, K = Bm.shape
    D = torch.zeros(128, N, dtype=torch.float32, device=DEV)
    rc = _C.lib().sonet_debug_tc_probe(A.data_ptr(), Bm.data_ptr(), N, K, mode, layout, swap,
                                       D.data_ptr(), None)
    _C.check(rc, "tc_probe")
    torch.cuda.synchronize()
    return D


def _ref(A, Bm):
    a = A.to(torch.bfloat16).double().cpu()
    b = Bm.to(torch.bfloat16).double().cpu()
    return (a @ b.t()).float()


@pytest.mark.parametrize("N,K", [(64, 64), (128, 128), (64, 32), (16, 256)])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("layout", [0, 1])
def test_tcgen05_probe_matches_bf16_reference(N, K, mode, layout):
    g = torch.Generator(device="cpu").manual_seed(N * 1000 + K)
    A = torch.randn(128, K, generator=g).to(DEV)
    Bm = torch.randn(N, K, generator=g).to(DEV)
    want = _ref(A, Bm)
    got = _probe(A, Bm, mode, layout, swap=0).cpu()
    err = float((got - want).abs().max())
    assert err <= 1e-3 * max(1.0, float(want.abs().max())), \
        "N=%d K=%d mode=%d layout=%d: max abs err %.3e" % (N, K, mode, layout, err)


# ---- the fused wgmma first PointResNet (csrc/pointmlp_tc.cu) -------------------------------------
def _resnet(cin, seed):
    from sonet_b200 import layers, synth
    net = layers.PointResNet(cin, [64, 128, 256, 384], 'relu', 'batch')
    net.load_state_dict(synth.synth_state_dict(net, seed=seed))
    return net.eval()


def _ref_chain(net, x):
    """fp64 restatement of PointResNet.forward in eval mode (models/layers.py:419-432)."""
    import torch.nn.functional as F
    def layer(l, t):
        y = F.conv1d(t, l.conv.weight.double(), l.conv.bias.double())
        if l.normalization == 'batch':
            n = l.norm
            y = (y - n.running_mean.double()[None, :, None]) / torch.sqrt(
                n.running_var.double()[None, :, None] + n.eps) * n.weight.double()[None, :, None] \
                + n.bias.double()[None, :, None]
            y = F.relu(y)
        return y
    x = x.double()
    l0 = layer(net.layers[0], x)
    t = layer(net.layers[2], layer(net.layers[1], l0))
    return layer(net.layers[3], torch.cat((l0, t), 1)).float()


@pytest.mark.parametrize("B,cin,P", [(2, 6, 3072), (1, 6, 1000), (3, 3, 77), (1, 6, 128),
                                     (2, 6, 15000), (150, 6, 129)])
def test_pointresnet_tc_vs_fp64_reference(B, cin, P, monkeypatch):
    from helpers import assert_close
    net = _resnet(cin, seed=B + P)
    g = torch.Generator().manual_seed(P)
    x = torch.randn(B, cin, P, generator=g)
    want = _ref_chain(net, x)
    net = net.to(DEV)
    with torch.no_grad():
        monkeypatch.setenv("SONET_TC", "1")
        got = net(x.to(DEV))
        monkeypatch.setenv("SONET_TC", "0")
        simt = net(x.to(DEV))
    assert got.shape == (B, 384, P)
    assert_close(simt, want, "fp32 CUDA-core path vs fp64")
    assert_close(got, want, "wgmma bf16x3 path vs fp64")
    # the 3-product split should sit around 1e-5, well inside the 1e-4 bar
    e = float(((got.cpu() - want).abs() / want.abs().clamp(min=1)).max())
    assert e < 5e-5, e


def test_pointresnet_tc_repacks_after_weight_update(monkeypatch):
    monkeypatch.setenv("SONET_TC", "1")
    net = _resnet(6, seed=3).to(DEV)
    x = torch.randn(1, 6, 256, device=DEV)
    with torch.no_grad():
        a = net(x)
        net.layers[3].conv.bias.add_(1.0)
        b = net(x)
    assert torch.allclose(b, a + 1.0, atol=1e-5)


# ---- the generic wgmma point-wise layer (csrc/pointwise_tc.cu) ------------------------------------
@pytest.mark.parametrize("B,C0,C1,P,Cout,relu", [
    (2, 387, 0, 576, 512, True),      # KNNModule layer 1 (K padded 387 -> 400)
    (2, 512, 0, 576, 512, True),      # KNNModule layer 2
    (16, 3, 512, 64, 768, True),      # final PointNet layer 1: two sources, 64 rows per cloud
    (16, 768, 0, 64, 1024, False),    # final PointNet layer 2 (bare), 4 out-channel tiles
    (1, 128, 0, 3072, 50, False),     # segmenter layer 5: Cout padded 50 -> 64
    (3, 64, 0, 1000, 128, True),      # ragged row count
    (2, 1024, 0, 1536, 512, True),    # segmenter layer 2
])
def test_pointwise_tc_vs_fp64(B, C0, C1, P, Cout, relu):
    import torch.nn.functional as F
    from helpers import assert_close
    from sonet_b200 import ops
    rs = np.random.RandomState(C0 + P + Cout)
    x0 = torch.from_numpy(rs.normal(size=(B, C0, P)).astype(np.float32))
    x1 = torch.from_numpy(rs.normal(size=(B, C1, P)).astype(np.float32)) if C1 else None
    W = torch.from_numpy((rs.normal(size=(Cout, C0 + C1)) * np.sqrt(2.0 / (C0 + C1))).astype(np.float32))
    shift = torch.from_numpy(rs.normal(size=Cout).astype(np.float32))
    xin = x0 if x1 is None else torch.cat((x0, x1), 1)
    want = F.conv1d(xin.double(), W.double().unsqueeze(2)) + shift.double()[None, :, None]
    want = (F.relu(want) if relu else want).float()
    blob, inv = ops.pointwise_tc_pack(W)
    got = ops.pointwise_layer_tc(x0.to(DEV), blob.to(DEV), inv, shift.to(DEV), Cout, relu,
                                 x1=None if x1 is None else x1.to(DEV))
    assert got.shape == (B, Cout, P)
    assert_close(got, want, "wgmma generic layer vs fp64", 2e-5)


def test_pointwise_tc_gathered_addend():
    import torch.nn.functional as F
    from helpers import assert_close
    from sonet_b200 import ops
    rs = np.random.RandomState(0)
    B, C0, P, Cout, G = 2, 396, 1536, 1024, 64
    x0 = torch.from_numpy(rs.normal(size=(B, C0, P)).astype(np.float32))
    W = torch.from_numpy((rs.normal(size=(Cout, C0)) / 20).astype(np.float32))
    add = torch.from_numpy(rs.normal(size=(B, Cout, G)).astype(np.float32))
    gidx = torch.from_numpy(rs.randint(0, G, size=(B, P)).astype(np.int32))
    want = F.relu(F.conv1d(x0.double(), W.double().unsqueeze(2)) +
                  torch.gather(add.double(), 2, gidx.long().unsqueeze(1).expand(B, Cout, P))).float()
    blob, inv = ops.pointwise_tc_pack(W)
    got = ops.pointwise_layer_tc(x0.to(DEV), blob.to(DEV), inv, None, Cout, True,
                                 addend=add.to(DEV), gidx=gidx.to(DEV))
    assert_close(got, want, "wgmma layer + gathered addend", 2e-5)


# ---- fused pool path: node-sorted copies -> wgmma PointResNet -> per-node max ---------------------
@pytest.mark.parametrize("B,N,mode", [(3, 1024, "sampled"), (2, 700, "uniform"), (2, 5000, "sampled")])
def test_fused_pool_matches_unfused_path(B, N, mode, monkeypatch):
    """first_pn_out_masked_max from the fused kernel == index_max(+gather) over the materialised
    first_pn_out of the same wgmma PointResNet (bit-exact: same MMAs, max is order-free), incl.
    empty nodes (feature of stacked copy 0) — models/networks.py:181-185."""
    from sonet_b200 import ops, synth
    monkeypatch.setenv("SONET_TC", "1")
    net = _resnet(6, seed=N).to(DEV)
    inp = synth.synth_inputs(B, N, 64, seed=N, node_mode=mode)
    x, sn, node = inp["pc"].to(DEV), inp["sn"].to(DEV), inp["node"].to(DEV)
    if mode == "uniform":
        node[:, :, 3:9] += 50.0          # six nodes nobody is near: empty nodes
    a = ops.som_assign(x, node, 3)
    if mode == "uniform":
        assert int((a["count"] == 0).sum()) >= 6 * B, "case must exercise empty nodes"
    with torch.no_grad():
        x_aug, _ = ops.som_decenter(x, sn, a["cluster_mean"], a["min_idx_i32"], 3)
        full = net(x_aug)
        _, want = ops.index_max(full, a["min_idx_i32"], 64, with_values=True)
        xs, ns, p0 = ops.som_sort_decenter(x, sn, a["cluster_mean"], a["min_idx_i32"], a["count"], 3)
        blob, fpar = net._tc_params()
        got = ops.pointresnet_tc_pool(xs, blob, fpar, ns, p0, 64)
        again = ops.pointresnet_tc_pool(xs, blob, fpar, ns, p0, 64)   # keys self-reset
    # sorted order really is grouped by node and a permutation of the stacked copies
    assert bool((ns[:, 1:] >= ns[:, :-1]).all())
    assert torch.equal(torch.bincount(ns[0].long(), minlength=64), a["count"][0].long())
    assert torch.equal(got, want)
    assert torch.equal(again, want)


def test_encoder_fused_and_lazy_attributes(monkeypatch):
    from helpers import assert_close, build_states
    from sonet_b200 import classifier, synth
    monkeypatch.setenv("SONET_TC", "1")
    opt = synth.make_opt("classifier", batch_size=4, input_pc_num=512, device=DEV)
    st = build_states("classifier", opt, seed=5)
    inp = synth.synth_inputs(4, 512, seed=5)
    m = classifier.Model(opt)
    m.encoder.load_state_dict(st["encoder"])
    m.classifier.load_state_dict(st["head"])
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    m.encoder.fuse_pool = True
    m.test_model()
    fused = m.score.clone()
    assert m.encoder._first_pn_out is None                       # never materialised
    lazy = m.encoder.first_pn_out                                # ... until somebody asks
    assert lazy.shape == (4, 384, 1536) and m.encoder.x_decentered.shape == (4, 3, 1536)
    m.encoder.fuse_pool = False
    m.test_model()
    # the fused path sums the cluster means in sorted-row order (som_group_kernel), the unfused one
    # in stacked order (som_stats_kernel): both fixed, equal to fp32 rounding of a 5000-term sum
    assert_close(m.encoder.first_pn_out, lazy, "lazy vs materialised first_pn_out", 1e-5)
    assert_close(fused, m.score, "fused vs unfused scores", 1e-5)
