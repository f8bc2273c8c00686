"""The fused KNN module (csrc/knn_tc.cu): per-node layer 1 + wgmma layer 2 + max over the K
neighbours, against fp64 with the tensor-core error bars of helpers.py, on both KNNModule routes
(forward and forward_pooled), and the fallback beyond the kernel's limits."""
import pytest
import torch

from helpers import TC_F, TC_R, tc_reference

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
C = 384


def _module(seed):
    from sonet_b200.layers import KNNModule
    torch.manual_seed(seed)
    mod = KNNModule(3 + C, (512, 512), 'relu', 'batch')
    with torch.no_grad():
        for l in mod.layers:
            n = l.conv.out_channels
            l.conv.bias.normal_(0, 0.1)
            l.norm.weight.uniform_(0.5, 1.5)
            l.norm.bias.normal_(0, 0.1)
            l.norm.running_mean.normal_(0, 0.2)
            l.norm.running_var.uniform_(0.5, 2.0)
            assert l.norm.running_var.numel() == n
    return mod.to(DEV).eval()


@torch.no_grad()
def _folded64(mod):
    out = []
    for l in mod.layers:
        W = l.conv.weight.double().view(l.conv.out_channels, -1)
        s = l.norm.weight.double() / torch.sqrt(l.norm.running_var.double() + l.norm.eps)
        out.append((W * s[:, None], (l.conv.bias.double() - l.norm.running_mean.double()) * s
                    + l.norm.bias.double()))
    return out


def _inputs(B, M, K, seed):
    g = torch.Generator().manual_seed(seed)
    coord = torch.rand(B, 3, M, generator=g) * 2 - 1
    x = torch.rand(B, C, M, generator=g) * 2
    d = ((coord.unsqueeze(3) - coord.unsqueeze(2)) ** 2).sum(1)
    knn_I = torch.topk(d, k=K, dim=2, largest=False, sorted=True)[1]
    return coord.to(DEV), x.to(DEV), knn_I.to(DEV)


def _reference(mod, coord, x, knn_I, K, center_type, y_exact=None):
    """fp64 (center, feature) and the feature's error bar: the layer-2 bar plus the layer-1 bar
    carried through |W2| (ReLU and the max over K are 1-Lipschitz). y_exact: Y = W1f x as the
    kernel gets it (the direct-kernel test), else computed here with its tensor-core bar."""
    (W1, s1), (W2, s2) = _folded64(mod)
    pk = mod._tc_params()
    B, _, M = coord.shape
    c64 = coord.double()
    idx = knn_I[:, :, :K]
    nb = torch.gather(c64.unsqueeze(2).expand(B, 3, M, M), 3,
                      idx.unsqueeze(1).expand(B, 3, M, K))               # [B,3,M,K] coord[nbr]
    if center_type == 'avg':
        center = coord.double().new_zeros(B, 3, M)
        for j in range(K):                                              # the kernels' sum order
            center = (center.float() + nb[..., j].float()).double()
        center = (center / K).float().double()   # correctly rounded, as __fdiv_rn
    else:
        center = c64
    dec = (nb.float() - center.float().unsqueeze(3)).double().reshape(B, 3, M * K)
    gidx = idx.reshape(B, 1, M * K)
    if y_exact is None:
        y, m1, f1 = tc_reference(W1[:, 3:].float(), x, w_scale=1 / pk["yinv"], parts=True)
        bar1_node = TC_R * m1 + TC_F * f1
    else:
        y = y_exact.double()
        bar1_node = 4 * 2.0 ** -24 * y.abs()
    yg = torch.gather(y, 2, gidx.expand(B, 512, M * K))
    b1g = torch.gather(bar1_node, 2, gidx.expand(B, 512, M * K))
    pre1 = torch.einsum("oc,bcp->bop", W1[:, :3], dec) + yg + s1[None, :, None]
    m1d = torch.einsum("oc,bcp->bop", W1[:, :3].abs(), dec.abs()) + yg.abs() + s1.abs()[None, :, None]
    h1 = pre1.clamp(min=0)
    bar1 = b1g + 4 * 2.0 ** -24 * m1d                                   # + the fp32 epilogue
    y2, bar2 = tc_reference(W2.float(), h1, shift=s2.float(), w_scale=1 / pk["inv2"])
    bar = bar2 + torch.einsum("oc,bcp->bop", W2.abs(), bar1)
    feat = y2.clamp(min=0).view(B, 512, M, K).max(3)[0]
    fbar = bar.view(B, 512, M, K).max(3)[0]
    return center, feat, fbar


def _profile(fn):
    from sonet_b200 import ops
    ops.PROFILE = []
    try:
        out = fn()
        torch.cuda.synchronize()
        return out, [n for n, _, _, _ in ops.PROFILE]
    finally:
        ops.PROFILE = None


def _check(got, ref, bar, what):
    u = float(((got.double() - ref).abs() / bar).max())
    assert u <= 1.0, "%s: error is %.3g x the tensor-core error bar" % (what, u)


@pytest.mark.parametrize("center_type", ["avg", "center"])
@pytest.mark.parametrize("K", [2, 4, 9])
@pytest.mark.parametrize("M", [16, 64, 121, 256])
def test_knn_module_forward(M, K, center_type):
    mod = _module(M + K)
    B = 3
    coord, x, knn_I = _inputs(B, M, K, seed=M * 31 + K)
    (center, feat), names = _profile(lambda: mod(coord, x, knn_I, K, center_type))
    assert "sonet_knn_mlp_tc_forward" in names and "sonet_rowmax_f32" not in names, names
    c_ref, f_ref, f_bar = _reference(mod, coord, x, knn_I, K, center_type)
    assert torch.equal(center.double(), c_ref)
    _check(feat, f_ref, f_bar, "knn_feature M=%d K=%d %s" % (M, K, center_type))
    center2, feat2 = mod(coord, x, knn_I, K, center_type)
    assert torch.equal(feat, feat2) and torch.equal(center, center2), "re-run differs"


@pytest.mark.parametrize("center_type", ["avg", "center"])
@pytest.mark.parametrize("M,K", [(16, 9), (64, 9), (121, 4), (256, 9), (64, 2)])
def test_knn_module_forward_pooled_with_empty_nodes(M, K, center_type):
    mod = _module(7 * M + K)
    B = 2
    coord, x, knn_I = _inputs(B, M, K, seed=M + 5 * K)
    bits = x.view(torch.int32)
    keys = bits ^ ((bits >> 31) & 0x7fffffff)
    empty = torch.zeros(B, 1, M, dtype=torch.bool, device=DEV)
    empty[:, :, ::5] = True                                             # nodes no point fell in
    keys = torch.where(empty, torch.full_like(keys, -2 ** 31), keys).contiguous()
    p0 = (torch.rand(B, C, device=DEV) * 2).contiguous()
    mm_ref = torch.where(empty, p0.unsqueeze(2).expand(B, C, M), x)
    (center, feat, mm), names = _profile(lambda: mod.forward_pooled(coord, (keys, p0), knn_I, K,
                                                                    center_type))
    assert "sonet_knn_assemble_pool_f32" in names and "sonet_knn_mlp_tc_forward" in names, names
    assert "sonet_pool_finalize" not in names and "sonet_rowmax_f32" not in names, names
    assert torch.equal(mm, mm_ref)
    assert int((keys == -2 ** 31).sum()) == keys.numel(), "keys must be reset"
    c_ref, f_ref, f_bar = _reference(mod, coord, mm_ref, knn_I, K, center_type)
    assert torch.equal(center.double(), c_ref)
    _check(feat, f_ref, f_bar, "pooled knn_feature M=%d K=%d %s" % (M, K, center_type))
    keys2 = torch.where(empty, torch.full_like(keys, -2 ** 31), bits ^ ((bits >> 31) & 0x7fffffff))
    _, feat2, _ = mod.forward_pooled(coord, (keys2.contiguous(), p0), knn_I, K, center_type)
    assert torch.equal(feat, feat2), "re-run differs"


@pytest.mark.parametrize("K", [2, 16])
def test_knn_mlp_tc_kernel(K):
    """ops.knn_mlp_tc on its own, with Y given, center 'center', a knn_I wider than K."""
    from sonet_b200 import ops
    mod = _module(K)
    B, M = 5, 40
    coord, x, knn_I = _inputs(B, M, K + 3, seed=K)
    pk = mod._tc_params()
    y = (torch.randn(B, 512, M, device=DEV) * 3).contiguous()
    out = ops.knn_mlp_tc(coord, coord, knn_I, K, y, pk["w1"], pk["blob2"], pk["inv2"], pk["shift2"])
    _, f_ref, f_bar = _reference(mod, coord, x, knn_I, K, "center", y_exact=y)
    _check(out, f_ref, f_bar, "knn_mlp_tc K=%d" % K)


@pytest.mark.parametrize("M,K", [(64, 1), (64, 17), (256, 10)])
def test_fallback_beyond_limits(M, K):
    mod = _module(3)
    coord, x, knn_I = _inputs(2, M, K, seed=11)
    (center, feat), names = _profile(lambda: mod(coord, x, knn_I, K, "avg"))
    assert "sonet_knn_mlp_tc_forward" not in names and "sonet_rowmax_f32" in names, names
    assert not mod._tc_fused(K, M)
    c_ref, f_ref, f_bar = _reference(mod, coord, x, knn_I, K, "avg")
    _check(feat, f_ref, 2 * f_bar, "fallback M=%d K=%d" % (M, K))
