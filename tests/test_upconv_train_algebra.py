"""The algebra of the train-mode up-convolution (nearest x2 up-sampling + 3x3 conv, pad 1) that
csrc/upconv.cu and train_ops.UpConvTC implement, restated in fp64 torch on the CPU and checked
against autograd of F.conv2d(F.interpolate(x, scale_factor=2)): the parity fold and its adjoint,
the forward over the im2col and the horizontal-shift operands, the gathered gradient D and the
dgrad GEMM, and wgrad per parity. Also: argument validation of the new C-ABI entries (no GPU)."""
import pytest
import torch
import torch.nn.functional as F

TAPS = (((0,), (1, 2)), ((0, 1), (2,)))     # [parity][tap] -> kernel rows (columns)


def fold(W):
    """W [Cout,Cin,3,3] -> Wg [4][Cout][4*Cin], Wg[g][co][t*Cin+ci] = the taps (g, t) collects."""
    Cout, Cin = W.shape[:2]
    Wg = torch.zeros(4, Cout, 4, Cin, dtype=W.dtype)
    for g in range(4):
        for t in range(4):
            for ky in TAPS[g >> 1][t >> 1]:
                for kx in TAPS[g & 1][t & 1]:
                    Wg[g, :, t] += W[:, :, ky, kx]
    return Wg.reshape(4, Cout, 4 * Cin)


def fold_dgrad(Wg, Cin):
    """the dgrad matrix [Cin][16*Cout], column (g*4 + t)*Cout + co."""
    Cout = Wg.shape[1]
    return Wg.view(4, Cout, 4, Cin).permute(3, 0, 2, 1).reshape(Cin, 16 * Cout)


def fold_adjoint(dWT):
    """dWT [4][4*Cin][Cout] -> dW [Cout,Cin,3,3]: every tap sums its one entry per parity."""
    _, K, Cout = dWT.shape
    Cin = K // 4
    dW = torch.zeros(Cout, Cin, 3, 3, dtype=dWT.dtype)
    for ky in range(3):
        for kx in range(3):
            for g in range(4):
                t = (ky > (g >> 1)) * 2 + (kx > (g & 1))
                dW[:, :, ky, kx] += dWT[g, t * Cin:(t + 1) * Cin].t()
    return dW


def shifted(x, g, t):
    """x read at [i + a-1+py, j + c-1+px] for all (i, j), zeros outside: [B,C,H,W]."""
    H, W = x.shape[2:]
    oy, ox = (t >> 1) - 1 + (g >> 1), (t & 1) - 1 + (g & 1)
    p = F.pad(x, (1, 1, 1, 1))
    return p[:, :, 1 + oy:1 + oy + H, 1 + ox:1 + ox + W]


def im2col(x):
    """x [B,Cin,H,W] -> xcol [4][B][4*Cin][H*W] (sonet_upconv_im2col_f32)."""
    B, C = x.shape[:2]
    return torch.stack([torch.cat([shifted(x, g, t) for t in range(4)], 1).reshape(B, 4 * C, -1)
                        for g in range(4)])


def conv_mode_operand(x):
    """The im2col-free form: the three horizontal shifts (sonet_upconv_hshift_f32), each tap of
    each parity fetched from block c-1+px+1 at point p + (a-1+py)*W, zeros out of range."""
    B, C, H, W = x.shape
    P = H * W
    hs = torch.stack([F.pad(x, (1, 1))[:, :, :, d:d + W].reshape(B, C, P) for d in range(3)])
    out = torch.zeros(4, B, 4 * C, P, dtype=x.dtype)
    for g in range(4):
        for t in range(4):
            blk = (t & 1) + (g & 1)
            off = ((t >> 1) - 1 + (g >> 1)) * W
            for p in range(P):
                q = p + off
                if 0 <= q < P:
                    out[g, :, t * C:(t + 1) * C, p] = hs[blk, :, :, q]
    return out


def scatter(zg, H, W):
    """[4][B][Cout][H*W] parity planes -> [B,Cout,2H,2W]."""
    _, B, C, _ = zg.shape
    return zg.view(2, 2, B, C, H, W).permute(2, 3, 4, 0, 5, 1).reshape(B, C, 2 * H, 2 * W)


def dgrad_im2col(dz, H, W):
    """dz [B,Cout,2H,2W] -> D [B][16*Cout][H*W] (sonet_upconv_dgrad_im2col_f32)."""
    B, C = dz.shape[:2]
    D = torch.zeros(B, 16, C, H, W, dtype=dz.dtype)
    for g in range(4):
        py, px = g >> 1, g & 1
        plane = dz[:, :, py::2, px::2]
        for t in range(4):
            oy, ox = (t >> 1) - 1 + py, (t & 1) - 1 + px
            # D[i, j] = plane[i - oy, j - ox]
            for i in range(H):
                for j in range(W):
                    if 0 <= i - oy < H and 0 <= j - ox < W:
                        D[:, g * 4 + t, :, i, j] = plane[:, :, i - oy, j - ox]
    return D.reshape(B, 16 * C, H * W)


SHAPES = [  # B, Cin, Cout, H, W
    (2, 3, 5, 1, 1),
    (2, 4, 3, 3, 5),
    (1, 2, 4, 4, 4),
    (3, 3, 2, 2, 6),
    (2, 2, 3, 5, 1),
]


def _case(B, Cin, Cout, H, W):
    g = torch.Generator().manual_seed(B * 1000 + Cin * 100 + Cout * 10 + H * 3 + W)
    x = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    Wt = torch.randn(Cout, Cin, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(Cout, generator=g, dtype=torch.float64, requires_grad=True)
    dz = torch.randn(B, Cout, 2 * H, 2 * W, generator=g, dtype=torch.float64)
    z = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), Wt, b, padding=1)
    z.backward(dz)
    return x.detach(), Wt.detach(), b.detach(), dz, z.detach(), x.grad, Wt.grad, b.grad


@pytest.mark.parametrize("B,Cin,Cout,H,W", SHAPES)
def test_parity_decomposition_matches_autograd(B, Cin, Cout, H, W):
    x, Wt, b, dz, z, dx, dW, db = _case(B, Cin, Cout, H, W)
    Wg = fold(Wt)
    xcol = im2col(x)
    # forward, over both operands
    zg = torch.einsum("gok,gbkp->gbop", Wg, xcol)
    assert torch.allclose(scatter(zg, H, W) + b[None, :, None, None], z, rtol=1e-12, atol=1e-12)
    assert torch.equal(conv_mode_operand(x), xcol)
    # the gathered gradient and the dgrad GEMM (K = 16*Cout)
    D = dgrad_im2col(dz, H, W)
    Wd = fold_dgrad(Wg, Cin)
    assert torch.allclose(torch.einsum("ik,bkp->bip", Wd, D).view_as(x), dx, rtol=1e-12, atol=1e-12)
    # the zero-offset tap of each parity is that parity's plane of dz
    for g in range(4):
        t0 = (1 - (g >> 1)) * 2 + (1 - (g & 1))
        plane = D.view(B, 4, 4, Cout, H * W)[:, g, t0]
        assert torch.equal(plane, dz[:, :, g >> 1::2, g & 1::2].reshape(B, Cout, H * W))
    # wgrad per parity in the [4*Cin][Cout] layout, then the adjoint fold
    dzg = dz.view(B, Cout, H, 2, W, 2).permute(3, 5, 0, 1, 2, 4).reshape(4, B, Cout, H * W)
    dWT = torch.einsum("gbkp,gbop->gko", xcol, dzg)
    assert torch.allclose(fold_adjoint(dWT), dW, rtol=1e-12, atol=1e-12)
    assert torch.allclose(dz.sum((0, 2, 3)), db, rtol=1e-12, atol=1e-12)


def test_fold_adjoint_is_the_transpose_of_the_fold():
    g = torch.Generator().manual_seed(3)
    W = torch.randn(6, 5, 3, 3, generator=g, dtype=torch.float64)
    G = torch.randn(4, 20, 6, generator=g, dtype=torch.float64)      # [4][4*Cin][Cout]
    lhs = (fold(W) * G.transpose(1, 2)).sum()
    rhs = (W * fold_adjoint(G)).sum()
    assert torch.allclose(lhs, rhs, rtol=1e-12)


@pytest.mark.parametrize("B,Cin,Cout", [(2, 3, 5), (4, 7, 2)])
def test_one_pixel_input_is_the_zero_offset_dense_layer(B, Cin, Cout):
    """train_ops.upconv_train on a 1x1 map (here on the CPU, in fp64, through its strict-fp32
    dense branch): the dense layer Cin -> 4*Cout of the zero-offset taps, forward and backward."""
    from sonet_b200 import train_ops
    x, Wt, b, dz, z, dx, dW, db = _case(B, Cin, Cout, 1, 1)
    xg, Wg, bg = (t.clone().requires_grad_(True) for t in (x, Wt, b))
    y = train_ops.upconv_train(xg, Wg, bg)
    assert y.shape == z.shape
    assert torch.allclose(y.detach(), z, rtol=1e-12, atol=1e-12)
    y.backward(dz)
    for got, want in ((xg.grad, dx), (Wg.grad, dW), (bg.grad, db)):
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    Wf = fold(Wt)
    t0 = [(1 - (g >> 1)) * 2 + 1 - (g & 1) for g in range(4)]
    W1 = torch.stack([Wf[g, :, t0[g] * Cin:(t0[g] + 1) * Cin] for g in range(4)], 1)
    assert torch.allclose(torch.einsum("ogi,bi->bog", W1, x.view(B, Cin)) + b[None, :, None],
                          z.view(B, Cout, 4), rtol=1e-12, atol=1e-12)


def test_new_entries_validate_arguments(lib_built):
    """Each new entry rejects bad arguments with SONET_ERR_BAD_ARG and a message before any CUDA
    call (this runs without a GPU)."""
    from sonet_b200 import _C
    lib = _C.lib()
    fold_w = lib.sonet_upconv_fold_weights_f32
    assert fold_w(8, 0, 4, 0, 8, None, None) == -1 and "Cout=0" in _C.last_error()
    assert fold_w(8, 4, 4, 2, 8, None, None) == -1 and "adjoint" in _C.last_error()
    assert fold_w(None, 4, 4, 0, 8, None, None) == -1 and "null" in _C.last_error()
    assert fold_w(8, 4, 4, 0, None, None, None) == -1 and "null" in _C.last_error()
    assert fold_w(8, 4, 4, 1, 8, 8, None) == -1 and "out_dgrad" in _C.last_error()
    dgi = lib.sonet_upconv_dgrad_im2col_f32
    assert dgi(8, -1, 4, 2, 2, 8, None) == -1 and "dimension" in _C.last_error()
    assert dgi(8, 1, 4, 0, 2, 8, None) == -1
    assert dgi(None, 1, 4, 2, 2, 8, None) == -1 and "null" in _C.last_error()
    assert dgi(None, 0, 4, 2, 2, None, None) == 0                         # empty batch: no-op
    pack = lib.sonet_pointwise_tc_pack_groups_device
    assert pack(16, 0, 4, 4, 16, 16, 16, None) == -1 and "G=0" in _C.last_error()
    assert pack(16, 4, 4, 4, None, 16, 16, None) == -1 and "null" in _C.last_error()
    assert pack(16, 4, 4, 4, 24, 16, 16, None) == -1 and "aligned" in _C.last_error()
    gfd = lib.sonet_pointwise_tc_grouped_forward_dev
    assert gfd(16, 64, 2, 64, 16, 0, None, None, 64, 0, 4, 1, 0, 0, 64, 0, 16, None, None) == -1
    assert "inv_scale" in _C.last_error()
    assert gfd(16, 64, 2, 64, 16, 0, 16, None, 64, 7, 4, 1, 0, 0, 64, 0, 16, None, None) == -1
    assert "activation code 7" in _C.last_error()
    assert gfd(16, 64, 2, 64, 16, 0, 16, None, 64, 0, 4, 2, 0, 0, 64, 0, 16, None, None) == -1
    assert "scratch" in _C.last_error()                                  # split-K, no scratch
