"""-m gpu: the train-mode device packers (csrc/train.cu) write the same weight blob and scale as
the host packer of the generic wgmma layer (csrc/pointwise_tc.cu) for the same matrix, at every
tile remainder. The blobs start filled with a non-zero byte, so the padding must be written too."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def rand(seed, *shape):
    rs = np.random.RandomState(seed)
    return torch.from_numpy((rs.normal(size=shape) * 10.0 ** rs.uniform(-6, 3)).astype(np.float32))


@pytest.mark.parametrize("transpose", [0, 1])
@pytest.mark.parametrize("cout", [3, 64, 320, 1000])
@pytest.mark.parametrize("cin", [16, 33, 500])
def test_pack_device_equals_host_pack(cout, cin, transpose):
    from sonet_b200 import _C, ops
    W = rand(cout * 1000 + cin, cout, cin)
    Wl = W.t().contiguous() if transpose else W
    n, k = Wl.shape
    blob = torch.full((int(_C.lib().sonet_pointwise_tc_blob_bytes(n, k)),), 0xA5, dtype=torch.uint8,
                      device=DEV)
    scale2 = torch.zeros(2, dtype=torch.float32, device=DEV)
    bits = torch.zeros(1, dtype=torch.int32, device=DEV)
    Wd = W.to(DEV)
    ops._call("sonet_pointwise_tc_pack_device", _C.ptr(Wd), cout, cin, transpose, _C.ptr(blob),
              _C.ptr(scale2), _C.ptr(bits), ops._stream(Wd), kernels=3)
    want, inv = ops.pointwise_tc_pack(Wl)
    assert torch.equal(blob.cpu(), want)
    s = scale2.cpu()
    assert float(s[1]) == inv and float(s[0]) * inv == 1.0


@pytest.mark.parametrize("cin", [3, 64, 320, 1000])
@pytest.mark.parametrize("B,P,splits", [(2, 333, 1), (3, 50, 4)])
def test_wgrad_x_blob_equals_host_pack(cin, B, P, splits):
    """sonet_wgrad_tc_f32 packs x [B,Cin,P] into its blob scratch as the weight matrix
    [Cin][k = (b, p)], zero-padded to Kpad columns, with x's own pre-scale in small[0..1]."""
    from sonet_b200 import _C, ops
    lib = _C.lib()
    cout = 64
    x = rand(cin + P, B, cin, P)
    dy = rand(cin + P + 1, B, cout, P)
    Kpad = int(lib.sonet_wgrad_kpad(B, P, splits))
    xd, dyd = x.to(DEV), dy.to(DEV)
    f32 = dict(dtype=torch.float32, device=DEV)
    dyT = torch.empty(Kpad * cout, **f32)
    blob = torch.full((int(lib.sonet_wgrad_blob_bytes(cin, Kpad)),), 0xA5, dtype=torch.uint8, device=DEV)
    part = torch.empty(splits * cin * cout, **f32)
    small = torch.zeros(int(lib.sonet_wgrad_small_floats(cout)), **f32)
    dWT = torch.empty(cin, cout, **f32)
    ops._call("sonet_wgrad_tc_f32", _C.ptr(dyd), _C.ptr(xd), B, cout, cin, P, splits, _C.ptr(dyT),
              _C.ptr(blob), _C.ptr(part), _C.ptr(small), _C.ptr(dWT), ops._stream(dyd))
    Xm = torch.zeros(cin, Kpad)
    Xm[:, :B * P] = x.permute(1, 0, 2).reshape(cin, B * P)
    want, inv = ops.pointwise_tc_pack(Xm)
    assert torch.equal(blob.cpu(), want)
    s = small.cpu()
    assert float(s[1]) == inv and float(s[0]) * inv == 1.0
