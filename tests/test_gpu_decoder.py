"""-m gpu: the up-convolution decoder kernels (SURVEY.md §8f-1; csrc/upconv.cu + the grouped /
split-K wgmma layer of csrc/pointwise_tc.cu) against an fp64 evaluation of the reference
composition UpConv.forward = conv3x3(pad 1)(upsample_nearest_x2(x)) + eval BN + ReLU
(models/layers.py:214-240). Tolerance |a-b| <= 1e-4 * max(|b|, 1)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import assert_close

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _upconv(cin, cout, seed):
    from sonet_b200 import layers, synth
    m = layers.UpConv(cin, cout, activation='relu', normalization='batch')
    m.load_state_dict(synth.synth_state_dict(m, seed=seed))
    return m.to(DEV).eval()


def _ref64(m, x):
    c, n = m.conv.conv, m.conv.norm
    y = F.conv2d(F.interpolate(x.double(), scale_factor=2, mode='nearest'), c.weight.double(),
                 c.bias.double(), padding=1)
    y = (y - n.running_mean.double()[None, :, None, None]) / torch.sqrt(
        n.running_var.double() + n.eps)[None, :, None, None]
    y = y * n.weight.double()[None, :, None, None] + n.bias.double()[None, :, None, None]
    return F.relu(y).float()


# the six stages of DecoderConv (models/networks.py:408-415) + odd sizes (non-square, B*H*W not a
# multiple of 128, one K chunk)
@pytest.mark.parametrize("B,cin,cout,H,W", [(32, 1024, 1024, 1, 1), (32, 1024, 512, 2, 2),
                                            (32, 512, 256, 4, 4), (32, 256, 128, 8, 8),
                                            (8, 128, 128, 16, 16), (4, 128, 128, 32, 32),
                                            (2, 1024, 1024, 1, 1), (3, 64, 64, 5, 7),
                                            (1, 16, 64, 3, 3)])
def test_upconv_vs_fp64(B, cin, cout, H, W):
    from sonet_b200 import ops
    m = _upconv(cin, cout, seed=cin + cout + H)
    g = torch.Generator().manual_seed(B * 131 + H)
    x = torch.randn(B, cin, H, W, generator=g).to(DEV)
    c0 = ops.LAUNCHES
    with torch.no_grad():
        y = m(x)
    assert ops.LAUNCHES > c0, "the up-convolution did not run on the sonet kernels"
    assert y.shape == (B, cout, 2 * H, 2 * W)
    with torch.no_grad():
        want = _ref64(m, x)
    assert_close(y, want, "upconv [%d,%d->%d,%dx%d]" % (B, cin, cout, H, W))
    # deterministic (split-K partial sums are reduced in a fixed order)
    with torch.no_grad():
        assert torch.equal(m(x), y)


def test_decoder_conv_pyramid_vs_fp64_and_torch_path():
    """The whole DecoderConv pyramid (6 up-convolutions + 3 ConvToPC heads) against the same
    modules evaluated in fp64 on the CPU, and the PyTorch (training) composition on the GPU."""
    from sonet_b200 import networks, synth
    opt = synth.make_opt("autoencoder", batch_size=4, input_pc_num=256)
    dec = networks.Decoder(opt)
    dec.load_state_dict(synth.synth_state_dict(dec, seed=9))
    dec = dec.to(DEV).eval()
    feat = torch.randn(4, 1024, generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad():
        got = dec(feat)
        pc4, pc5 = dec.conv_pc4.clone(), dec.conv_pc5.clone()
    ref = networks.Decoder(opt)
    ref.load_state_dict(synth.synth_state_dict(ref, seed=9))
    ref = ref.double().eval()                       # CPU fp64: every layer takes the PyTorch path
    with torch.no_grad():
        want = ref(feat.cpu().double())
    assert_close(got, want.float(), "predicted_pc")
    assert_close(pc4, ref.conv_pc4.float(), "conv_pc4")
    assert_close(pc5, ref.conv_pc5.float(), "conv_pc5")
