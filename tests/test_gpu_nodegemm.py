"""The node-level wgmma GEMM (csrc/nodegemm_tc.cu) behind the encoder's final PointNet: its fp16
operand images against a numpy restatement of the core-matrix addressing, its two-layer chain bit
for bit against the generic layer (ops.pointwise_layer_tc) at every tile remainder and operand
magnitude, and the row-count rule that selects it."""
import contextlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@contextlib.contextmanager
def profiled():
    from sonet_b200 import ops
    calls = []
    ops.PROFILE = calls
    try:
        yield calls
    finally:
        ops.PROFILE = None


def same_bits(a, b):
    """Equal everywhere, NaN matching NaN (a NaN's payload is not part of any contract)."""
    na, nb = torch.isnan(a), torch.isnan(b)
    zero = torch.zeros((), device=a.device)
    return a.shape == b.shape and torch.equal(na, nb) and \
        torch.equal(torch.where(na, zero, a), torch.where(nb, zero, b))


def _params(cin, cout, seed, bias=0.3):
    from sonet_b200 import ops
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(cout, cin, generator=g) * (2.0 / cin) ** 0.5
    W[cout // 2] *= 1e-3                                   # a row far below the matrix's pre-scale
    blob, inv = ops.pointwise_tc_pack(W)
    return blob.to(DEV), inv, (torch.randn(cout, generator=g) * bias).to(DEV)


def _both(x0, x1, p1, c1, act, p2, c2, f16):
    from sonet_b200 import ops
    with profiled() as calls:
        got = ops.nodegemm_pointnet(x0, x1, p1, c1, act, p2, c2, f16=f16)
    assert [c[0] for c in calls] == ["sonet_nodegemm_split_pack"] + ["sonet_nodegemm_tc_forward"] * 2
    h = ops.pointwise_layer_tc(x0, *p1, c1, act, x1=x1, f16=f16)
    want = ops.pointwise_layer_tc(h, *p2, c2, None, f16=f16)
    torch.cuda.synchronize()
    return got, want


# ---- 1. the operand images -----------------------------------------------------------------------
def _r16(x):
    """cvt.rn.satfinite.f16.f32 of finite or infinite x, as fp16."""
    return np.clip(x, -65504.0, 65504.0).astype(np.float16)


@pytest.mark.parametrize("f16", [False, True], ids=["split", "fp16"])
def test_split_pack_layout(f16):
    """[128-row tile][32-channel stage][hi | lo] images of 8-row x 16-byte core matrices: element
    (r, k) of an image at (r / 8) * 512 + (k / 8) * 128 + (r % 8) * 16 + (k % 8) * 2; zero padding."""
    from sonet_b200 import _C, ops
    B, C0, C1, P = 3, 3, 70, 50                           # 150 rows: 2 tiles; 73 channels: 3 stages
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, C0 + C1, P, generator=g)
    x[0, 5, 3], x[1, 6, 4], x[2, 7, 5], x[2, 8, 6] = 70000.0, -2e5, float("inf"), 2.0 ** -14
    x0, x1 = x[:, :C0].contiguous().to(DEV), x[:, C0:].contiguous().to(DEV)
    lib = _C.lib()
    nimg = 1 if f16 else 2
    nbytes = lib.sonet_nodegemm_image_bytes(B * P, C0 + C1, int(f16))
    assert nbytes == 2 * 3 * nimg * 8192
    img = torch.full((nbytes,), 0xAB, dtype=torch.uint8, device=DEV)
    ops._call("sonet_nodegemm_split_pack", _C.ptr(x0), C0, _C.ptr(x1), C1, B, P, int(f16),
              _C.ptr(img), ops._stream(img))
    got = img.cpu().numpy().view(np.float16)

    rows = np.zeros((256, 96), np.float32)
    rows[:B * P, :C0 + C1] = x.permute(0, 2, 1).reshape(B * P, C0 + C1).numpy()
    hi = _r16(rows)
    with np.errstate(invalid="ignore"):
        lo = _r16(rows - hi.astype(np.float32))
    want = np.zeros(nbytes // 2, np.float16)
    r, k = np.meshgrid(np.arange(256), np.arange(96), indexing="ij")
    off = ((r // 128) * 3 + k // 32) * nimg * 8192 + (r % 128 // 8) * 512 + (k % 32 // 8) * 128 \
        + (r % 8) * 16 + (k % 8) * 2
    want[off // 2] = hi
    if not f16:
        want[(off + 8192) // 2] = lo
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))


# ---- 2. bit identity with the generic layer ---------------------------------------------------------
# (B, P, C0, C1, c1, c2)
SHAPES = [
    (64, 64, 3, 512, 768, 1024),     # cfg2's final PointNet
    (16, 16, 3, 512, 768, 1024),     # P = 16: eight clouds per tile
    (8, 36, 3, 512, 768, 1024),      # P = 36: tiles straddle clouds, 288 rows
    (3, 121, 3, 512, 768, 1024),     # 363 rows
    (2, 144, 3, 512, 768, 1024),
    (1, 256, 3, 512, 768, 1024),     # B = 1
    (5, 64, 3, 384, 192, 1000),      # Cin 387; n-tiles of 192 and of 232 -> 256 columns
    (4, 100, 3, 512, 1000, 192),     # hidden width 1000: image stage padded, K extent 1008
    (4, 64, 3, 61, 70, 130),         # one 64-channel chunk; hidden n-tile wider than its images
    (2, 128, 40, 0, 64, 64),         # single source, 64-column n-tiles
]


def _sid(c):
    return "B%d-P%d-C%d+%d-%d-%d" % c


@pytest.mark.parametrize("f16", [False, True], ids=["split", "fp16"])
@pytest.mark.parametrize("act", ["relu", "elu"])
@pytest.mark.parametrize("case", SHAPES, ids=_sid)
def test_chain_bit_identical_to_generic_layers(case, act, f16):
    B, P, C0, C1, c1, c2 = case
    g = torch.Generator().manual_seed(sum(case))
    x0 = (torch.rand(B, C0, P, generator=g) * 2 - 1).to(DEV)
    x1 = (torch.randn(B, C1, P, generator=g).abs() * 1.5).to(DEV) if C1 else None
    got, want = _both(x0, x1, _params(C0 + C1, c1, 1), c1, act, _params(c1, c2, 2), c2, f16)
    assert bool(torch.isfinite(want).all())
    assert torch.equal(got, want)


@pytest.mark.parametrize("f16", [False, True], ids=["split", "fp16"])
@pytest.mark.parametrize("act", ["relu", "elu"])
@pytest.mark.parametrize("kind", ["saturating", "tiny", "nonfinite"])
def test_chain_bit_identical_at_operand_extremes(kind, act, f16):
    """Inputs at the fp16 saturation edge (65504, 131008), near 2^-14 where lo(x) is subnormal,
    and NaN / +-inf rows: whatever the generic layer makes of them, bit for bit."""
    B, P, C0, C1, c1, c2 = 3, 100, 3, 125, 192, 320
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, C0 + C1, P, generator=g)
    if kind == "saturating":
        x[:, ::3] *= 65504.0
        x[:, 1::7] = 131008.0
        x[0, :, 5] = -70000.0
    elif kind == "tiny":
        x *= 2.0 ** -14
    else:
        x[0, :, 7] = float("nan")
        x[1, 4, :] = float("inf")
        x[2, 9, 50:] = float("-inf")
        x[2, 100, 3] = float("nan")
    x0, x1 = x[:, :C0].contiguous().to(DEV), x[:, C0:].contiguous().to(DEV)
    # a large hidden bias drives layer 1's output, layer 2's operand, to the edge as well
    p1 = _params(C0 + C1, c1, 3, bias=60000.0 if kind == "saturating" else 0.3)
    got, want = _both(x0, x1, p1, c1, act, _params(c1, c2, 4), c2, f16)
    assert same_bits(got, want)


# ---- 3. the route -------------------------------------------------------------------------------------
def _pointnet(cin, widths, act, seed):
    from sonet_b200 import layers
    torch.manual_seed(seed)
    net = layers.PointNet(cin, widths, act, 'batch')
    with torch.no_grad():
        for l in net.layers:
            l.conv.bias.normal_(0, 0.1)
            if l.normalization == 'batch':
                l.norm.weight.uniform_(0.5, 1.5)
                l.norm.bias.normal_(0, 0.1)
                l.norm.running_mean.normal_(0, 0.2)
                l.norm.running_var.uniform_(0.5, 2.0)
    return net.to(DEV).eval()


@pytest.mark.parametrize("act", ["relu", "elu"])
def test_pointnet_takes_the_node_route_by_row_count(act):
    """forward_pair: at most ops.NODEGEMM_MAX_ROWS rows -> the node-level GEMM, same bits as the
    per-layer chain; the segmenter's 49 k rows, fewer than two tiles, or three layers -> the
    generic layers as before."""
    from sonet_b200 import ops
    net = _pointnet(3 + 125, [192, 256], act, 5)
    g = torch.Generator().manual_seed(6)

    def run(n, B, P):
        x0 = torch.randn(B, 3, P, generator=g).to(DEV)
        x1 = torch.randn(B, 125, P, generator=g).to(DEV)
        with profiled() as calls, torch.no_grad():
            y = n.forward_pair(x0, x1)
        return x0, x1, y, [c[0] for c in calls]

    x0, x1, y, names = run(net, 4, 100)
    assert names == ["sonet_nodegemm_split_pack"] + ["sonet_nodegemm_tc_forward"] * 2
    l1, l2 = net.layers
    with torch.no_grad():
        assert torch.equal(y, l2.forward_points(l1.forward_points(x0, x1)))
    again = run(net, 4, 100)[2]
    assert y.data_ptr() != again.data_ptr()              # the images are cached, the result is not

    assert ops.NODEGEMM_MAX_ROWS < 16 * 3072
    assert run(net, 16, 3072)[3] == ["sonet_pointwise_tc_forward"] * 2
    assert run(net, 2, 100)[3] == ["sonet_pointwise_layer_f32"] * 2          # rows < 256
    deep = _pointnet(3 + 125, [192, 256, 128], act, 7)
    assert run(deep, 4, 100)[3] == ["sonet_pointwise_tc_forward"] * 3
    net.train()
    assert not any("nodegemm" in n for n in run(net, 4, 100)[3])


@pytest.mark.parametrize("mode", [None, "fp16"], ids=["split", "fp16"])
def test_cfg2_encoder_takes_the_node_route(monkeypatch, mode):
    """The benchmark's headline shape (B=64, N=5000, 8x8 SOM): the final PointNet runs on the
    node-level GEMM and final_pn_out / feature keep the generic chain's bits."""
    from sonet_b200 import classifier, networks, ops, synth
    if mode:
        monkeypatch.setenv("SONET_TC", mode)
    else:
        monkeypatch.delenv("SONET_TC", raising=False)
    B, N = 64, 5000
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device=DEV)
    cpu = synth.make_opt("classifier", batch_size=B, input_pc_num=N)
    inp = synth.synth_inputs(B, N, seed=0)
    m = classifier.Model(opt)
    m.encoder.load_state_dict(synth.synth_state_dict(networks.Encoder(cpu), seed=1))
    m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    with profiled() as calls:
        m.test_model()
        torch.cuda.synchronize()
    names = [c[0] for c in calls]
    assert names.count("sonet_nodegemm_split_pack") == 1
    assert names.count("sonet_nodegemm_tc_forward") == 2
    gemms = [c[3] for c in calls if c[0] == "sonet_nodegemm_tc_forward"]
    assert [(a[1], a[7], a[9]) for a in gemms] == [(515, 768, int(bool(mode))), (768, 1024, int(bool(mode)))]
    enc = m.encoder
    l1, l2 = enc.final_pointnet.layers
    with torch.no_grad():
        want = l2.forward_points(l1.forward_points(enc.knn_center_1.contiguous(),
                                                   enc.knn_feature_1.contiguous()))
    assert enc.final_pn_out.shape == (B, 1024, 64)
    assert torch.equal(enc.final_pn_out, want)
    assert torch.equal(enc.feature, want.max(dim=2)[0])
