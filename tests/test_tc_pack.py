"""Host-side packing of the wgmma point-MLP weights (no GPU needed): the fp16 hi/lo K-major
core-matrix images, times the stored inverse power-of-two scale, must reproduce the fp32 weights
to ~2^-21 and sit at the documented offsets; and every host packer must write the same bytes as
the numpy packer below, which restates the blob format independently."""
import numpy as np
import pytest
import torch


def test_pack_images_round_trip_128_row_layer3(lib_built):
    from sonet_b200 import ops
    rs = np.random.RandomState(0)
    W = [torch.from_numpy((rs.normal(size=s) * sc).astype(np.float32))
         for s, sc in (((64, 6), 1.0), ((128, 64), 0.2), ((256, 128), 0.1), ((384, 320), 3.0))]
    sh = [torch.from_numpy(rs.normal(size=s).astype(np.float32)) for s in (64, 128, 256, 384)]
    blob, fpar = ops.pointresnet_tc_pack(W, sh, 6)
    assert blob.numel() == 20 * 32768
    b = blob.numpy().view(np.float16)
    f = fpar.numpy()
    assert f.size == 384 + 64 + 128 + 256 + 384 + 4
    inv = f[384 + 64 + 128 + 256 + 384:]

    def unpack(base, rows, kt, hi_bytes):
        out = np.zeros((rows, kt), np.float64)
        for r in range(rows):
            for k in range(kt):
                off = (r >> 3) * kt * 16 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2
                out[r, k] = float(b[(base + off) // 2]) + float(b[(base + hi_bytes + off) // 2])
        return out

    for li in (1, 2, 3):
        scale = 1.0 / inv[li - 1]
        m = float(W[li].abs().max()) * scale
        assert 256.0 <= m < 512.0 and np.log2(scale) == np.round(np.log2(scale))
    tol = 2.0 ** -20
    w1 = unpack(0, 128, 64, 16384) * inv[0]
    assert np.abs(w1 - W[1].numpy()).max() <= tol * np.abs(W[1].numpy()).max()
    # layer 2 streams four K slabs [256 rows x 32 k]; slab 3 (k 96..127) is the 4th stage
    w2c = unpack(32768 + 3 * 32768, 256, 32, 16384) * inv[1]
    assert np.abs(w2c - W[2].numpy()[:, 96:128]).max() <= tol * np.abs(W[2].numpy()).max()
    # layer 3 streams [128 rows x 64 k] stages, chunk-major: chunk 1 (rows 128..255), slab 4 (k 256..319)
    base = 32768 + 4 * 32768 + (1 * 5 + 4) * 32768
    w3c = unpack(base, 128, 64, 16384) * inv[2]
    assert np.abs(w3c - W[3].numpy()[128:256, 256:320]).max() <= tol * np.abs(W[3].numpy()).max()
    assert np.array_equal(f[:384].reshape(64, 6), W[0].numpy())
    assert np.array_equal(f[384:448], sh[0].numpy())
    assert np.array_equal(f[448 + 128 + 256:448 + 128 + 256 + 384], sh[3].numpy())


# ---- reference packer -----------------------------------------------------------------------------
def ref_scale(W):
    """Power of two s with max|s W| in [256, 512), at most 2^126 (1/s stays a normal float); 1 for
    an all-zero matrix."""
    m = np.float32(np.abs(W).max())
    if not (m > 0 and np.isfinite(m)):
        return np.float32(1.0)
    return np.float32(np.ldexp(1.0, min(9 - int(np.frexp(m)[1]), 126)))


def ref_split(Ws):
    """fp16 hi/lo halves of pre-scaled fp32 weights (round to nearest even, no saturation)."""
    hi = Ws.astype(np.float16)
    lo = (Ws - hi.astype(np.float32)).astype(np.float16)
    return hi.view(np.uint16), lo.view(np.uint16)


def ref_off(r, k, kt):
    """Byte offset of element (r, k) in a K-major no-swizzle image with K extent kt."""
    return (r >> 3) * kt * 16 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2


def ref_stage(Ws, kt):
    """One stage: the hi image of Ws [rows, kt], then its lo image."""
    rows = Ws.shape[0]
    r, k = np.meshgrid(np.arange(rows), np.arange(kt), indexing="ij")
    hi, lo = ref_split(Ws)
    img = np.zeros((2, rows * kt), np.uint16)
    img[0, ref_off(r, k, kt) // 2] = hi
    img[1, ref_off(r, k, kt) // 2] = lo
    return img.view(np.uint8).ravel()


def ref_pointwise_blob(W, scale):
    """The generic layer's blob of W [N, K]: N padded to 64 in n-tiles of <= 256 rows; per tile,
    K padded to 16 in chunks of 64, each chunk two [nw x 32] stages."""
    N, K = W.shape
    npad = (N + 63) // 64 * 64
    kch = ((K + 15) // 16 * 16 + 63) // 64
    Wp = np.zeros((npad, kch * 64), np.float32)
    Wp[:N, :K] = W * scale
    return np.concatenate([ref_stage(Wp[n0:n0 + 256, k0:k0 + 32], 32)
                           for n0 in range(0, npad, 256) for k0 in range(0, kch * 64, 32)])


def rand_weights(rs, *shape):
    W = rs.normal(size=shape) * 10.0 ** rs.uniform(-6, 3)
    W.flat[rs.randint(W.size)] = 0.0
    return W.astype(np.float32)


@pytest.mark.parametrize("cout", [3, 64, 320, 1000])
@pytest.mark.parametrize("cin", [16, 33, 500])
def test_pointwise_pack_matches_reference(lib_built, cout, cin):
    from sonet_b200 import ops
    rs = np.random.RandomState(cout * 1000 + cin)
    W = rand_weights(rs, cout, cin)
    blob, inv = ops.pointwise_tc_pack(torch.from_numpy(W))
    s = ref_scale(W)
    assert inv == np.float32(1.0) / s
    assert np.array_equal(blob.numpy(), ref_pointwise_blob(W, s))


@pytest.mark.parametrize("e", [-149, -140, -125, -120, -119, -118, -117])
def test_pointwise_pack_scale_is_capped_for_tiny_matrices(lib_built, e):
    """A matrix with max |W| = 2^e below 2^-118 gets the capped scale 2^126, not 2^(9 - e - 1),
    which overflows to inf from e = -119 down; at 2^-118 and above the cap changes nothing."""
    from sonet_b200 import ops
    rs = np.random.RandomState(-e)
    W = rs.normal(size=(70, 40))
    W = (W / np.abs(W).max() * 2.0 ** e).astype(np.float32)
    assert np.float32(np.abs(W).max()) == np.float32(2.0 ** e)
    blob, inv = ops.pointwise_tc_pack(torch.from_numpy(W))
    s = ref_scale(W)
    assert s == np.float32(2.0 ** min(8 - e, 126)) and np.isfinite(s)
    assert inv == np.float32(1.0) / s and inv >= np.finfo(np.float32).tiny
    assert np.array_equal(blob.numpy(), ref_pointwise_blob(W, s))


@pytest.mark.parametrize("cout,cin", [(3, 33), (320, 500), (1000, 16)])
def test_pointwise_pack_groups_matches_reference(lib_built, cout, cin):
    """G = 4 blobs back to back with ONE scale, from the largest weight of all groups."""
    from sonet_b200 import ops
    rs = np.random.RandomState(cout + cin)
    Wg = rand_weights(rs, 4, cout, cin)
    Wg[2] *= 64.0                                   # the shared scale comes from group 2
    blob, per, inv = ops.pointwise_tc_pack_groups(torch.from_numpy(Wg))
    s = ref_scale(Wg)
    assert inv == np.float32(1.0) / s and s != ref_scale(Wg[0])
    want = np.concatenate([ref_pointwise_blob(Wg[g], s) for g in range(4)])
    assert per * 4 == want.size and np.array_equal(blob.numpy(), want)


@pytest.mark.parametrize("cin", [3, 6])
def test_pointresnet_pack_matches_reference(lib_built, cin):
    """Layer 1 [128 x 64], four layer-2 K slabs [256 x 32], then layer 3 as 3 row chunks of 128
    x 5 K slabs of 64 (chunk-major): 20 stages of 32 KB in the order the kernel consumes them."""
    from sonet_b200 import ops
    rs = np.random.RandomState(cin)
    W = [rand_weights(rs, *s) for s in ((64, cin), (128, 64), (256, 128), (384, 320))]
    sh = [rs.normal(size=n).astype(np.float32) for n in (64, 128, 256, 384)]
    blob, fpar = ops.pointresnet_tc_pack([torch.from_numpy(w) for w in W],
                                         [torch.from_numpy(s) for s in sh], cin)
    s1, s2, s3 = (ref_scale(w) for w in W[1:])
    stages = [ref_stage(W[1] * s1, 64)]
    stages += [ref_stage(W[2][:, 32 * kc:32 * kc + 32] * s2, 32) for kc in range(4)]
    stages += [ref_stage(W[3][128 * nc:128 * nc + 128, 64 * kc:64 * kc + 64] * s3, 64)
               for nc in range(3) for kc in range(5)]
    assert all(st.size == 32768 for st in stages)
    assert np.array_equal(blob.numpy(), np.concatenate(stages))
    w0 = np.zeros((64, 6), np.float32)
    w0[:, :cin] = W[0]
    inv = np.float32(1.0) / np.array([s1, s2, s3], np.float32)
    want = np.concatenate([w0.ravel(), *sh, inv, np.zeros(1, np.float32)])
    assert np.array_equal(fpar.numpy(), want)


def test_knn_mlp_pack_matches_reference(lib_built):
    """Two passes of 256 output rows, each 16 K slabs [256 x 32]."""
    from sonet_b200 import ops
    rs = np.random.RandomState(11)
    W2 = rand_weights(rs, 512, 512)
    blob, inv = ops.knn_mlp_tc_pack(torch.from_numpy(W2))
    s = ref_scale(W2)
    assert inv == np.float32(1.0) / s
    want = np.concatenate([ref_stage(W2[256 * p:256 * p + 256, 32 * ks:32 * ks + 32] * s, 32)
                           for p in range(2) for ks in range(16)])
    assert np.array_equal(blob.numpy(), want)
