"""Host-side packing of the wgmma point-MLP weights (no GPU needed): the fp16 hi/lo K-major
core-matrix images, times the stored inverse power-of-two scale, must reproduce the fp32 weights
to ~2^-21 and sit at the documented offsets."""
import numpy as np
import torch


def test_pack_images_round_trip(lib_built):
    from sonet_b200 import ops
    rs = np.random.RandomState(0)
    W = [torch.from_numpy((rs.normal(size=s) * sc).astype(np.float32))
         for s, sc in (((64, 6), 1.0), ((128, 64), 0.2), ((256, 128), 0.1), ((384, 320), 3.0))]
    sh = [torch.from_numpy(rs.normal(size=s).astype(np.float32)) for s in (64, 128, 256, 384)]
    blob, fpar = ops.pointresnet_tc_pack(W, sh, 6)
    assert blob.numel() == 32768 + 4 * 32768 + 6 * (32768 * 2 + 16384)
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
    # layer 3 streams [96 rows x 64 k] stages, chunk-major: chunk 1 (rows 96..191), slab 4 (k 256..319)
    base = 32768 + 4 * 32768 + (1 * 5 + 4) * 24576
    w3c = unpack(base, 96, 64, 12288) * inv[2]
    assert np.abs(w3c - W[3].numpy()[96:192, 256:320]).max() <= tol * np.abs(W[3].numpy()).max()
    assert np.array_equal(f[:384].reshape(64, 6), W[0].numpy())
    assert np.array_equal(f[384:448], sh[0].numpy())
    assert np.array_equal(f[448 + 128 + 256:448 + 128 + 256 + 384], sh[3].numpy())
