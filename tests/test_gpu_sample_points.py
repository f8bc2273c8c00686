"""-m gpu: the on-device loader — csrc/sample_points.cu behind augmentation.DeviceDataset.batch.

Against the reference's own loaders (tests/golden/loader.npz, tools/make_golden_loader.py) with the
loader's numpy draws (host_noise=True), and, for the in-kernel draws, on sources whose x coordinate
is the point's index, so that the chosen indices can be read back from the output."""

import numpy as np
import pytest
import torch

from helpers import golden
from test_sample_points_host import fixture_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# chi^2 quantiles at p = 1e-6 (scipy.stats.chi2.isf(1e-6, dof)): every statistic below is computed
# from fixed seeds, so each test is deterministic; the bound says how far from uniform it may be
CHI2_1E6 = {9: 44.81, 19: 63.68, 49: 111.14, 1999: 2314.08}


def _ds(g, case):
    from sonet_b200 import augmentation as A
    pts, labels, som, seg, opt = fixture_case(g, case)
    return A.DeviceDataset(pts, labels, som, seg=seg, device=DEV), opt


def _names(opt):
    return (["pc", "sn", "label", "seg", "som_node", "som_knn_I"] if opt.dataset == "shapenet"
            else ["pc", "sn", "label", "som_node", "som_knn_I"])


def _ulp_close(a, b, what):
    """numpy's BLAS may fuse the 3-term rotation products of the loader (not the kernel): <= 1 fp32
    ulp on < 0.01 % of the elements, as in test_gpu_augment."""
    neq = a != b
    assert neq.mean() <= 1e-4, "%s: %.4f%% elements differ" % (what, 100 * neq.mean())
    if neq.any():
        ulp = np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))
        assert ulp.max() <= 1, "%s: %d ulp" % (what, ulp.max())


@pytest.mark.parametrize("case", ["modelnet", "modelnet_rot", "shrec", "shrec64", "shapenet"])
@pytest.mark.parametrize("mode", ["test", "train"])
def test_batches_reproduce_the_reference_loaders(case, mode):
    g = golden("loader")
    if case == "shrec64" and mode == "train":
        pytest.skip("float64 sources in train mode: test_float64_source_bound")
    ds, opt = _ds(g, case)
    S = len(ds)
    out = ds.batch(np.arange(S), opt, train=(mode == "train"),
                   rng=np.random.RandomState(int(g["seed_" + mode])), seed=3, host_noise=True)
    names = _names(opt)
    assert len(out) == len(names)
    for name, t in zip(names, out):
        want = torch.from_numpy(g["%s_%s_%s" % (case, mode, name)])
        assert t.is_cuda and t.dtype == want.dtype and t.shape == want.shape, (case, name)
        if case == "modelnet_rot" and mode == "train" and t.is_floating_point():
            _ulp_close(t.cpu().numpy(), want.numpy(), name)
        else:
            assert torch.equal(t.cpu(), want), (case, mode, name)


def test_float64_source_bound():
    """SHREC-like float64 sources are rounded to fp32 once at upload; the loader jitters, scales and
    shifts in float64 before its one rounding. Each output value is within
    2^-24 * scale * |v| (v the source 3-vector) plus one fp32 ulp of the loader's value."""
    from sonet_b200 import augmentation as A, ops
    g = golden("loader")
    ds, opt = _ds(g, "shrec64")
    pts, _, som, _, _ = fixture_case(g, "shrec64")
    seed = int(g["seed_train"])
    out = ds.batch(np.arange(len(ds)), opt, train=True, rng=np.random.RandomState(seed),
                   host_noise=True)
    flags = dict(rot_horizontal=opt.rot_horizontal, rot_perturbation=opt.rot_perturbation,
                 translation_perturbation=opt.translation_perturbation)
    sel, params = A.draw_batch_host(np.random.RandomState(seed), [len(p) for p in pts],
                                    opt.input_pc_num, opt.node_num, ops.SAMPLE_SUBSET, True, **flags)
    src = np.stack([p[s] for p, s in zip(pts, sel)])                    # [B,N,6] float64
    vecs = {"pc": src[:, :, :3], "sn": src[:, :, 3:], "som_node": np.stack(som)}
    differs = 0
    for name, t in zip(_names(opt), out):
        if name not in vecs:
            continue
        got = t.cpu().numpy().astype(np.float64)
        ref = g["shrec64_train_" + name]
        norm = np.linalg.norm(vecs[name], axis=2)[:, None, :]           # [B,1,P]
        bound = 2.0 ** -24 * params["scale"][:, None, None] * norm * (1 + 1e-9) + \
            np.spacing(np.abs(ref)).astype(np.float64)
        assert (np.abs(got - ref) <= bound).all(), name
        differs += int((got != ref).sum())
    print("float64 sources: %d values differ from the loader's, all within the bound" % differs)


# ---- in-kernel draws -------------------------------------------------------------------------------
def _index_dataset(counts, M=16, seg=False):
    """Clouds whose x coordinate is the point index (exact in fp32), y the cloud, part label = index."""
    from sonet_b200 import augmentation as A
    pts = []
    for c, P in enumerate(counts):
        p = np.zeros((P, 6), np.float32)
        p[:, 0] = np.arange(P)
        p[:, 1] = c
        p[:, 3] = -np.arange(P)
        pts.append(p)
    return A.DeviceDataset(pts, np.arange(len(counts)), [np.zeros((M, 3))] * len(counts),
                           seg=[np.arange(P) % 50 for P in counts] if seg else None, device=DEV)


def _draw(ds, cloud_ids, N, rule, seed=0, indices=None):
    from sonet_b200 import ops
    cid = torch.as_tensor(np.asarray(cloud_ids, np.int64)).to(DEV)
    P = ds.counts[np.asarray(cloud_ids)]
    pc, sn, seg = ops.sample_points(ds.data, ds.offsets, cid, N, rule, int(P.max()),
                                    labels=ds.seg, indices=indices, seed=seed)
    idx = pc[:, 0, :].long()
    assert torch.equal(sn[:, 0, :], -pc[:, 0, :])                      # one source row per point
    assert torch.equal(pc[:, 1, :].long(), cid.view(-1, 1).expand_as(idx))
    if seg is not None:
        assert torch.equal(seg, idx % 50)
    return idx.cpu().numpy()


def _check_subset(idx, P):
    assert idx.min() >= 0 and idx.max() < P
    s = np.sort(idx, axis=1)
    assert (s[:, 1:] != s[:, :-1]).all(), "repeated index"


def test_subset_indices_are_distinct_and_uniform():
    from sonet_b200 import ops
    P, N, B = 20, 5, 4000
    ds = _index_dataset([P])
    incl = np.zeros(P)
    first = np.zeros(P)
    last = np.zeros(P)
    for seed in range(5):
        idx = _draw(ds, [0] * B, N, ops.SAMPLE_SUBSET, seed=seed)
        _check_subset(idx, P)
        incl += np.bincount(idx.ravel(), minlength=P)
        first += np.bincount(idx[:, 0], minlength=P)
        last += np.bincount(idx[:, -1], minlength=P)
    T = 5 * B
    for what, obs, e in (("inclusion", incl, T * N / P), ("first", first, T / P),
                         ("last", last, T / P)):
        chi2 = float(((obs - e) ** 2 / e).sum())
        assert chi2 < CHI2_1E6[P - 1], "%s: chi2 %.1f" % (what, chi2)


def test_subset_uniform_across_digit_buckets():
    """P = 2000 keys fall into many 12-bit buckets: the inclusion counts stay uniform."""
    from sonet_b200 import ops
    P, N, B = 2000, 700, 2000
    ds = _index_dataset([P])
    idx = _draw(ds, [0] * B, N, ops.SAMPLE_SUBSET, seed=11)
    _check_subset(idx, P)
    obs = np.bincount(idx.ravel(), minlength=P)
    e = B * N / P
    assert float(((obs - e) ** 2 / e).sum()) < CHI2_1E6[P - 1]
    pos = np.bincount(idx[:, 0] * 50 // P, minlength=50)                # first position, 50 bins
    assert float(((pos - B / 50) ** 2 / (B / 50)).sum()) < CHI2_1E6[49]


def test_fill_layout_and_uniform_draws():
    from sonet_b200 import ops
    P, N, B = 10, 40, 2000
    ds = _index_dataset([P, 60, N], seg=True)
    idx = _draw(ds, [0] * B, N, ops.SAMPLE_FILL, seed=5)
    assert (idx[:, :P] == np.arange(P)).all()
    extra = idx[:, P:]
    assert extra.min() >= 0 and extra.max() < P
    obs = np.bincount(extra.ravel(), minlength=P)
    e = extra.size / P
    assert float(((obs - e) ** 2 / e).sum()) < CHI2_1E6[P - 1]
    both = _draw(ds, [1, 2], N, ops.SAMPLE_FILL, seed=5)
    _check_subset(both[0:1], 60)                                        # N < P: a subset
    assert (both[1] == np.arange(N)).all()                              # N == P: the cloud in order


def test_seeds_and_batch_independence():
    from sonet_b200 import ops
    ds = _index_dataset([300, 500, 250, 400])
    ids = [0, 1, 2, 3, 1]
    a = _draw(ds, ids, 200, ops.SAMPLE_SUBSET, seed=9)
    b = _draw(ds, ids, 200, ops.SAMPLE_SUBSET, seed=9)
    c = _draw(ds, ids, 200, ops.SAMPLE_SUBSET, seed=10)
    assert np.array_equal(a, b)
    assert all(not np.array_equal(a[i], c[i]) for i in range(len(ids)))
    assert not np.array_equal(a[1], a[4])                               # keyed by batch position
    d = _draw(ds, [0, 1, 3, 3, 1], 200, ops.SAMPLE_SUBSET, seed=9)      # position 2 changed
    assert np.array_equal(np.delete(a, 2, 0), np.delete(d, 2, 0))


@pytest.mark.parametrize("P", [1, 99, 100, 101, 1023, 1024, 1025, 4095, 4096, 4097, 65535, 65536])
def test_envelope_edges(P):
    """N = 100 around P: rule edges at N -1/0/+1, the CTA's 1024 threads, the 4096 radix bins,
    and the in-kernel envelope's end."""
    from sonet_b200 import ops
    N = 100
    ds = _index_dataset([P, 7])
    f = _draw(ds, [0, 1, 0], N, ops.SAMPLE_FILL, seed=P)
    if P >= N:
        _check_subset(f[[0, 2]], P)
        if P == N:
            assert (f[0] == np.arange(N)).all()
    else:
        assert (f[0, :P] == np.arange(P)).all() and f[0].max() < P
    if P >= N:
        s = _draw(ds, [0, 0], N, ops.SAMPLE_SUBSET, seed=P)
        _check_subset(s, P)
        one = _draw(ds, [0], 1, ops.SAMPLE_SUBSET, seed=P)             # N = 1, B = 1
        assert one.shape == (1, 1) and 0 <= one[0, 0] < P


@pytest.mark.parametrize("P", [100, 4097, 65536])
def test_whole_cloud_permutation(P):
    """SUBSET with N == P: a permutation of the whole cloud (every key selected and sorted)."""
    from sonet_b200 import ops
    idx = _draw(_index_dataset([P]), [0, 0], P, ops.SAMPLE_SUBSET, seed=1)
    assert (np.sort(idx, axis=1) == np.arange(P)).all()
    assert not (idx[0] == np.arange(P)).all() and not np.array_equal(idx[0], idx[1])


def test_large_batch():
    from sonet_b200 import ops
    ds = _index_dataset([30, 12, 64])
    B = 65535
    ids = np.arange(B) % 3
    idx = _draw(ds, ids, 12, ops.SAMPLE_SUBSET, seed=4)
    P = ds.counts[ids][:, None]
    assert (idx >= 0).all() and (idx < P).all()
    s = np.sort(idx, axis=1)
    assert (s[:, 1:] != s[:, :-1]).all()
    assert not np.array_equal(idx[1], idx[4])                           # same cloud, other position


def test_given_indices_any_P_and_clamp():
    """Given indices: a cloud beyond the in-kernel envelope, out-of-range values clamped."""
    from sonet_b200 import ops
    P = 100000
    ds = _index_dataset([P, 5], seg=True)
    given = np.array([[0, P - 1, 70000, -3, P + 9], [4, 0, 9, -1, 2]], np.int32)
    idx = _draw(ds, [0, 1], 5, ops.SAMPLE_SUBSET, indices=torch.from_numpy(given).to(DEV))
    assert (idx == np.clip(given, 0, np.array([[P - 1], [4]]))).all()
    with pytest.raises(RuntimeError, match="envelope"):
        _draw(ds, [0], 5, ops.SAMPLE_SUBSET)


def test_device_draw_batches_have_the_loader_layout():
    """host_noise=False: the same tuple layout, dtypes and label/seg semantics."""
    g = golden("loader")
    for case in ("modelnet", "shapenet"):
        ds, opt = _ds(g, case)
        a = ds.batch(np.arange(len(ds)), opt, train=True, rng=np.random.RandomState(1), seed=2)
        b = ds.batch(np.arange(len(ds)), opt, train=True, rng=np.random.RandomState(1), seed=2)
        want = [g["%s_train_%s" % (case, n)] for n in _names(opt)]
        for x, y, w in zip(a, b, want):
            assert torch.equal(x, y) and x.dtype == torch.from_numpy(w).dtype and x.shape == w.shape
        assert torch.equal(a[2].cpu(), torch.from_numpy(g[case + "_train_label"]))


# ---- end to end ------------------------------------------------------------------------------------
def _model_dataset(M, counts, seed):
    from sonet_b200 import augmentation as A
    rs = np.random.RandomState(seed)
    pts = []
    for P in counts:
        xyz = rs.uniform(-1, 1, size=(P, 3))
        n = rs.normal(size=(P, 3))
        pts.append(np.concatenate([xyz, n / np.linalg.norm(n, axis=1, keepdims=True)], 1))
    som = [p[rs.permutation(len(p))[:M], :3] for p in pts]
    seg = [rs.randint(0, 50, size=P) for P in counts]
    return A.DeviceDataset(pts, rs.randint(0, 16, size=len(counts)), som, seg=seg, device=DEV)


@pytest.mark.parametrize("task", ["classifier", "segmenter"])
def test_models_fed_device_batches_match_host_tensors(task):
    from sonet_b200 import classifier, segmenter, synth
    B, N = 4, 512
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, device=DEV)
    opt.dataset = "shapenet" if task == "segmenter" else "modelnet"
    opt.rot_horizontal = opt.rot_perturbation = opt.translation_perturbation = True
    counts = [700, 400, 512, 900, 650] if task == "segmenter" else [700, 800, 512, 900, 650]
    ds = _model_dataset(opt.node_num, counts, seed=3)
    torch.manual_seed(0)
    m = (segmenter if task == "segmenter" else classifier).Model(opt)
    batch = ds.batch([4, 0, 2, 3], opt, train=True, rng=np.random.RandomState(5), seed=6)
    assert all(t.is_cuda for t in batch)
    out = "score_segmenter" if task == "segmenter" else "score"
    m.set_input(*batch)
    m.test_model()
    s_dev = getattr(m, out).clone()
    m.set_input(*[t.cpu() for t in batch])
    m.test_model()
    torch.cuda.synchronize()
    assert torch.equal(s_dev, getattr(m, out))
