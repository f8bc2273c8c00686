"""Host side of the on-device loader (sonet_sample_points_f32, augmentation.DeviceDataset), no GPU:
the C entry's argument validation, its export and declaration, DeviceDataset's input checks, and
the loader's draw order — the host draws of batch(host_noise=True), applied with a numpy gather
(and, where the pipeline is elementwise, numpy float64 augmentation), reproduce the batches that
the reference's own loaders produced (tests/golden/loader.npz, tools/make_golden_loader.py)."""
import argparse
import ctypes
import os
import re

import numpy as np
import pytest

from helpers import golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "sonet_sample_points_f32"
P_ = 8       # a non-null placeholder pointer: validation must fail before anything is read


def _call(lib, data=P_, offsets=P_, S=4, labels=None, ids=P_, B=2, N=16, max_P=100, rule=0,
          indices=None, seed=0, pc=P_, sn=P_, seg=None):
    return lib.sonet_sample_points_f32(data, offsets, S, labels, ids, B, N, max_P, rule, indices,
                                       seed, pc, sn, seg, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(rule=2), "rule 2"), (dict(rule=-1), "rule -1"),
    (dict(N=0), "N=0"), (dict(N=-5), "N=-5"),
    (dict(B=-1), "B=-1"), (dict(B=65536), "B=65536"),
    (dict(S=0), "S=0"), (dict(max_P=0), "max_P=0"),
    (dict(max_P=65537), "max_P=65537"),
    (dict(labels=P_), "labels and seg_out"), (dict(seg=P_), "labels and seg_out"),
    (dict(data=None), "null"), (dict(offsets=None), "null"), (dict(ids=None), "null"),
    (dict(pc=None), "null"), (dict(sn=None), "null"),
])
def test_bad_arguments_fail_before_any_cuda_call(lib_built, kw, msg):
    from sonet_b200 import _C
    lib = _C.lib()
    assert _call(lib, **kw) == -1
    assert msg in _C.last_error(), _C.last_error()


def test_envelope_edges_are_accepted_arguments(lib_built):
    """max_P at the in-kernel envelope, and any max_P with given indices, pass validation (B = 0
    then returns before any launch)."""
    from sonet_b200 import _C
    lib = _C.lib()
    assert _call(lib, B=0, max_P=65536) == 0
    assert _call(lib, B=0, max_P=1 << 30, indices=P_) == 0
    assert _call(lib, B=0, rule=1, labels=P_, seg=P_) == 0


def test_symbol_exported_and_declared(lib_built):
    from sonet_b200 import _C, ops
    h = ctypes.CDLL(lib_built)
    assert hasattr(h, NAME)
    text = open(os.path.join(ROOT, "include", "sonet_b200.h")).read()
    assert re.search(r"\b%s\s*\(" % NAME, text)
    assert NAME in _C.EXPORTED_SYMBOLS
    for name, val in (("SUBSET", ops.SAMPLE_SUBSET), ("FILL", ops.SAMPLE_FILL),
                      ("MAX_P", ops.SAMPLE_MAX_P)):
        assert re.search(r"#define SONET_SAMPLE_%s %d\b" % (name, val), text), name


def _cpu_dataset(counts, M=4, seg=False):
    from sonet_b200 import augmentation as A
    rs = np.random.RandomState(0)
    pts = [rs.uniform(size=(p, 6)).astype(np.float32) for p in counts]
    return A.DeviceDataset(pts, np.arange(len(counts)), [rs.uniform(size=(M, 3)) for _ in counts],
                           seg=[np.zeros(p, np.int32) for p in counts] if seg else None,
                           device="cpu")


def test_empty_cloud_and_shape_checks():
    from sonet_b200 import augmentation as A
    with pytest.raises(ValueError, match="cloud 1 is empty"):
        A.DeviceDataset([np.zeros((5, 6)), np.zeros((0, 6))], [0, 1], [np.zeros((4, 3))] * 2)
    with pytest.raises(ValueError, match="expected \\[P, 6\\]"):
        A.DeviceDataset([np.zeros((5, 3))], [0], [np.zeros((4, 3))])
    with pytest.raises(ValueError, match="one M"):
        A.DeviceDataset([np.zeros((5, 6))] * 2, [0, 1], [np.zeros((4, 3)), np.zeros((9, 3))])
    with pytest.raises(ValueError, match="one entry per cloud"):
        A.DeviceDataset([np.zeros((5, 6))], [0, 1], [np.zeros((4, 3))])
    with pytest.raises(ValueError, match="seg"):
        A.DeviceDataset([np.zeros((5, 6))], [0], [np.zeros((4, 3))], seg=[np.zeros(4)])


def test_subset_of_a_small_cloud_raises_value_error_from_the_counts():
    ds = _cpu_dataset([300, 99, 200], seg=True)
    opt = argparse.Namespace(dataset="modelnet", input_pc_num=100, som_k=1)
    with pytest.raises(ValueError, match="larger sample than population"):
        ds.batch([0, 1], opt, train=False)
    with pytest.raises(ValueError, match="larger sample than population"):   # numpy's own words
        np.random.RandomState(0).choice(99, 100, replace=False)
    with pytest.raises(IndexError):
        ds.batch([3], opt, train=False)
    with pytest.raises(ValueError, match="unknown dataset"):
        ds.batch([0], argparse.Namespace(dataset="kitti", input_pc_num=10, som_k=1), train=False)
    with pytest.raises(ValueError, match="needs seg"):
        _cpu_dataset([300]).batch([0], argparse.Namespace(dataset="shapenet", input_pc_num=10,
                                                          som_k=1), train=False)


def fixture_case(g, case):
    src = str(g[case + "_source"])
    counts = g[src + "_counts"]
    off = np.concatenate([[0], np.cumsum(counts)])
    pts = [g[src + "_points"][off[i]:off[i + 1]] for i in range(len(counts))]
    seg = None
    if src + "_seg" in g.files:
        seg = [g[src + "_seg"][off[i]:off[i + 1]] for i in range(len(counts))]
    flags = {k: bool(g["%s_opt_%s" % (case, k)]) for k in
             ("rot_horizontal", "rot_perturbation", "translation_perturbation")}
    opt = argparse.Namespace(dataset=str(g[case + "_dataset"]), input_pc_num=int(g["N"]),
                             node_num=int(g["node_num"]), som_k=int(g["som_k"]), **flags)
    return pts, g[src + "_labels"], list(g[src + "_som"]), seg, opt


CASES = ["modelnet", "modelnet_rot", "shrec", "shrec64", "shapenet"]


def _host_batch(g, case, mode):
    """batch(host_noise=True)'s draws, applied in numpy: gather, then (train) the loader's float64
    jitter / scale / shift, one rounding to fp32."""
    from sonet_b200 import augmentation as A, ops
    pts, labels, som, seg, opt = fixture_case(g, case)
    rule = ops.SAMPLE_FILL if opt.dataset == "shapenet" else ops.SAMPLE_SUBSET
    counts = [len(p) for p in pts]
    flags = dict(rot_horizontal=opt.rot_horizontal, rot_perturbation=opt.rot_perturbation,
                 translation_perturbation=opt.translation_perturbation)
    rng = np.random.RandomState(int(g["seed_" + mode]))
    sel, params = A.draw_batch_host(rng, counts, opt.input_pc_num, opt.node_num, rule,
                                    mode == "train", **flags)
    # the device dataset holds fp32 sources
    v = np.stack([p.astype(np.float32)[s] for p, s in zip(pts, sel)])       # [B,N,6]
    arrays = [v[:, :, 0:3], v[:, :, 3:6], np.stack(som).astype(np.float32)]
    if mode == "train":
        out = []
        for a, x in enumerate(arrays):
            x = x.astype(np.float64)
            sig, clip = A.JITTER_SOM if a == 2 else A.JITTER_PC
            x = np.clip(sig * params["noise"][a], -clip, clip) + x
            x = x * params["scale"][:, None, None]
            if a != 1 and params["shift"] is not None:
                x = x + params["shift"][:, None, :]
            out.append(x)
        arrays = out
    res = dict(pc=arrays[0], sn=arrays[1], som_node=arrays[2], label=labels)
    if seg is not None:
        res["seg"] = np.stack([q[s] for q, s in zip(seg, sel)]).astype(np.int64)
    return {k: (x.transpose(0, 2, 1).astype(np.float32) if x.ndim == 3 else x)
            for k, x in res.items()}


@pytest.mark.parametrize("case", CASES)
def test_host_draws_reproduce_the_loader_in_test_mode(case):
    g = golden("loader")
    want = _host_batch(g, case, "test")
    for name, x in want.items():
        assert np.array_equal(x, g["%s_test_%s" % (case, name)]), (case, name)


@pytest.mark.parametrize("case", ["modelnet", "shrec", "shapenet"])
def test_host_draws_reproduce_the_loader_in_train_mode(case):
    """Without rotations the augmentation is elementwise: the numpy restatement is bitwise."""
    g = golden("loader")
    want = _host_batch(g, case, "train")
    for name, x in want.items():
        assert np.array_equal(x, g["%s_train_%s" % (case, name)]), (case, name)


def test_fixture_covers_the_fill_rule_edges():
    g = golden("loader")
    N = int(g["N"])
    c = g["shapenet_counts"]
    assert (c < N).any() and (c == N).any() and (c > N).any()
    assert g["shrec64_points"].dtype == np.float64
