"""seg_iou_golden.py — TEST INFRASTRUCTURE for the part-segmentation metric.

    python -m oracle.seg_iou_golden          # needs the reference's source tree

load_ref_losses() imports the reference's own models/losses.py (source tree, or the bytecode build
product oracle/_ref/pyref where only that exists) as a standalone module under another name, with a
`faiss` stub in place while it executes (its only use of faiss is ChamferLoss). Nothing else is
registered, so it can sit next to sonet_b200.install()'s `models.losses`.

gen_seg_iou() runs the reference's compute_iou_np_array / compute_iou (models/losses.py:73-189) on
seeded batches and writes tests/golden/seg_iou.npz with the inputs stored in full.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

from oracle import ref_shims  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
C = 50


def _faiss_stub():
    faiss = types.ModuleType("faiss")
    faiss.IndexFlatL2 = ref_shims._IndexFlatL2
    faiss.index_cpu_to_gpu = lambda res, dev, idx: idx
    return faiss


def load_ref_losses(name="ref_models_losses", prefer_pyref=True):
    """The reference's models/losses.py as a module called `name`."""
    import importlib.util
    root = ref_shims.ref_root(prefer_pyref)
    if root is None:
        raise RuntimeError("neither the reference tree nor oracle/_ref/pyref is present")
    path = os.path.join(root, "models", "losses.py" if root == ref_shims.REF else "losses.pyc")
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    prev = sys.modules.get("faiss")
    sys.modules["faiss"] = _faiss_stub()
    try:
        spec.loader.exec_module(mod)
    finally:
        if prev is None:
            del sys.modules["faiss"]
        else:
            sys.modules["faiss"] = prev
    return mod


def _case(rs, labels, N, table):
    """Scores quantised to 1/256 (they compress), and ground truth drawn from the shape's parts,
    with the true part's score raised at 70 % of the points so that predictions are mostly right."""
    B = len(labels)
    score = np.round(rs.normal(size=(B, C, N)) * 256) / 256
    seg = np.stack([rs.choice(table[k], size=N) for k in labels]).astype(np.int64)
    hit = rs.uniform(size=(B, N)) < 0.7
    b_i, n_i = np.nonzero(hit)
    score[b_i, seg[b_i, n_i], n_i] += 2.0
    return score.astype(np.float32), seg, np.asarray(labels, dtype=np.int64)


def gen_seg_iou(ref_losses):
    """Cases: random scores over all 16 categories, exact ties, NaN scores, parts absent from both
    gt and prediction, seg values of other categories (and outside [0, C)), B = 1, and N not a
    multiple of 32. Also stores the reference module's public callables."""
    from sonet_b200.ops import SHAPENET_PART_TABLE as table    # only shapes the inputs
    rs = np.random.RandomState(23)
    cases = {}
    cases["random"] = _case(rs, list(range(16)) * 2, 97, table)
    score, seg, label = _case(rs, rs.randint(0, 16, size=8), 64, table)
    score = rs.randint(0, 3, size=score.shape).astype(np.float32)     # ties everywhere
    for b in range(8):                                                # and between two of its parts
        parts = table[label[b]]
        n = rs.choice(64, size=20, replace=False)
        score[b, :, n] = 0.0
        score[b, parts[0], n] = score[b, parts[-1], n] = 5.0
    cases["ties"] = (score, seg, label)
    score, seg, label = _case(rs, rs.randint(0, 16, size=6), 50, table)
    for b in range(6):
        n = rs.choice(50, size=10, replace=False)
        score[b, rs.randint(0, C, size=10), n] = np.nan               # one NaN
        score[b, 0, n[:3]] = np.nan                                   # first NaN at class 0
        score[b, 49, n[3:6]] = np.nan                                 # two NaNs at these points
    cases["nan"] = (score, seg, label)
    score, seg, label = _case(rs, [0, 3, 10, 15], 40, table)
    for b in range(4):                                                # only the first part occurs
        p = table[label[b]][0]
        seg[b] = p
        score[b, p] += 100.0
    cases["absent"] = (score, seg, label)
    score, seg, label = _case(rs, rs.randint(0, 16, size=6), 45, table)
    seg = rs.randint(-3, 61, size=seg.shape).astype(np.int64)         # any category, and outside
    seg[:, ::9] = 1 << 40
    cases["foreign"] = (score, seg, label)
    cases["b1"] = _case(rs, [10], 300, table)
    cases["odd_n"] = _case(rs, rs.randint(0, 16, size=5), 333, table)
    out = {}
    for tag, (score, seg, label) in cases.items():
        args = (torch.from_numpy(score), torch.from_numpy(seg), torch.from_numpy(label), None, None,
                None)
        per_shape = ref_losses.compute_iou_np_array(*args)
        miou = ref_losses.compute_iou(*args)
        assert per_shape.dtype == np.float64 and miou == per_shape.mean()
        out[tag + "_score"], out[tag + "_seg"], out[tag + "_label"] = score, seg, label
        out[tag + "_iou"], out[tag + "_miou"] = per_shape, np.float64(miou)
    out["cases"] = np.asarray(list(cases))
    out["ref_public_callables"] = np.asarray(sorted(
        k for k, v in vars(ref_losses).items()
        if not k.startswith("_") and callable(v) and getattr(v, "__module__", None) == ref_losses.__name__))
    np.savez_compressed(os.path.join(GOLDEN, "seg_iou.npz"), **out)
    print("wrote seg_iou.npz:", ", ".join(cases), "/", " ".join(out["ref_public_callables"]))


def main():
    torch.set_num_threads(8)
    gen_seg_iou(load_ref_losses(prefer_pyref=False))


if __name__ == "__main__":
    main()
