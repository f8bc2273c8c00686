"""retrieval_golden.py — TEST INFRASTRUCTURE for the SHREC'16 retrieval ranking.

    python -m oracle.retrieval_golden          # needs the reference's source tree

Runs the reference's own shrec16/test.py, unmodified, as __main__ (runpy) on the CPU and writes
tests/golden/retrieval.npz. Its `Options` parse a prepared argv (--gpu_id -1 --nThreads 0, a
temporary --checkpoints_dir). Stub modules stand in for models.classifier (a Model whose forward()
serves fixture scores in loader order), data.modelnet_shrec_loader (the real one needs faiss, h5py
and matplotlib) and util.visualizer. torch.load returns an empty state, Tensor.cuda is the identity,
and np.savetxt is captured: file name, the float64 [n,2] array and the fmt.

Cases (55 classes, the script's width):
  quant    1,500 shapes, scores multiples of 1/64 (every distance exact, every tie a real tie),
           skewed class sizes with one class of 1,100 (the 1000-row cut; only a fixed subset of its
           files is stored), a singleton class, duplicate rows, argmax ties, model ids 0, 7-digit
           and one repeated id, and a final partial batch;
  float    600 shapes with unquantised scores, one row containing a NaN, a final partial batch.
"""
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
C = 55
BIG_CLASS_FILES = 40          # files stored of the class larger than the 1000-row cut


def run_reference(scores, ids, batch_size):
    """Run shrec16/test.py on `scores` [Q,55] f32 / `ids` [Q] int64; returns the captured
    np.savetxt calls [(file name, float64 array, fmt, delimiter)] in call order."""
    ref = ref_shims.REF
    state = {"pos": 0}

    class _Net:
        def load_state_dict(self, *a, **k):
            return None

        def eval(self):
            return self

    class Model:
        def __init__(self, opt):
            self.encoder, self.classifier = _Net(), _Net()

        def set_input(self, input_pc, input_sn, input_label, input_node, input_node_knn_I):
            self.batch = input_pc.shape[0]

        def forward(self):
            p = state["pos"]
            self.score = torch.from_numpy(scores[p:p + self.batch].copy())
            state["pos"] = p + self.batch

    class Loader(torch.utils.data.Dataset):
        def __init__(self, root, mode, opt):
            assert mode == "test"

        def __len__(self):
            return len(ids)

        def __getitem__(self, i):
            z = torch.zeros(1)
            return z, z, 0, z, z, torch.tensor(int(ids[i]), dtype=torch.int64)

    class Visualizer:
        def __init__(self, opt):
            pass

    stubs = {"models": types.ModuleType("models"), "models.classifier": types.ModuleType("m.c"),
             "data": types.ModuleType("data"), "data.modelnet_shrec_loader": types.ModuleType("d.l"),
             "util.visualizer": types.ModuleType("u.v")}
    stubs["models.classifier"].Model = Model
    stubs["data.modelnet_shrec_loader"].ModelNet_Shrec_Loader = Loader
    stubs["util.visualizer"].Visualizer = Visualizer
    captured = []

    def savetxt(fname, X, fmt="%.18e", delimiter=" ", **kw):
        captured.append((os.path.basename(fname), np.array(X, copy=True), fmt, delimiter))

    saved = dict(argv=sys.argv, path=list(sys.path), load=torch.load, cuda=torch.Tensor.cuda,
                 savetxt=np.savetxt, mods={k: sys.modules.get(k) for k in list(stubs) + ["util"]})
    with tempfile.TemporaryDirectory() as tmp:
        sys.argv = ["test.py", "--gpu_id", "-1", "--nThreads", "0", "--batch_size", str(batch_size),
                    "--checkpoints_dir", tmp]
        sys.path.insert(0, ref)
        sys.modules.pop("util", None)
        sys.modules.update(stubs)
        torch.load = lambda *a, **k: {}
        torch.Tensor.cuda = lambda self, *a, **k: self
        np.savetxt = savetxt
        try:
            runpy.run_path(os.path.join(ref, "shrec16", "test.py"), run_name="__main__")
        finally:
            sys.argv, sys.path[:] = saved["argv"], saved["path"]
            torch.load, torch.Tensor.cuda, np.savetxt = saved["load"], saved["cuda"], saved["savetxt"]
            for k, v in saved["mods"].items():
                if v is None:
                    sys.modules.pop(k, None)
                else:
                    sys.modules[k] = v
            for k in [k for k in sys.modules if k == "shrec16" or k.startswith(("shrec16.", "util."))]:
                sys.modules.pop(k, None)
    assert state["pos"] == len(ids)
    return captured


def _labels(rs, sizes):
    lab = np.concatenate([np.full(n, c) for c, n in enumerate(sizes)])
    return lab[rs.permutation(len(lab))]


def case_quant(rs):
    sizes = [1100, 1] + [int(v) for v in np.maximum(1, 130 / np.arange(2, 55) ** 1.1).round()]
    sizes[-1] += 1500 - sum(sizes)
    assert min(sizes) >= 1 and sum(sizes) == 1500
    lab = _labels(rs, sizes)
    Q = len(lab)
    score = np.clip(np.round(rs.normal(scale=0.5, size=(Q, C)) * 64) / 64, -1.5, 1.5)
    score[np.arange(Q), lab] = 2.0
    dup = rs.choice(Q, size=60, replace=False)
    score[dup[30:]] = score[dup[:30]]                    # duplicate rows: distance-0 ties
    lab[dup[30:]] = lab[dup[:30]]
    tie = np.nonzero(lab < 50)[0][:25]                   # argmax ties go to the lower class
    score[tie, lab[tie] + 3] = 2.0
    ids = rs.choice(np.arange(1, 900000), size=Q, replace=False).astype(np.int64)
    ids[7], ids[8] = 0, 1234567
    ids[20] = ids[21]                                    # a repeated id: the last file wins
    return score.astype(np.float32), ids, 64


def case_float(rs):
    Q = 600
    p = 1.0 / np.arange(1, C + 1) ** 0.9
    lab = rs.choice(C, size=Q, p=p / p.sum())
    score = rs.normal(size=(Q, C)).astype(np.float32)
    score[np.arange(Q), lab] += 3.0
    score[17, 9] = np.nan
    ids = rs.choice(np.arange(100000, 9999999), size=Q, replace=False).astype(np.int64)
    return score.astype(np.float32), ids, 32


def gen_retrieval():
    rs = np.random.RandomState(16)
    out, fmts = {}, set()
    for tag, make in (("quant", case_quant), ("float", case_float)):
        score, ids, bs = make(rs)
        calls = run_reference(score, ids, bs)
        assert len(calls) == len(ids)
        pred = np.array([int(torch.max(torch.from_numpy(r), 0)[1]) for r in score])
        keep = np.ones(len(ids), dtype=bool)
        big = np.nonzero(np.bincount(pred, minlength=C) > 1000)[0]
        if len(big):
            members = np.nonzero(pred == big[0])[0]
            keep[members] = False
            keep[np.sort(rs.choice(members, size=BIG_CLASS_FILES, replace=False))] = True
        rows, qs, names, off = [], [], [], [0]
        for q, (name, X, fmt, delim) in enumerate(calls):
            fmts.add((fmt, delim))
            assert name == "%06d" % ids[q] and X.dtype == np.float64 and X.shape[1] == 2
            if keep[q]:
                qs.append(q)
                names.append(name)
                rows.append(X)
                off.append(off[-1] + len(X))
        out[tag + "_score"], out[tag + "_ids"], out[tag + "_batch"] = score, ids, np.int64(bs)
        out[tag + "_file_q"] = np.asarray(qs, dtype=np.int64)
        out[tag + "_file_name"] = np.asarray(names)
        out[tag + "_file_off"] = np.asarray(off, dtype=np.int64)
        out[tag + "_rows"] = np.concatenate(rows)
        print("%s: Q=%d, %d of %d files stored, %d rows, big class %s"
              % (tag, len(ids), len(qs), len(calls), off[-1], list(big)))
    assert len(fmts) == 1
    out["fmt"], out["delimiter"] = np.asarray(next(iter(fmts))[0]), np.asarray(next(iter(fmts))[1])
    out["cases"] = np.asarray(["quant", "float"])
    np.savez_compressed(os.path.join(GOLDEN, "retrieval.npz"), **out)


def main():
    torch.set_num_threads(8)
    gen_retrieval()


if __name__ == "__main__":
    main()
