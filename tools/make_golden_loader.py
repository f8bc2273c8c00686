"""make_golden_loader.py — generates ONLY tests/golden/loader.npz from the REFERENCE ITSELF: the
collated batches of data/modelnet_shrec_loader.py:ModelNet_Shrec_Loader and
data/shapenet_loader.py:ShapeNetLoader, in train and test mode, with np.random seeded, on seeded
synthetic datasets. What sonet_b200.augmentation.DeviceDataset.batch(host_noise=True) must
reproduce bit for bit.

Run in the build container only (needs the reference checkout):

    python tools/make_golden_loader.py [--force]

The datasets are written to a temporary directory in the layouts that make_dataset_modelnet40_10k,
make_dataset_shrec2016 and make_dataset_shapenet_normal read (a few hundred points per cloud). The
reference imports h5py, faiss and matplotlib; oracle/ref_shims stubs them (faiss as an exact
brute-force IndexFlatL2). Cases:
  modelnet      float32 .npy clouds, rotations off, random shift on
  modelnet_rot  the same clouds with both rotations on (numpy's BLAS may fuse the 3-term rotation
                products, so its train outputs are pinned to within 1 fp32 ulp, not bitwise)
  shrec         float32 npz clouds, shift on
  shrec64       float64 npz clouds, as SHREC's np.loadtxt data (DeviceDataset rounds them to fp32)
  shapenet      clouds with P < N, P == N and P > N, with part labels
Existing fixtures are not touched.
"""
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

from oracle import ref_shims  # noqa: E402
from oracle.make_golden import GOLDEN  # noqa: E402

N = 128                 # input_pc_num
NODE_NUM = 16           # 4x4 SOM
SOM_K = 3
SEEDS = {"train": 101, "test": 202}
SHAPENET_FOLDERS = ["02691156", "02773838", "02954340", "02958343"]


def make_opt(dataset, B, rot=False, shift=True):
    return types.SimpleNamespace(dataset=dataset, input_pc_num=N, node_num=NODE_NUM, som_k=SOM_K,
                                 classes=10, batch_size=B, rot_horizontal=rot, rot_perturbation=rot,
                                 translation_perturbation=shift)


def synth_clouds(rs, counts, dtype):
    pts, som = [], []
    for P in counts:
        xyz = rs.uniform(-1, 1, size=(P, 3))
        nrm = rs.normal(size=(P, 3))
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        pts.append(np.concatenate([xyz, nrm], axis=1).astype(dtype))
        som.append(rs.uniform(-1, 1, size=(NODE_NUM, 3)).astype(dtype))
    return pts, som


def write_modelnet(root, pts, som, labels):
    names = ["shape%d" % c for c in range(10)]
    with open(os.path.join(root, "modelnet10_shape_names.txt"), "w") as f:
        f.write("\n".join(names) + "\n")
    lines = []
    for i, (p, s, c) in enumerate(zip(pts, som, labels)):
        name = "%s_%04d" % (names[c], i + 1)
        for sub, arr in (("", p), ("4x4_som_nodes", s)):
            d = os.path.join(root, sub, names[c])
            os.makedirs(d, exist_ok=True)
            np.save(os.path.join(d, name + ".npy"), arr)
        lines.append(name)
    for mode in ("train", "test"):
        with open(os.path.join(root, "modelnet10_%s.txt" % mode), "w") as f:
            f.write("\n".join(lines) + "\n")


def write_shrec(root, pts, som, labels):
    cats = ["cat%02d" % c for c in range(55)]
    with open(os.path.join(root, "category.txt"), "w") as f:
        f.write("\n".join(cats) + "\n")
    train, test = [], []
    for i, (p, s, c) in enumerate(zip(pts, som, labels)):
        name = "%06d" % (55 * (i + 1) + c)       # test mode reads the class as int(name) % 55
        for mode in ("train", "test"):
            d = os.path.join(root, "4x4", mode)
            os.makedirs(d, exist_ok=True)
            np.savez(os.path.join(d, "model_%s.npz" % name), pc=p[:, :3], sn=p[:, 3:], som_node=s)
        train.append("%s,%s" % (name, cats[c]))
        test.append(name)
    for mode, lines in (("train", train), ("test", test)):
        with open(os.path.join(root, mode + ".txt"), "w") as f:
            f.write("\n".join(lines) + "\n")


def write_shapenet(root, pts, som, labels, seg):
    files = []
    for i, (p, s, c, q) in enumerate(zip(pts, som, labels, seg)):
        rel = "%s/model%03d" % (SHAPENET_FOLDERS[c], i)
        os.makedirs(os.path.join(root, SHAPENET_FOLDERS[c]), exist_ok=True)
        np.savez(os.path.join(root, rel + "_4x4.npz"), pc=p[:, :3], sn=p[:, 3:], part_label=q,
                 som_node=s)
        files.append("shape_data/" + rel)
    os.makedirs(os.path.join(root, "train_test_split"), exist_ok=True)
    for mode in ("train", "test"):
        with open(os.path.join(root, "train_test_split", "shuffled_%s_file_list.json" % mode), "w") as f:
            json.dump(files, f)


def collate(loader, S, seed):
    """Items 0..S-1 in order with np.random seeded, collated as the DataLoader does."""
    np.random.seed(seed)
    items = [loader[i] for i in range(S)]
    return [torch.stack([it[k] for it in items]) if torch.is_tensor(items[0][k])
            else torch.tensor([it[k] for it in items]) for k in range(len(items[0]))]


def main():
    torch.set_num_threads(4)
    ref_shims.install(use_ref_plugin=False)
    from data.modelnet_shrec_loader import ModelNet_Shrec_Loader
    from data.shapenet_loader import ShapeNetLoader

    rs = np.random.RandomState(1234)
    out = dict(N=np.int64(N), node_num=np.int64(NODE_NUM), som_k=np.int64(SOM_K),
               seed_train=np.int64(SEEDS["train"]), seed_test=np.int64(SEEDS["test"]))
    sources = {
        "modelnet": ([300, 200, N, 257], np.float32),
        "shrec": ([240, N + 1, 300, 150], np.float32),
        "shrec64": ([220, 300, N, 190], np.float64),
        "shapenet": ([100, N, N + 1, 300, N - 1], np.float32),
    }
    cases = [("modelnet", "modelnet", dict()), ("modelnet_rot", "modelnet", dict(rot=True)),
             ("shrec", "shrec", dict()), ("shrec64", "shrec64", dict()),
             ("shapenet", "shapenet", dict(shift=False))]
    with tempfile.TemporaryDirectory() as tmp:
        roots = {}
        for ds, (counts, dtype) in sources.items():
            S = len(counts)
            pts, som = synth_clouds(rs, counts, dtype)
            labels = rs.randint(0, 4, size=S)
            root = roots[ds] = os.path.join(tmp, ds)
            os.makedirs(root)
            seg = None
            if ds == "modelnet":
                write_modelnet(root, pts, som, labels)
            elif ds.startswith("shrec"):
                write_shrec(root, pts, som, labels)
            else:
                seg = [rs.randint(0, 50, size=P).astype(np.int64) for P in counts]
                write_shapenet(root, pts, som, labels, seg)
                out[ds + "_seg"] = np.concatenate(seg).astype(np.int32)
            out[ds + "_points"] = np.concatenate(pts)
            out[ds + "_counts"] = np.asarray(counts, dtype=np.int64)
            out[ds + "_labels"] = labels.astype(np.int64)
            out[ds + "_som"] = np.stack(som)
        for case, ds, kw in cases:
            S = len(sources[ds][0])
            dataset = "shrec" if ds.startswith("shrec") else ds
            opt = make_opt(dataset, S, **kw)
            out[case + "_source"] = np.asarray(ds)
            out[case + "_dataset"] = np.asarray(dataset)
            for key in ("rot_horizontal", "rot_perturbation", "translation_perturbation"):
                out["%s_opt_%s" % (case, key)] = np.asarray(getattr(opt, key))
            for mode in ("train", "test"):
                cls = ShapeNetLoader if dataset == "shapenet" else ModelNet_Shrec_Loader
                loader = cls(roots[ds], mode, opt)
                assert len(loader) == S
                batch = collate(loader, S, SEEDS[mode])
                names = (["pc", "sn", "label", "seg", "som_node", "som_knn_I"] if dataset == "shapenet"
                         else ["pc", "sn", "label", "som_node", "som_knn_I"])
                for name, t in zip(names, batch):
                    out["%s_%s_%s" % (case, mode, name)] = t.numpy()
                assert np.array_equal(batch[2].numpy(), out[ds + "_labels"]), case
                print("%s/%s: pc %s" % (case, mode, tuple(batch[0].shape)))
    path = os.path.join(GOLDEN, "loader.npz")
    assert not os.path.exists(path) or "--force" in sys.argv, "%s exists (--force rewrites)" % path
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
