"""Small instances of every kernel family for compute-sanitizer (memcheck / racecheck / synccheck):

    compute-sanitizer --tool racecheck python tools/sanitize_all.py

classifier (fused wgmma + pool at N=5000, graph replay), segmenter, auto-encoder (up-conv decoder,
grouped / split-K GEMMs, Chamfer incl. the arg-min pass), BatchSOM training, augmentation,
query_topk with the fused mask, standalone index_max, per-cloud k-NN, normal estimation and
orientation, and one training step (BN / scatter / device pack kernels)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "so-net_b200")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sonet_b200 import (augmentation, autoencoder, classifier, networks, ops, segmenter, som,  # noqa: E402
                        synth)

dev = "cuda:0"


def build(task, B, N):
    mod = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}[task]
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, device=dev)
    cpu = synth.make_opt(task, batch_size=B, input_pc_num=N)
    m = mod.Model(opt)
    m.encoder.load_state_dict(synth.synth_state_dict(networks.Encoder(cpu), seed=1))
    head = {"classifier": ("classifier", networks.Classifier), "segmenter": ("segmenter", networks.Segmenter),
            "autoencoder": ("decoder", networks.Decoder)}[task]
    getattr(m, head[0]).load_state_dict(synth.synth_state_dict(head[1](cpu), seed=2))
    inp = synth.synth_inputs(B, N, seed=3)
    args = [inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"]]
    if task == "segmenter":
        args.insert(3, torch.zeros(B, N, dtype=torch.int64))
    return m, args


m, a = build("classifier", 2, 5000)
m.set_input(*a); m.test_model()
m.enable_cuda_graph(True)
for _ in range(2):
    m.set_input(*a); m.test_model()
print("classifier", float(m.score.sum()))
m, a = build("segmenter", 2, 512)
m.set_input(*a); m.test_model()
print("segmenter", float(m.score_segmenter.sum()))
m, a = build("autoencoder", 2, 1024)
m.set_input(*a); m.test_model()
print("autoencoder", float(m.loss))
g = torch.Generator(device=dev).manual_seed(0)
pred = torch.rand(2, 3, 300, device=dev, generator=g)
gt = torch.rand(2, 3, 1100, device=dev, generator=g)
r = ops.chamfer(pred, gt, want_idx=True)
print("chamfer idx", int(r["idx_fwd"].sum()))
pts = torch.rand(1 + 1100 + 2500, 6, device=dev, generator=g)
off = torch.tensor([0, 1, 1101, 3601], dtype=torch.int64, device=dev)
r = ops.chamfer_ragged(torch.rand(3, 3, 300, device=dev, generator=g), pts, off, want_idx=True)
print("chamfer_ragged idx", int(r["idx_fwd"].sum()), int(r["idx_bwd"].sum()))
tgt = torch.randint(0, 50, (3601,), device=dev, generator=g)
loss, arr = ops.seg_loss_ragged(torch.randn(3601, 50, device=dev, generator=g), tgt, off)
print("seg_loss_ragged", float(loss), float(arr.sum()))
x = torch.rand(2, 3, 1000, device=dev, generator=g) * 2 - 1
s = som.BatchSOM(8, 8, 3, 0, 2)
s.optimize(x)
mask, rm, idx = s.query_topk(x, 3)
print("som", float(s.node.sum()), int(mask.sum()))
opt = synth.make_opt("classifier")
opt.rot_horizontal = opt.rot_perturbation = opt.translation_perturbation = True
out = augmentation.prepare_batch(x, x.clone(), s.node, opt, True, rng=np.random.RandomState(0), seed=1)
print("augment", float(out[0].sum()), int(out[3].sum()))
data = torch.randn(2, 40, 1000, device=dev, generator=g)
index = torch.randint(0, 64, (2, 1000), device=dev, generator=g, dtype=torch.int32)
print("index_max", int(ops.index_max(data, index, 64).sum()))
pts = torch.rand(1500, 6, device=dev, generator=g)
offs = torch.tensor([0, 100, 100, 1500], dtype=torch.int64, device=dev)
nb, _ = ops.point_knn(pts, offs, 16)
nrm, _ = ops.estimate_normals(pts, offs, nb, ops.NORMALS_AWAY_FROM_CENTROID, out=pts[:, 3:6])
print("normals", int(nb.sum()), float(nrm.sum()))
_, comp = ops.orient_normals(pts, offs, nb, pts[:, 3:6], ops.NORMALS_AWAY_FROM_CENTROID, want_component=True)
print("orient", int(comp.sum()), float(pts[:, 3:6].sum()))
m, a = build("classifier", 4, 256)
m.set_input(*a)
m.optimize()
print("train step", float(m.loss))
torch.cuda.synchronize()
print("done")
