"""Whole clouds of any size: classifier.Model.score_clouds (networks.Encoder.forward_ragged),
autoencoder.Model.reconstruct_clouds and segmenter.Model.segment_clouds against the dense
test_model() on the same clouds, and batches of clouds of mixed sizes.

    python tools/ragged_bench.py [--reps 20] [--task all|classifier|autoencoder|segmenter]
                                 [--out results.json]

  A  64 clouds x 10,000 points as one ragged batch, against dense test_model() at N = 10,000 and
     N = 5,000 on the same clouds (eager and with the eval CUDA graph).
  B  1,024 clouds with P uniform in [2,000, 10,000]: clouds/s and points/s, and the time split
     between assignment + sort, the first PointResNet + pool and the node-level stage (a separate
     run with per-call CUDA events, ops.PROFILE).

  AE_A, AE_B  the same two cases for the auto-encoder (reconstruct_clouds: the ragged encoder, the
     decoder once over all features and the Chamfer terms against the whole clouds), the dense
     side at N = 10,000; AE_B splits the time into encoder, decoder and Chamfer (CUDA events
     around each stage) and gives the Chamfer's pair rate.

  SEG_A  the segmenter on B = 32 shapes of 2,000 - 3,000 points (tools/seg_full_bench.py's shapes):
     segment_clouds with its loss, against test_model() at N = 1,024 + score_points over every point
     of the same shapes.
  SEG_B  segment_clouds with its loss on 64 clouds x 10,000 points. Both split the time into the
     ragged encoder, the per-point head (node/cloud addend and every point through the head) and
     the ragged loss (CUDA events around each stage).

  TRAIN_A  optimize_clouds on 32 clouds x 10,000 points (augmented by DeviceDataset.full_batch(train=
     True)), against eager dense optimize() on the same clouds at N = 10,000 and N = 5,000.
  TRAIN_B  optimize_clouds on 32 clouds with P uniform in [2,000, 10,000]. Both split one step into
     augmentation, SOM (assignment, cluster means, decentring), the first PointResNet's forward +
     backward (with the per-node max), the node-level stage's forward + backward (KNN module, final
     PointNet, head and loss) and the optimizer (CUDA events; the backward split by a gradient hook
     on the pooled features), and give the peak device memory of a step.

Times are medians of --reps warm calls, each bracketed by CUDA events. Synthetic clouds and weights
(synth.py), the default options of each task (k = 3, 8x8 SOM, som_k = 9; the auto-encoder's
256 + 1024 output points); SONET_TC as set.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "so-net_b200")]

from sonet_b200 import (augmentation, autoencoder, classifier, networks, ops, synth,  # noqa: E402
                        train_ops)

DEV = torch.device("cuda:0")


def median_ms(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def model(B, N, states, graph=False):
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device=DEV)
    m = classifier.Model(opt)
    m.encoder.load_state_dict(states[0])
    m.classifier.load_state_dict(states[1])
    m.encoder.eval()
    m.classifier.eval()
    m.enable_cuda_graph(graph)
    return m


def clouds(sizes, M, seed):
    rs = np.random.RandomState(seed)
    pts, nodes = [], []
    for P in sizes:
        xyz = rs.uniform(-1, 1, size=(P, 3)).astype(np.float32)
        n = rs.normal(size=(P, 3)).astype(np.float32)
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        pts.append(np.concatenate([xyz, n], axis=1))
        nodes.append(xyz[rs.choice(P, M, replace=False)].T)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return (torch.from_numpy(np.concatenate(pts)).to(DEV), torch.from_numpy(off).to(DEV),
            torch.from_numpy(np.ascontiguousarray(np.stack(nodes))).to(DEV))


def stage_split(m, pts, off, node, knn):
    """Per-stage device time of one score_clouds call from per-call CUDA events."""
    ops.PROFILE = []
    m.score_clouds(pts, off, node, knn)
    torch.cuda.synchronize()
    split = {"assign_sort": 0.0, "first_pointresnet_pool": 0.0, "node_level": 0.0}
    for name, e0, e1, _ in ops.PROFILE:
        ms = e0.elapsed_time(e1)
        if "ragged" in name and "pointresnet" not in name:
            split["assign_sort"] += ms
        elif "pointresnet_tc_pool_ragged" in name or name == "sonet_pool_finalize":
            split["first_pointresnet_pool"] += ms
        else:
            split["node_level"] += ms
    ops.PROFILE = None
    return split


def ae_model(B, N, states, graph=False):
    opt = synth.make_opt("autoencoder", batch_size=B, input_pc_num=N, device=DEV)
    m = autoencoder.Model(opt)
    m.encoder.load_state_dict(states[0])
    m.decoder.load_state_dict(states[1])
    m.encoder.eval()
    m.decoder.eval()
    m.enable_cuda_graph(graph)
    return m


def ae_stage_split(m, pts, off, node, knn, reps):
    """Median device time of reconstruct_clouds' three stages, each between CUDA events: the
    ragged encoder, the decoder, and the Chamfer terms (with their offsets checks)."""
    from sonet_b200 import losses
    ts = {"encoder": [], "decoder": [], "chamfer": []}
    for i in range(reps + 3):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        with torch.no_grad():
            ev[0].record()
            feat = m.encoder.forward_ragged(pts, off, node, knn)
            ev[1].record()
            pc, parts = m.decoder.outputs(feat)
            ev[2].record()
            for t in (parts["conv_pc4"], pc):
                losses.chamfer_ragged(t, pts, off)
            ev[3].record()
        ev[3].synchronize()
        if i >= 3:
            for j, k in enumerate(ts):
                ts[k].append(ev[j].elapsed_time(ev[j + 1]))
    return {k: float(np.median(v)) for k, v in ts.items()}


def autoencoder_cases(res, reps):
    cpu_opt = synth.make_opt("autoencoder")
    states = (synth.synth_state_dict(networks.Encoder(cpu_opt), seed=1),
              synth.synth_state_dict(networks.Decoder(cpu_opt), seed=2))
    B, P, M = 64, 10000, 64
    pts, off, node = clouds([P] * B, M, seed=0)
    knn = augmentation.som_knn(node, 9, M)
    m = ae_model(B, P, states)
    res["AE_A_ragged_64x10000_ms"] = median_ms(lambda: m.reconstruct_clouds(pts, off, node, knn),
                                               reps)
    pc = pts.view(B, P, 6)[:, :, :3].permute(0, 2, 1).contiguous().cpu()
    sn = pts.view(B, P, 6)[:, :, 3:].permute(0, 2, 1).contiguous().cpu()
    for graph in (False, True):
        md = ae_model(B, P, states, graph)

        def dense():
            md.set_input(pc, sn, torch.zeros(B, dtype=torch.int64), node.cpu(), knn.cpu())
            md.test_model()
        res["AE_A_dense_N%d_%s_ms" % (P, "graph" if graph else "eager")] = median_ms(dense, reps)
        del md
    del m
    torch.cuda.empty_cache()

    rs = np.random.RandomState(5)
    sizes = rs.randint(2000, 10001, size=1024)
    pts, off, node = clouds(sizes, M, seed=1)
    knn = augmentation.som_knn(node, 9, M)
    m = ae_model(1, 256, states)
    t = median_ms(lambda: m.reconstruct_clouds(pts, off, node, knn), reps)
    res["AE_B_mixed_1024_ms"] = t
    res["AE_B_points"] = int(sizes.sum())
    res["AE_B_clouds_per_s"] = 1024 / (t[0] * 1e-3)
    split = ae_stage_split(m, pts, off, node, knn, reps)
    res["AE_B_split_ms"] = split
    # predicted_pc (1,280 points) and conv_pc4 (256) against every point, both directions at once
    pairs = (1280 + 256) * float(sizes.sum())
    res["AE_B_chamfer_pairs"] = pairs
    res["AE_B_chamfer_pairs_per_s"] = pairs / (split["chamfer"] * 1e-3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--task", choices=("all", "classifier", "autoencoder", "segmenter", "train"),
                    default="all")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_bench: needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = dict(gpu=gpu, sonet_tc=os.environ.get("SONET_TC", "1"), reps=a.reps)
    if a.task in ("all", "autoencoder"):
        autoencoder_cases(res, a.reps)
    if a.task in ("all", "classifier"):
        classifier_cases(res, a.reps)
    if a.task in ("all", "segmenter"):
        segmenter_cases(res, a.reps)
    if a.task in ("all", "train"):
        train_cases(res, a.reps)
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


def classifier_cases(res, reps):
    cpu_opt = synth.make_opt("classifier")
    states = (synth.synth_state_dict(networks.Encoder(cpu_opt), seed=1),
              synth.synth_state_dict(networks.Classifier(cpu_opt), seed=2))

    # ---- A: 64 x 10,000 ragged against dense N = 10,000 and N = 5,000 ----
    B, P, M = 64, 10000, 64
    pts, off, node = clouds([P] * B, M, seed=0)
    knn = augmentation.som_knn(node, 9, M)
    m = model(B, P, states)
    res["A_ragged_64x10000_ms"] = median_ms(lambda: m.score_clouds(pts, off, node, knn), reps)
    for N in (10000, 5000):
        pc = pts.view(B, P, 6)[:, :N, :3].permute(0, 2, 1).contiguous().cpu()
        sn = pts.view(B, P, 6)[:, :N, 3:].permute(0, 2, 1).contiguous().cpu()
        for graph in (False, True):
            md = model(B, N, states, graph)

            def dense():
                md.set_input(pc, sn, torch.zeros(B, dtype=torch.int64), node.cpu(), knn.cpu())
                md.test_model()
            # set_input's host-to-device copy is part of the dense call, as in bench.py
            res["A_dense_N%d_%s_ms" % (N, "graph" if graph else "eager")] = median_ms(dense, reps)
            del md
    del m
    torch.cuda.empty_cache()

    # ---- B: 1,024 clouds of 2,000 - 10,000 points ----
    rs = np.random.RandomState(5)
    sizes = rs.randint(2000, 10001, size=1024)
    pts, off, node = clouds(sizes, M, seed=1)
    knn = augmentation.som_knn(node, 9, M)
    m = model(1, 256, states)
    t = median_ms(lambda: m.score_clouds(pts, off, node, knn), reps)
    res["B_mixed_1024_ms"] = t
    res["B_points"] = int(sizes.sum())
    res["B_clouds_per_s"] = 1024 / (t[0] * 1e-3)
    res["B_points_per_s"] = float(sizes.sum()) / (t[0] * 1e-3)
    res["B_split_ms"] = stage_split(m, pts, off, node, knn)


def seg_stage_split(m, pts, off, label, node, knn, seg, reps):
    """Median device time of segment_clouds' three stages, each between CUDA events: the ragged
    encoder, the per-point head (node/cloud addend + every point through the head) and the loss."""
    from sonet_b200 import losses
    enc, head, T = m.encoder, m.segmenter, pts.shape[0]
    ts = {"encoder": [], "head": [], "loss": []}
    for i in range(reps + 3):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        with torch.no_grad():
            ev[0].record()
            feat, nodes = enc.forward_ragged(pts, off, node, knn, return_nodes=True)
            ev[1].record()
            addend, packed = head._node_addend(12, 384, nodes["first_pn_out_masked_max"],
                                               nodes["knn_feature_1"], nodes["final_pn_out"],
                                               feat, label)
            score = m._point_head(pts, off, node, nodes["som_node"], addend, packed, T, None)
            ev[2].record()
            losses.seg_loss_ragged(score, seg, off)
            ev[3].record()
        ev[3].synchronize()
        if i >= 3:
            for j, k in enumerate(ts):
                ts[k].append(ev[j].elapsed_time(ev[j + 1]))
    return {k: float(np.median(v)) for k, v in ts.items()}


def segmenter_cases(res, reps):
    import seg_full_bench
    from sonet_b200 import segmenter
    cpu_opt = synth.make_opt("segmenter")
    states = (synth.synth_state_dict(networks.Encoder(cpu_opt), seed=1),
              synth.synth_state_dict(networks.Segmenter(cpu_opt), seed=2))

    def seg_model(B, N):
        opt = synth.make_opt("segmenter", batch_size=B, input_pc_num=N, device=DEV)
        m = segmenter.Model(opt)
        m.encoder.load_state_dict(states[0])
        m.segmenter.load_state_dict(states[1])
        m.encoder.eval()
        m.segmenter.eval()
        return m

    # ---- SEG_A: 32 shapes of 2,000 - 3,000 points, dense N = 1,024 + score_points ----
    batch, h_pts, h_off, h_seg, sizes = seg_full_bench.make_case()
    B, N = seg_full_bench.B, seg_full_bench.N
    batch = [t.to(DEV) for t in batch]
    pts, off = torch.from_numpy(h_pts).to(DEV), torch.from_numpy(h_off).to(DEV)
    seg, label, node, knn = torch.from_numpy(h_seg).to(DEV), batch[2], batch[4], batch[5]
    m = seg_model(B, N)
    m.set_input(*batch)

    def dense():
        m.test_model()
        m.score_points(pts, off)
    res["SEG_A_points"] = int(sizes.sum())
    res["SEG_A_dense_N%d_test_model_score_points_ms" % N] = median_ms(dense, reps)
    res["SEG_A_ragged_ms"] = median_ms(
        lambda: m.segment_clouds(pts, off, label, node, knn, seg=seg), reps)
    res["SEG_A_split_ms"] = seg_stage_split(m, pts, off, label, node, knn, seg, reps)
    del m
    torch.cuda.empty_cache()

    # ---- SEG_B: 64 clouds x 10,000 points ----
    B, P, M = 64, 10000, 64
    pts, off, node = clouds([P] * B, M, seed=0)
    knn = augmentation.som_knn(node, 9, M)
    rs = np.random.RandomState(3)
    label = torch.from_numpy(rs.randint(0, 16, size=B).astype(np.int64)).to(DEV)
    seg = torch.from_numpy(np.concatenate([rs.choice(ops.SHAPENET_PART_TABLE[l], size=P)
                                           for l in label.tolist()])).to(DEV)
    m = seg_model(1, 256)
    t = median_ms(lambda: m.segment_clouds(pts, off, label, node, knn, seg=seg), reps)
    res["SEG_B_ragged_64x10000_ms"] = t
    res["SEG_B_points_per_s"] = B * P / (t[0] * 1e-3)
    res["SEG_B_split_ms"] = seg_stage_split(m, pts, off, label, node, knn, seg, reps)
    del m
    torch.cuda.empty_cache()



# ---- training on whole clouds -----------------------------------------------------------------------
def train_model(B, N, states):
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, device=DEV, rot_horizontal=True,
                         rot_perturbation=True, translation_perturbation=True)
    m = classifier.Model(opt)
    m.encoder.load_state_dict(states[0])
    m.classifier.load_state_dict(states[1])
    return m


def train_stage_split(m, ds, idx, reps):
    """Median device time of one optimize_clouds step's stages, each between CUDA events: the step
    written out as optimize_clouds runs it, the backward split by a hook on the pooled features'
    gradient (the node-level stage's backward ends there, the first PointResNet's begins)."""
    enc, opt = m.encoder, m.opt
    k, M = opt.k, ds.node_num
    names = ("augment", "som", "first_pointresnet_fwd_bwd", "node_level_fwd_bwd", "optimizer")
    ts = {n: [] for n in names}
    rng = np.random.RandomState(0)
    for i in range(reps + 3):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(8)]
        ev[0].record()
        pts, off, label, node, knn = ds.full_batch(idx, opt, train=True, rng=rng, seed=i)
        ev[1].record()
        m.encoder.train()
        m.classifier.train()
        with torch.no_grad():
            a, _, _ = ops.som_assign_ragged(pts, off, node, k)
            _, _, _, cm = ops.som_group_decenter_ragged(pts, off, a, M, k, True)
            x_aug = ops.som_decenter_ragged(pts, off, a, cm, k, True)
            cols = off * k
        ev[2].record()
        with torch.enable_grad():
            fpo = enc.first_pointnet(x_aug, 0, cols=cols)
            mm = train_ops.IndexMaxGatherRagged.apply(fpo, a, off, cols, M, k)
            mm.register_hook(lambda g: ev[5].record())
            ev[3].record()
            c, f = enc.knnlayer(cm, mm, knn, opt.som_k, opt.som_k_type, 0)
            feature = enc.final_pointnet.forward_pair(c, f, 0).max(dim=2)[0]
            loss = m.softmax_criteria(m.classifier(feature, 0, store=False), label)
            enc.zero_grad()
            m.classifier.zero_grad()
            ev[4].record()
            loss.backward()
        ev[6].record()
        for o in m._optim:
            o.step()
        ev[7].record()
        ev[7].synchronize()
        if i >= 3:
            e = lambda a, b: ev[a].elapsed_time(ev[b])  # noqa: E731
            ts["augment"].append(e(0, 1))
            ts["som"].append(e(1, 2))
            ts["first_pointresnet_fwd_bwd"].append(e(2, 3) + e(5, 6))
            ts["node_level_fwd_bwd"].append(e(3, 4) + e(4, 5))
            ts["optimizer"].append(e(6, 7))
    return {n: float(np.median(v)) for n, v in ts.items()}


def train_cases(res, reps):
    cpu_opt = synth.make_opt("classifier")
    states = (synth.synth_state_dict(networks.Encoder(cpu_opt), seed=1),
              synth.synth_state_dict(networks.Classifier(cpu_opt), seed=2))
    M = 64
    rs = np.random.RandomState(5)
    for case, sizes in (("TRAIN_A_32x10000", [10000] * 32),
                        ("TRAIN_B_mixed_32", list(rs.randint(2000, 10001, size=32)))):
        B = len(sizes)
        pts, off, node = clouds(sizes, M, seed=2)
        ds = augmentation.DeviceDataset.from_device(
            pts, off, torch.from_numpy(rs.randint(0, 40, size=B)).to(DEV), node)
        idx = np.arange(B)
        m = train_model(B, 256, states)
        rng = np.random.RandomState(1)
        batch = ds.full_batch(idx, m.opt, train=True, rng=rng, seed=0)
        res[case + "_points"] = int(sum(sizes))
        res[case + "_step_ms"] = median_ms(lambda: m.optimize_clouds(*batch, epoch=0), reps)
        res[case + "_augment_ms"] = median_ms(
            lambda: ds.full_batch(idx, m.opt, train=True, rng=rng, seed=1), reps)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(DEV)
        base = torch.cuda.memory_allocated(DEV)
        m.optimize_clouds(*batch, epoch=0)
        torch.cuda.synchronize()
        res[case + "_peak_step_bytes"] = int(torch.cuda.max_memory_allocated(DEV) - base)
        res[case + "_split_ms"] = train_stage_split(m, ds, idx, reps)
        del m
        torch.cuda.empty_cache()
        if case.startswith("TRAIN_A"):
            P = sizes[0]
            for N in (10000, 5000):
                md = train_model(B, N, states)
                pc = pts.view(B, P, 6)[:, :N, :3].permute(0, 2, 1).contiguous()
                sn = pts.view(B, P, 6)[:, :N, 3:].permute(0, 2, 1).contiguous()
                knn = augmentation.som_knn(node, 9, M)
                label = ds.labels

                def dense():
                    md.set_input(pc, sn, label, node, knn)
                    md.optimize(epoch=0)
                res["TRAIN_A_dense_optimize_N%d_ms" % N] = median_ms(dense, reps)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats(DEV)
                base = torch.cuda.memory_allocated(DEV)
                dense()
                torch.cuda.synchronize()
                res["TRAIN_A_dense_optimize_N%d_peak_step_bytes" % N] = int(
                    torch.cuda.max_memory_allocated(DEV) - base)
                del md
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
