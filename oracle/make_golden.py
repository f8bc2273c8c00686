"""make_golden.py — TEST INFRASTRUCTURE. Generates tests/golden/*.npz from the REFERENCE ITSELF.

Run in the build container only (needs /root/reference):

    python -m oracle.make_golden

It imports the unmodified reference on CPU (oracle/ref_shims.py), loads the seeded synthetic
weights/inputs of sonet_b200.synth into the reference's own Model classes, runs their
test_model()/forward() and stores the outputs (large tensors as a strided sample). While doing so
it also checks the oracle restatement (oracle/oracle.py) against the reference — the "pin".
The fixtures are what travels to the GPU box, where /root/reference does not exist.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

from oracle import oracle, ref_shims  # noqa: E402
from sonet_b200 import synth  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
MAX_ELEMS = 1 << 15


def sample(t):
    """Strided sample of a tensor (all of it when small). Returns (values, stride)."""
    flat = t.detach().contiguous().view(-1)
    stride = max(1, -(-flat.numel() // MAX_ELEMS))
    if stride > 1 and stride % 2 == 0:
        stride += 1  # odd stride: walks over all residues of the power-of-two dims
    return flat[::stride].numpy().copy(), stride


def put(out, name, t):
    v, s = sample(t)
    out[name] = v
    out[name + "__stride"] = np.int64(s)
    out[name + "__shape"] = np.asarray(t.shape, dtype=np.int64)


def rel_err(a, b):
    return float(((a - b).abs() / b.abs().clamp(min=1.0)).max())


def load_encoder(ref_encoder, seed):
    sd = synth.synth_state_dict(ref_encoder, seed=seed)
    ref_encoder.load_state_dict(sd)
    return sd


def gen_index_max(ref):
    """Known-answer facts of SURVEY.md §8c + a random case, from the reference binary."""
    assert ref.index_max.is_reference_binary, "oracle/_ref not built"
    out = {}
    d = torch.tensor([[[1, 5, 5, -2000, 3, 3]]], dtype=torch.float32)
    i = torch.tensor([[0, 1, 1, 2, 3, 3]], dtype=torch.int32)
    r = ref.index_max.forward_cpu(d, i, 5)
    assert r.tolist() == [[[0, 1, 0, 4, 0]]], r
    out["kat_data"], out["kat_index"], out["kat_out"] = d.numpy(), i.numpy(), r.numpy()
    rs = np.random.RandomState(7)
    for tag, (B, C, N, K) in {"a": (3, 17, 301, 11), "b": (2, 40, 1024, 64)}.items():
        data = torch.from_numpy(rs.normal(size=(B, C, N)).astype(np.float32))
        data[:, :, ::7] = data[:, :, 1::7][:, :, :data[:, :, ::7].shape[2]]      # exact ties
        data[0, 0, :] = -1500.0                                                    # below sentinel
        index = torch.from_numpy(rs.randint(0, K, size=(B, N)).astype(np.int32))
        index[index == 3] = 4                                                      # node 3 empty
        r1 = ref.index_max.forward_cpu(data, index, K)
        r2 = ref.index_max.forward_multi_thread_cpu(data, index, K, 4)
        assert torch.equal(r1, r2)
        assert torch.equal(r1, oracle.index_max(data, index, K)), "oracle != reference binary"
        out[tag + "_data"], out[tag + "_index"], out[tag + "_out"] = (data.numpy(), index.numpy(),
                                                                      r1.numpy())
        out[tag + "_K"] = np.int64(K)
    np.savez_compressed(os.path.join(GOLDEN, "index_max.npz"), **out)
    print("index_max.npz: reference binary == oracle C restatement")


def run_encoder_checks(tag, opt, enc, inp, st_enc, out):
    """Store the reference encoder's cached attributes and pin the oracle against them."""
    k = opt.k
    orc = oracle.encoder_forward(st_enc, opt, inp["pc"], inp["sn"], inp["node"], inp["node_knn_I"])
    ref_min_idx = torch.max(enc.mask, dim=2)[1]                          # [B,kN] node of each copy
    sets_ref = oracle.canon_sets(ref_min_idx, k)
    c_idx, _ = oracle.som_topk(inp["pc"], inp["node"], k)
    assert torch.equal(sets_ref, oracle.canon_sets(c_idx, k)), "C top-k != reference sets"
    assert torch.equal(sets_ref, oracle.canon_sets(orc["min_idx"], k))
    out["knn_sets"] = sets_ref.numpy().astype(np.int16)
    # the reference's own slot order (topk(sorted=False) is implementation defined): needed to
    # compare per-copy tensors (first_pn_out, centers, x_decentered) position by position
    out["min_idx_ref"] = ref_min_idx.numpy().astype(np.int16)
    out["mask_row_max"] = torch.max(enc.mask, dim=1)[0].numpy()
    out["mask_row_sum"] = torch.sum(enc.mask, dim=1).numpy()
    names = ["som_node", "first_pn_out_masked_max", "final_pn_out", "feature"]
    if opt.som_k >= 2:
        names += ["knn_center_1", "knn_feature_1"]
    worst = 0.0
    for n in names:
        r = getattr(enc, n).detach()
        put(out, n, r)
        worst = max(worst, rel_err(orc[n], r))
    put(out, "first_pn_out", enc.first_pn_out.detach())
    worst = max(worst, rel_err(orc["first_pn_out"], enc.first_pn_out.detach()))
    print("  %s: oracle vs reference encoder, worst rel err %.2e" % (tag, worst))
    assert worst < 2e-5, worst
    return orc


# options a fixture may set away from synth.make_opt's defaults; each one is stored in the
# fixture (tests/helpers.golden_case rebuilds `opt` from them)
OPTION_KEYS = ("node_num", "k", "som_k", "som_k_type", "surface_normal", "input_pc_num",
               "output_fc_pc_num", "output_conv_pc_num")


def header(opt, B, N, seed, node_mode, over):
    unknown = set(over) - set(OPTION_KEYS)
    assert not unknown, "options not stored in the fixture: %s" % sorted(unknown)
    out = dict(B=np.int64(B), N=np.int64(N), seed=np.int64(seed), node_mode=np.asarray(node_mode),
               som_k=np.int64(opt.som_k), classes=np.int64(opt.classes))
    for key in over:
        if key != "som_k":                       # stored above for every fixture
            out["opt_" + key] = np.asarray(getattr(opt, key))
    return out


def gen_classifier(ref, tag, B, N, node_mode, seed, **over):
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, **over)
    model = ref.classifier.Model(opt)
    st_enc = load_encoder(model.encoder, seed)
    st_cls = synth.synth_state_dict(model.classifier, seed=seed + 1)
    model.classifier.load_state_dict(st_cls)
    inp = synth.synth_inputs(B, N, opt.node_num, max(opt.som_k, 1), seed=seed, node_mode=node_mode)
    model.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    with torch.no_grad():
        model.test_model()
    out = header(opt, B, N, seed, node_mode, over)
    orc = run_encoder_checks(tag, opt, model.encoder, inp, st_enc, out)
    put(out, "score", model.score.detach())
    s = oracle.classifier_forward(st_cls, orc["feature"])
    assert rel_err(s, model.score.detach()) < 2e-5
    np.savez_compressed(os.path.join(GOLDEN, tag + ".npz"), **out)
    print("wrote", tag)


def gen_segmenter(ref, tag, B, N, seed, node_mode="sampled", **over):
    opt = synth.make_opt("segmenter", batch_size=B, input_pc_num=N, **over)
    model = ref.segmenter.Model(opt)
    st_enc = load_encoder(model.encoder, seed)
    st_seg = synth.synth_state_dict(model.segmenter, seed=seed + 1)
    model.segmenter.load_state_dict(st_seg)
    inp = synth.synth_inputs(B, N, opt.node_num, max(opt.som_k, 1), seed=seed, node_mode=node_mode)
    seg = torch.zeros(B, N, dtype=torch.int64)
    model.set_input(inp["pc"], inp["sn"], inp["label"], seg, inp["node"], inp["node_knn_I"])
    with torch.no_grad():
        model.test_model()
    out = header(opt, B, N, seed, node_mode, over)
    orc = run_encoder_checks(tag, opt, model.encoder, inp, st_enc, out)
    put(out, "score_segmenter", model.score_segmenter.detach())
    put(out, "centers", model.encoder.centers.detach())
    put(out, "x_decentered", model.encoder.x_decentered.detach())
    s = oracle.segmenter_forward(st_seg, opt, orc, inp["pc"], inp["sn"], inp["label"])
    e = rel_err(s, model.score_segmenter.detach())
    print("  %s: oracle vs reference segmenter score rel err %.2e" % (tag, e))
    assert e < 2e-5
    np.savez_compressed(os.path.join(GOLDEN, tag + ".npz"), **out)
    print("wrote", tag)


def gen_autoencoder(ref, tag, B, N, seed, node_mode="sampled", **over):
    opt = synth.make_opt("autoencoder", batch_size=B, input_pc_num=N, **over)
    model = ref.autoencoder.Model(opt)
    st_enc = load_encoder(model.encoder, seed)
    model.decoder.load_state_dict(synth.synth_state_dict(model.decoder, seed=seed + 1))
    inp = synth.synth_inputs(B, N, opt.node_num, max(opt.som_k, 1), seed=seed, node_mode=node_mode)
    model.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    with torch.no_grad():
        model.test_model()
    out = header(opt, B, N, seed, node_mode, over)
    run_encoder_checks(tag, opt, model.encoder, inp, st_enc, out)
    put(out, "predicted_pc", model.predicted_pc.detach())
    put(out, "conv_pc4", model.decoder.conv_pc4.detach())
    if opt.output_conv_pc_num == 4096:           # the test-time conv5 loss exists only then
        put(out, "conv_pc5", model.decoder.conv_pc5.detach())
        put(out, "conv_pc6", model.decoder.conv_pc6.detach())
        out["loss_chamfer_conv5"] = model.loss_chamfer_conv5.detach().numpy()
    out["loss_chamfer"] = model.loss_chamfer.detach().numpy()
    out["loss_chamfer_conv4"] = model.loss_chamfer_conv4.detach().numpy()
    out["loss"] = model.loss.detach().numpy()
    crit = model.chamfer_criteria                     # state after the last call = predicted_pc
    out["forward_loss"] = crit.forward_loss.detach().numpy()
    out["backward_loss"] = crit.backward_loss.detach().numpy()
    out["loss_array"] = crit.loss_array.detach().numpy()
    o = oracle.chamfer(model.predicted_pc.detach(), inp["pc"])
    assert abs(float(o["loss"]) - float(model.loss_chamfer)) < 1e-6 * max(1, float(o["loss"]))
    assert rel_err(o["loss_array"], crit.loss_array.detach()) < 1e-6
    # a standalone Chamfer fixture (inputs stored in full): pred [2,3,96] vs gt [2,3,200]
    rs = np.random.RandomState(99)
    pred = torch.from_numpy(rs.uniform(-1, 1, size=(2, 3, 96)).astype(np.float32))
    gt = torch.from_numpy(rs.uniform(-1, 1, size=(2, 3, 200)).astype(np.float32))
    loss = crit(pred, gt)
    out["ch_pred"], out["ch_gt"], out["ch_loss"] = pred.numpy(), gt.numpy(), loss.numpy()
    out["ch_loss_array"] = crit.loss_array.numpy()
    out["ch_forward_loss"] = crit.forward_loss.numpy()
    out["ch_backward_loss"] = crit.backward_loss.numpy()
    np.savez_compressed(os.path.join(GOLDEN, tag + ".npz"), **out)
    print("wrote", tag)


def som_cloud(rs, B, N):
    """Seeded surface-like clouds for SOM training: points on randomly scaled ellipsoids."""
    x = rs.normal(size=(B, 3, N)).astype(np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    x *= rs.uniform(0.3, 1.0, size=(B, 3, 1)).astype(np.float32)
    return np.ascontiguousarray(x, dtype=np.float32)


# SOM training fixtures: (file, grid side, clouds, points, cloud seed). The reference's scripts
# default to an 8x8 grid; the others cover the library's range of square grids (3x3 .. 16x16).
SOM_TRAIN_CASES = (("som_train", 8, 3, 700, 17), ("som_train_m9", 3, 2, 700, 18),
                   ("som_train_m121", 11, 2, 700, 19), ("som_train_m256", 16, 2, 700, 20))


def gen_som_train(ref):
    """§8f-4: BatchSOM.optimize / batch_update of the reference (util/som.py:295-366) on seeded
    clouds, one fixture per grid size of SOM_TRAIN_CASES; pins the oracle restatement
    bit-exactly against it at every size."""
    for tag, rows, B, N, seed in SOM_TRAIN_CASES:
        gen_som_train_grid(ref, tag, rows, B, N, seed)


def gen_som_train_grid(ref, tag, rows, B, N, seed):
    rs = np.random.RandomState(seed)
    x = torch.from_numpy(som_cloud(rs, B, N))
    som = ref.som.BatchSOM(rows, rows, 3, 0, B)
    out = dict(x=x.numpy(), node_init_value=som.node_init_value.numpy().copy())
    som.node_init(B)
    som.batch_update(x, 0.5, 0.4)                       # one step from the potential-field start
    out["node_after_1"] = som.node.numpy().copy()
    som.batch_update(x, 0.31, 0.22)                     # a second one with a narrower neighbourhood
    out["node_after_2"] = som.node.numpy().copy()
    init_w = oracle.som_init_weighting_matrix(rows, rows)
    assert torch.equal(init_w, som.init_weighting_matrix)
    n0 = som.node_init_value.unsqueeze(0).expand(B, -1, -1).contiguous()
    n1, _ = oracle.som_batch_update(n0, x, init_w, 0.5, 0.4)
    n2, _ = oracle.som_batch_update(n1, x, init_w, 0.31, 0.22)
    assert torch.equal(n1, torch.from_numpy(out["node_after_1"])), "oracle batch_update != reference"
    assert torch.equal(n2, torch.from_numpy(out["node_after_2"]))
    som.optimize(x)
    out["node_optimized"] = som.node.numpy().copy()
    o = oracle.som_optimize(x, som.node_init_value, rows, rows)
    assert torch.equal(o, som.node), "oracle som_optimize != reference"
    np.savez_compressed(os.path.join(GOLDEN, tag + ".npz"), **out)
    print("%s.npz: reference BatchSOM == oracle restatement (bit-exact)" % tag)


def gen_augment(ref):
    """§8f-3: the loader's augmentation tail (data/modelnet_shrec_loader.py:218-247) executed with
    the REFERENCE's own data/augmentation.py functions on seeded clouds, numpy global RNG seeded —
    the fixture the on-device augmentation must reproduce from the same seed."""
    import importlib
    aug = importlib.import_module("data.augmentation")          # the reference's module
    rs = np.random.RandomState(31)
    B, N, M = 3, 257, 64
    pc = rs.uniform(-1, 1, size=(B, N, 3)).astype(np.float32)
    sn = rs.normal(size=(B, N, 3)).astype(np.float32)
    sn /= np.linalg.norm(sn, axis=2, keepdims=True)
    som = rs.uniform(-1, 1, size=(B, M, 3)).astype(np.float32)
    out = dict(pc=pc.transpose(0, 2, 1).copy(), sn=sn.transpose(0, 2, 1).copy(),
               som=som.transpose(0, 2, 1).copy(), np_seed=np.int64(4242))
    for tag, (rh, rp, tp) in {"all": (True, True, True), "plain": (False, False, False)}.items():
        np.random.seed(4242)
        res = [[], [], []]
        for b in range(B):                                        # loader :224-247, verbatim order
            pc_np, sn_np, som_np = pc[b], sn[b], som[b]
            if rh:
                pc_np, sn_np, som_np = aug.rotate_point_cloud_with_normal_som(pc_np, sn_np, som_np)
            if rp:
                pc_np, sn_np, som_np = aug.rotate_perturbation_point_cloud_with_normal_som(
                    pc_np, sn_np, som_np)
            pc_np = aug.jitter_point_cloud(pc_np)
            sn_np = aug.jitter_point_cloud(sn_np)
            som_np = aug.jitter_point_cloud(som_np, sigma=0.04, clip=0.1)
            scale = np.random.uniform(low=0.8, high=1.2)
            pc_np, som_np, sn_np = pc_np * scale, som_np * scale, sn_np * scale
            if tp:
                shift = np.random.uniform(-0.1, 0.1, (1, 3))
                pc_np += shift
                som_np += shift
            for lst, a in zip(res, (pc_np, sn_np, som_np)):
                lst.append(a.transpose().astype(np.float32))      # loader :250-256
        out[tag + "_pc"], out[tag + "_sn"], out[tag + "_som"] = (np.stack(r) for r in res)
    np.random.seed()
    np.savez_compressed(os.path.join(GOLDEN, "augment.npz"), **out)
    print("wrote augment.npz")


STATE_KEY_CASES = (("classifier", 9, True), ("classifier", 0, True), ("segmenter", 9, True),
                   ("autoencoder", 9, True), ("classifier", 1, True), ("segmenter", 1, True),
                   ("classifier", 9, False), ("segmenter", 9, False), ("autoencoder", 9, False))


def gen_options(ref):
    """Fixtures at non-default options of the reference's scripts: node_num (any square, up to the
    library's 256), k from 1 to 4, som_k / som_k_type, surface_normal off, the 4096-point
    auto-encoder output. Each run also pins the oracle against the reference at those options."""
    gen_classifier(ref, "classifier_b2_n300_m121_k4", 2, 300, "sampled", seed=6, node_num=121, k=4,
                   som_k=9, som_k_type="center", surface_normal=False)
    gen_classifier(ref, "classifier_b3_n150_m16_k1", 3, 150, "uniform", seed=7, node_num=16, k=1,
                   som_k=2, som_k_type="avg")
    gen_classifier(ref, "classifier_b1_n700_m256_k2", 1, 700, "sampled", seed=8, node_num=256, k=2,
                   som_k=9, som_k_type="avg")
    gen_segmenter(ref, "segmenter_b2_n200_m100_k2", 2, 200, seed=9, node_num=100, k=2, som_k=9,
                  som_k_type="avg", surface_normal=False)
    gen_autoencoder(ref, "autoencoder_b2_n300_m36_conv4096", 2, 300, seed=10, node_num=36, k=3,
                    som_k=5, som_k_type="avg", output_conv_pc_num=4096)


def gen_state_keys(ref):
    """Names and shapes of every state_dict tensor of the reference networks (checkpoint
    compatibility contract, SURVEY.md §5 'Checkpoint / resume')."""
    import json
    out = {}
    for task, som_k, sn in STATE_KEY_CASES:
        opt = synth.make_opt(task, batch_size=2, input_pc_num=64, som_k=som_k, surface_normal=sn)
        mods = {"encoder": ref.networks.Encoder(opt)}
        if task == "classifier":
            mods["classifier"] = ref.networks.Classifier(opt)
        elif task == "segmenter":
            mods["segmenter"] = ref.networks.Segmenter(opt)
        else:
            mods["decoder"] = ref.networks.Decoder(opt)
        for name, m in mods.items():
            key = "%s/som_k=%d%s/%s" % (task, som_k, "" if sn else "/no_sn", name)
            out[key] = {k: list(v.shape) for k, v in m.state_dict().items()}
    with open(os.path.join(GOLDEN, "state_keys.json"), "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print("wrote state_keys.json")


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    os.makedirs(GOLDEN, exist_ok=True)
    ref = ref_shims.install()
    only = sys.argv[1:]
    if only:                                     # e.g. `python -m oracle.make_golden som_train`
        for name in only:
            globals()["gen_" + name](ref)
        return
    gen_index_max(ref)
    gen_som_train(ref)
    gen_augment(ref)
    gen_state_keys(ref)
    gen_classifier(ref, "classifier_b2_n256", 2, 256, "sampled", seed=1)
    gen_classifier(ref, "classifier_b2_n200_emptynodes", 2, 200, "uniform", seed=2)
    gen_classifier(ref, "classifier_b2_n256_somk0", 2, 256, "sampled", seed=3, som_k=0)
    gen_segmenter(ref, "segmenter_b2_n128", 2, 128, seed=4)
    gen_autoencoder(ref, "autoencoder_b2_n256", 2, 256, seed=5)
    gen_options(ref)


if __name__ == "__main__":
    main()
