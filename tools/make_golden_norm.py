"""make_golden_norm.py — generates ONLY the normalization='instance' fixtures of tests/golden from the
REFERENCE ITSELF (the reference's `--normalization instance`: nn.InstanceNorm1d/2d(C, affine=True)
in every normalised layer).

Run in the build container only (needs the reference checkout and `build()`'s oracle/_ref):

    python tools/make_golden_norm.py [--force]

Same procedure and file layout as tools/make_golden_act.py (seeded synthetic weights and inputs
from sonet_b200.synth, whose state dicts already randomise norm.weight and norm.bias, the
reference's own Model classes on CPU, large tensors as strided samples); each fixture stores
opt_normalization = 'instance', from which tests/helpers.golden_case rebuilds the options. The
files are named inst_<the fixture they mirror>, outside the <task>_* names that other suites
enumerate as batch-norm models.

The reference's classifier head and the auto-encoder's FC branch cannot run with instance norm
(MyLinear's nn.InstanceNorm1d on a [B, C] input raises under torch 2.x), so the auto-encoder runs
with output_fc_pc_num=0 and the shrec16 encoder (som_k=0) is stored from a direct call of the
reference's networks.Encoder (encoder_only = 1 in the fixture).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "so-net_b200"))

from oracle import ref_shims  # noqa: E402
from oracle.make_golden import GOLDEN, put  # noqa: E402
from sonet_b200 import synth  # noqa: E402

NORM = "instance"


def header(opt, B, N, seed, node_mode, over):
    out = dict(B=np.int64(B), N=np.int64(N), seed=np.int64(seed), node_mode=np.asarray(node_mode),
               som_k=np.int64(opt.som_k), classes=np.int64(opt.classes))
    for key in over:
        if key != "som_k":
            out["opt_" + key] = np.asarray(getattr(opt, key))
    return out


def encoder_outputs(opt, enc, out):
    """The reference encoder's cached attributes, as oracle/make_golden.py stores them."""
    from oracle import oracle
    ref_min_idx = torch.max(enc.mask, dim=2)[1]
    out["knn_sets"] = oracle.canon_sets(ref_min_idx, opt.k).numpy().astype(np.int16)
    out["min_idx_ref"] = ref_min_idx.numpy().astype(np.int16)
    out["mask_row_max"] = torch.max(enc.mask, dim=1)[0].numpy()
    out["mask_row_sum"] = torch.sum(enc.mask, dim=1).numpy()
    names = ["som_node", "first_pn_out_masked_max", "final_pn_out", "feature", "first_pn_out"]
    if opt.som_k >= 2:
        names += ["knn_center_1", "knn_feature_1"]
    for n in names:
        put(out, n, getattr(enc, n).detach())


def run(ref, task, tag, B, N, seed, node_mode="sampled", encoder_only=False, **over):
    over = dict(over, normalization=NORM)
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, **over)
    model = {"classifier": ref.classifier, "segmenter": ref.segmenter,
             "autoencoder": ref.autoencoder}[task].Model(opt)
    model.encoder.load_state_dict(synth.synth_state_dict(model.encoder, seed=seed))
    head = {"classifier": "classifier", "segmenter": "segmenter", "autoencoder": "decoder"}[task]
    getattr(model, head).load_state_dict(synth.synth_state_dict(getattr(model, head), seed=seed + 1))
    inp = synth.synth_inputs(B, N, opt.node_num, max(opt.som_k, 1), seed=seed, node_mode=node_mode)
    if task == "segmenter":
        seg = torch.zeros(B, N, dtype=torch.int64)
        model.set_input(inp["pc"], inp["sn"], inp["label"], seg, inp["node"], inp["node_knn_I"])
    else:
        model.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
    assert any(isinstance(m, torch.nn.InstanceNorm1d) for m in model.encoder.modules()), \
        "not an instance-norm model"
    with torch.no_grad():
        if encoder_only:
            model.encoder.eval()
            model.encoder(model.pc, model.sn, model.input_node, model.input_node_knn_I, False)
        else:
            model.test_model()
    out = header(opt, B, N, seed, node_mode, over)
    out["encoder_only"] = np.int64(encoder_only)
    encoder_outputs(opt, model.encoder, out)
    if encoder_only:
        pass
    elif task == "segmenter":
        put(out, "score_segmenter", model.score_segmenter.detach())
        put(out, "centers", model.encoder.centers.detach())
        put(out, "x_decentered", model.encoder.x_decentered.detach())
    else:
        put(out, "predicted_pc", model.predicted_pc.detach())
        put(out, "conv_pc4", model.decoder.conv_pc4.detach())
        out["loss_chamfer"] = model.loss_chamfer.detach().numpy()
        out["loss"] = model.loss.detach().numpy()
    path = os.path.join(GOLDEN, tag + ".npz")
    assert not os.path.exists(path) or "--force" in sys.argv, "%s exists (--force rewrites)" % path
    np.savez_compressed(path, **out)
    print("wrote", tag)


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    ref = ref_shims.install()
    # the seeds, sizes and node modes of the fixtures they mirror (oracle/make_golden.py,
    # tools/make_golden_act.py)
    run(ref, "segmenter", "inst_segmenter_b2_n128", 2, 128, seed=4)
    run(ref, "segmenter", "inst_segmenter_b2_n200_m100_k2", 2, 200, seed=9, node_num=100, k=2,
        som_k=9, som_k_type="avg", surface_normal=False)
    run(ref, "segmenter", "inst_segmenter_b2_n200_emptynodes", 2, 200, seed=2, node_mode="uniform")
    run(ref, "segmenter", "inst_elu_segmenter_b2_n128", 2, 128, seed=4, activation="elu")
    run(ref, "autoencoder", "inst_autoencoder_b2_n256", 2, 256, seed=5, output_fc_pc_num=0)
    run(ref, "classifier", "inst_shrec16_encoder_b2_n256_somk0", 2, 256, seed=3, som_k=0,
        encoder_only=True)


if __name__ == "__main__":
    main()
