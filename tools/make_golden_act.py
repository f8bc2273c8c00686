"""make_golden_act.py — generates ONLY the activation='elu' fixtures of tests/golden from the
REFERENCE ITSELF (the reference's `--activation elu`, nn.ELU(alpha=1.0) in every layer class).

Run in the build container only (needs the reference checkout and `build()`'s oracle/_ref):

    python tools/make_golden_act.py

Same procedure and file layout as oracle/make_golden.py (seeded synthetic weights with randomised
BatchNorm statistics and inputs from sonet_b200.synth, the reference's own Model classes on CPU,
large tensors as strided samples); each fixture also stores opt_activation = 'elu', from which
tests/helpers.golden_case rebuilds the options. Existing fixtures are not touched. The files are
named elu_<the ReLU fixture they mirror>, outside the <task>_* names that other suites enumerate
as ReLU models. The oracle restatement computes ReLU models only, so there is no oracle pin here:
the numbers are the reference's.
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

ACT = "elu"


def header(opt, B, N, seed, node_mode, over):
    out = dict(B=np.int64(B), N=np.int64(N), seed=np.int64(seed), node_mode=np.asarray(node_mode),
               som_k=np.int64(opt.som_k), classes=np.int64(opt.classes))
    for key in over:
        if key != "som_k":
            out["opt_" + key] = np.asarray(getattr(opt, key))
    return out


def encoder_outputs(opt, enc, out):
    """The reference encoder's cached attributes, as oracle/make_golden.py stores them."""
    ref_min_idx = torch.max(enc.mask, dim=2)[1]
    from oracle import oracle
    out["knn_sets"] = oracle.canon_sets(ref_min_idx, opt.k).numpy().astype(np.int16)
    out["min_idx_ref"] = ref_min_idx.numpy().astype(np.int16)
    out["mask_row_max"] = torch.max(enc.mask, dim=1)[0].numpy()
    out["mask_row_sum"] = torch.sum(enc.mask, dim=1).numpy()
    names = ["som_node", "first_pn_out_masked_max", "final_pn_out", "feature", "first_pn_out"]
    if opt.som_k >= 2:
        names += ["knn_center_1", "knn_feature_1"]
    for n in names:
        put(out, n, getattr(enc, n).detach())
    # the point of these fixtures: negative activations are present
    neg = float((enc.first_pn_out_masked_max < 0).float().mean())
    print("  share of negative first_pn_out_masked_max: %.2f" % neg)


def run(ref, task, tag, B, N, seed, node_mode="sampled", **over):
    over = dict(over, activation=ACT)
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
    assert any(isinstance(m, torch.nn.ELU) for m in model.encoder.modules()), "not an ELU model"
    with torch.no_grad():
        model.test_model()
    out = header(opt, B, N, seed, node_mode, over)
    encoder_outputs(opt, model.encoder, out)
    if task == "classifier":
        put(out, "score", model.score.detach())
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
    # the seeds, sizes and node modes of the ReLU fixtures they mirror (oracle/make_golden.py)
    run(ref, "classifier", "elu_classifier_b2_n256", 2, 256, seed=1)
    run(ref, "classifier", "elu_classifier_b2_n200_emptynodes", 2, 200, seed=2, node_mode="uniform")
    run(ref, "classifier", "elu_classifier_b2_n256_somk0", 2, 256, seed=3, som_k=0)
    run(ref, "segmenter", "elu_segmenter_b2_n128", 2, 128, seed=4)
    run(ref, "autoencoder", "elu_autoencoder_b2_n256", 2, 256, seed=5)


if __name__ == "__main__":
    main()
