"""The oracle (CPU restatement) against the golden vectors produced by the REFERENCE ITSELF
(oracle/make_golden.py, run in the build container). This is the oracle's pin: SURVEY.md §8c —
the reference has no tests/fixtures of its own."""
import numpy as np
import pytest
import torch

from helpers import (assert_close, assert_golden, build_states, golden, golden_case,
                     golden_options, to_ref_slot_order)


def test_index_max_oracle_vs_reference_binary(oracle_mod):
    g = golden("index_max")
    out = oracle_mod.index_max(torch.from_numpy(g["kat_data"]), torch.from_numpy(g["kat_index"]), 5)
    assert out.tolist() == [[[0, 1, 0, 4, 0]]] == g["kat_out"].tolist()
    for tag in ("a", "b"):
        out = oracle_mod.index_max(torch.from_numpy(g[tag + "_data"]),
                                   torch.from_numpy(g[tag + "_index"]), int(g[tag + "_K"]))
        assert np.array_equal(out.numpy(), g[tag + "_out"])


def test_reference_plugin_binary_if_present(oracle_mod):
    m = oracle_mod.ref_plugin()
    if m is None:
        pytest.skip("oracle/_ref not built on this machine")
    g = golden("index_max")
    out = m.forward_cpu(torch.from_numpy(g["b_data"]), torch.from_numpy(g["b_index"]), int(g["b_K"]))
    assert np.array_equal(out.numpy(), g["b_out"])


# fixtures at non-default options (oracle/make_golden.py:gen_options)
OPTION_CLASSIFIERS = ["classifier_b2_n300_m121_k4", "classifier_b3_n150_m16_k1",
                      "classifier_b1_n700_m256_k2"]
AUTOENCODERS = ["autoencoder_b2_n256", "autoencoder_b2_n300_m36_conv4096"]


def _encoder_vs_reference(oracle_mod, g, opt, st, inp):
    o = oracle_mod.encoder_forward(st["encoder"], opt, inp["pc"], inp["sn"], inp["node"],
                                   inp["node_knn_I"])
    assert tuple(g["som_node__shape"]) == (opt.batch_size, 3, opt.node_num)
    assert np.array_equal(oracle_mod.canon_sets(o["min_idx"], opt.k).numpy(), g["knn_sets"])
    c_idx, _ = oracle_mod.som_topk(inp["pc"], inp["node"], opt.k)
    assert np.array_equal(oracle_mod.canon_sets(c_idx, opt.k).numpy(), g["knn_sets"])
    assert np.array_equal(o["mask_row_max"].numpy(), g["mask_row_max"])
    assert np.array_equal(o["mask_row_sum"].numpy(), g["mask_row_sum"])
    if str(g["node_mode"]) == "uniform":
        assert (g["mask_row_max"] == 0).any(), "fixture must exercise empty nodes"
    names = ["som_node", "first_pn_out_masked_max", "final_pn_out", "feature"]
    if opt.som_k >= 2:
        names += ["knn_center_1", "knn_feature_1"]
    for n in names:
        assert_golden(g, n, o[n], tol=1e-5)
    # per-copy tensors: compare in the slot order of the reference run (torch.topk(sorted=False)
    # order may differ between machines)
    assert_golden(g, "first_pn_out", to_ref_slot_order(o["first_pn_out"], o["min_idx"], g, opt.k),
                  tol=1e-5)
    return o


@pytest.mark.parametrize("name", ["classifier_b2_n256", "classifier_b2_n200_emptynodes",
                                  "classifier_b2_n256_somk0"] + OPTION_CLASSIFIERS)
def test_classifier_oracle_vs_reference(oracle_mod, name):
    g = golden(name)
    opt, inp, seed = golden_case(g, "classifier")
    st = build_states("classifier", opt, seed)
    o = _encoder_vs_reference(oracle_mod, g, opt, st, inp)
    score = oracle_mod.classifier_forward(st["head"], o["feature"])
    assert_golden(g, "score", score, tol=1e-5)


def test_option_fixtures_cover_the_options_they_are_named_for():
    """Each fixture at non-default options must still hold them (a regenerated file with the
    defaults would silently turn its tests into duplicates)."""
    want = {"classifier_b2_n300_m121_k4": dict(node_num=121, k=4, som_k_type="center",
                                               surface_normal=False),
            "classifier_b3_n150_m16_k1": dict(node_num=16, k=1),
            "classifier_b1_n700_m256_k2": dict(node_num=256, k=2),
            "segmenter_b2_n200_m100_k2": dict(node_num=100, k=2, som_k_type="avg",
                                              surface_normal=False),
            "autoencoder_b2_n300_m36_conv4096": dict(node_num=36, output_conv_pc_num=4096)}
    somk = {"classifier_b2_n300_m121_k4": 9, "classifier_b3_n150_m16_k1": 2,
            "classifier_b1_n700_m256_k2": 9, "segmenter_b2_n200_m100_k2": 9,
            "autoencoder_b2_n300_m36_conv4096": 5}
    for name, opts in want.items():
        g = golden(name)
        got = golden_options(g)
        for key, v in opts.items():
            assert got.get(key) == v, (name, key, got.get(key))
        assert int(g["som_k"]) == somk[name]
    assert int(golden("classifier_b1_n700_m256_k2")["som_k"]) * 256 == 2304   # KA_MAX_MK


def test_segmenter_oracle_vs_reference(oracle_mod):
    _segmenter_vs_reference(oracle_mod, "segmenter_b2_n128")


def test_segmenter_oracle_vs_reference_k2_without_normals(oracle_mod):
    """k=2, M=100, surface_normal=False, som_k_type='avg': the 9-channel point part of layer 1
    and the two-copy average of the head."""
    _segmenter_vs_reference(oracle_mod, "segmenter_b2_n200_m100_k2")


def _segmenter_vs_reference(oracle_mod, name):
    g = golden(name)
    opt, inp, seed = golden_case(g, "segmenter")
    st = build_states("segmenter", opt, seed)
    o = _encoder_vs_reference(oracle_mod, g, opt, st, inp)
    assert_golden(g, "centers", to_ref_slot_order(o["centers"], o["min_idx"], g, opt.k), tol=1e-6)
    assert_golden(g, "x_decentered",
                  to_ref_slot_order(o["x_decentered"], o["min_idx"], g, opt.k), tol=1e-6)
    s = oracle_mod.segmenter_forward(st["head"], opt, o, inp["pc"], inp["sn"], inp["label"])
    assert_golden(g, "score_segmenter", s, tol=1e-5)


def _decoder_cpu(opt, st):
    """networks.Decoder on CPU tensors: every layer takes the PyTorch composition of the
    reference's modules (the hand-written kernels run on CUDA tensors only)."""
    from sonet_b200 import networks
    dec = networks.Decoder(opt)
    dec.load_state_dict(st)
    return dec.eval()


@pytest.mark.parametrize("name", AUTOENCODERS)
def test_autoencoder_oracle_vs_reference(oracle_mod, name):
    g = golden(name)
    opt, inp, seed = golden_case(g, "autoencoder")
    st = build_states("autoencoder", opt, seed)
    o = _encoder_vs_reference(oracle_mod, g, opt, st, inp)
    with torch.no_grad():
        dec = _decoder_cpu(opt, st["head"])
        pred = dec(o["feature"])
    assert_golden(g, "predicted_pc", pred, tol=1e-5)
    assert_golden(g, "conv_pc4", dec.conv_pc4, tol=1e-5)
    losses = {"loss_chamfer": oracle_mod.chamfer(pred, inp["pc"]),
              "loss_chamfer_conv4": oracle_mod.chamfer(dec.conv_pc4, inp["pc"])}
    if opt.output_conv_pc_num == 4096:
        assert tuple(g["predicted_pc__shape"]) == (opt.batch_size, 3, 256 + 4096)
        assert_golden(g, "conv_pc5", dec.conv_pc5, tol=1e-5)
        assert_golden(g, "conv_pc6", dec.conv_pc6, tol=1e-5)
        losses["loss_chamfer_conv5"] = oracle_mod.chamfer(dec.conv_pc5, inp["pc"])
    for n, ch in losses.items():
        assert_close(ch["loss"], g[n], n, 1e-5)
    assert_close(sum(ch["loss"] for ch in losses.values()), g["loss"], "loss", 1e-5)
    assert_close(losses["loss_chamfer"]["loss_array"], g["loss_array"], "loss_array", 1e-5)


def test_chamfer_oracle_vs_reference(oracle_mod):
    g = golden("autoencoder_b2_n256")
    o = oracle_mod.chamfer(torch.from_numpy(g["ch_pred"]), torch.from_numpy(g["ch_gt"]))
    assert_close(o["loss"], g["ch_loss"], "chamfer loss", 1e-6)
    assert_close(o["loss_array"], g["ch_loss_array"], "chamfer loss_array", 1e-6)
    assert_close(o["forward_loss"], g["ch_forward_loss"], "forward", 1e-6)
    assert_close(o["backward_loss"], g["ch_backward_loss"], "backward", 1e-6)


def test_topk_c_restatement_matches_aten_expression(oracle_mod):
    """((x-n)**2).sum(1) == (d0*d0+d1*d1)+d2*d2 bitwise (SURVEY.md §8c) — distances, not just sets."""
    rs = np.random.RandomState(3)
    x = torch.from_numpy(rs.uniform(-1, 1, size=(2, 3, 333)).astype(np.float32))
    node = torch.from_numpy(rs.uniform(-1, 1, size=(2, 3, 64)).astype(np.float32))
    idx, dist = oracle_mod.som_topk(x, node, 3)
    d = ((x.unsqueeze(3) - node.unsqueeze(2)) ** 2).sum(dim=1)                    # B,N,M
    got = torch.gather(d, 2, idx.view(2, 3, 333).permute(0, 2, 1).long())           # B,N,k
    assert torch.equal(got, dist.view(2, 3, 333).permute(0, 2, 1))
    want = torch.topk(d, 3, dim=2, largest=False, sorted=True)[0]
    assert torch.equal(got, want)


def test_som_training_oracle_vs_reference(oracle_mod):
    """§8f-4: the oracle restatement of BatchSOM.batch_update / optimize (util/som.py:295-366)
    against what the reference itself produced (bit-exact: same ATen ops)."""
    g = golden("som_train")
    x = torch.from_numpy(g["x"])
    ni = torch.from_numpy(g["node_init_value"])
    init_w = oracle_mod.som_init_weighting_matrix(8, 8)
    n0 = ni.unsqueeze(0).expand(x.shape[0], -1, -1).contiguous()
    n1, _ = oracle_mod.som_batch_update(n0, x, init_w, 0.5, 0.4)
    n2, _ = oracle_mod.som_batch_update(n1, x, init_w, 0.31, 0.22)
    assert_close(n1, g["node_after_1"], "batch_update 1", 1e-6)
    assert_close(n2, g["node_after_2"], "batch_update 2", 1e-6)
    assert_close(oracle_mod.som_optimize(x, ni, 8, 8), g["node_optimized"], "optimize", 1e-5)


def test_potential_field_start_matches_reference():
    """BatchSOM.node_init_value (util/som.py:203-206, util/potential_field.py) restated in
    vectorised numpy: bit-equal after the reference's float32 cast."""
    from sonet_b200 import som
    g = golden("som_train")
    s = som.BatchSOM(8, 8, 3, 0, 2)
    assert np.array_equal(s.node_init_value.numpy(), g["node_init_value"])
