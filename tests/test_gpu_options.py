"""-m gpu: model parity at SO-Net's non-default options (node_num, k, som_k, som_k_type,
surface_normal, output_conv_pc_num) and on every dispatch path of the encoder.

  (a) against the fixtures the reference itself produced at those options;
  (b) against the oracle on fresh seeded inputs, one case on each side of every dispatch
      boundary (som_group staged / unstaged / not at all, knn_assemble_pool's M*K limit, empty
      nodes, one point per cloud), with the boundaries taken from the library's own arithmetic;
  (c) one non-default configuration per task through every route (fused pool, unfused,
      CUDA-core kernels only, the segmenter's reference call signature);
  (d) options outside the library's envelope (node_num > 256, k > 4) raise.

Every case asserts the path it was written for, from the C-ABI calls recorded by ops.PROFILE, so
that a moved threshold cannot silently turn it into a duplicate of the default case. Parity as in
SURVEY.md Appendix C: k-sets and counts exact, fp32 within |a-b| <= 1e-4 * max(|b|, 1), per-copy
tensors in the oracle's slot order, the oracle with ascending slots where nodes are empty."""
import copy

import pytest
import torch

from helpers import (assert_close, assert_golden, build_states, check_encoder_against_golden,
                     golden, golden_case, to_ref_slot_order, to_slot_order)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEYS = ("pc", "sn", "label", "node", "node_knn_I")
HEAD = {"classifier": "classifier", "segmenter": "segmenter", "autoencoder": "decoder"}


def _model(task, opt, st):
    from sonet_b200 import autoencoder, classifier, segmenter
    gopt = copy.copy(opt)
    gopt.device, gopt.gpu_id = torch.device(DEV), 0
    mod = {"classifier": classifier, "segmenter": segmenter, "autoencoder": autoencoder}[task]
    m = mod.Model(gopt)
    m.encoder.load_state_dict(st["encoder"])
    getattr(m, HEAD[task]).load_state_dict(st["head"])
    return m


def _set_input(m, task, inp):
    if task == "segmenter":
        seg = torch.zeros(inp["pc"].shape[0], inp["pc"].shape[2], dtype=torch.int64)
        m.set_input(inp["pc"], inp["sn"], inp["label"], seg, inp["node"], inp["node_knn_I"])
    else:
        m.set_input(*[inp[k] for k in KEYS])


def _run(m, task, inp):
    """set_input + test_model(); returns the C-ABI calls of the forward as [(name, args)]."""
    from sonet_b200 import ops
    _set_input(m, task, inp)
    ops.PROFILE = []
    try:
        m.test_model()
        torch.cuda.synchronize()
        return [(name, args) for name, _, _, args in ops.PROFILE]
    finally:
        ops.PROFILE = None


def _names(calls):
    return {name for name, _ in calls}


def _args(calls, name):
    got = [a for n, a in calls if n == name]
    assert got, "%s was not called" % name
    return got


def _assert_path(calls, must=(), must_not=()):
    names = _names(calls)
    for n in must:
        assert n in names, "expected %s on this path; calls: %s" % (n, sorted(names))
    for n in must_not:
        assert n not in names, "%s must not run on this path" % n


def _layer1_split(calls, G):
    """C0 (point-part channels) of the segmenter's decomposed layer-1 GEMM, the one point-wise
    launch that gathers a per-node addend over G = M groups."""
    got = [a[1] for a in _args(calls, "sonet_pointwise_tc_forward") if a[13] == G]
    assert len(got) == 1, got
    return got[0]


def _group_mode_of_launch(calls):
    """The som_group mode of the recorded sonet_som_group_decenter launch."""
    from sonet_b200 import ops
    (a,) = _args(calls, "sonet_som_group_decenter")
    N, M, k = a[4], a[5], a[6]
    return ops.som_group_mode(N, M, k, a[1] is not None, DEV)


def _last_true(pred, hi=1 << 24):
    """Largest N in [1, hi) with pred(N), pred monotone (True then False)."""
    assert pred(1) and not pred(hi)
    lo = 1
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if pred(mid) else (lo, mid)
    return lo


def _group_limits(M, k, with_sn):
    """(N_s, N_u): the largest N whose som_group launch is staged, and the largest N that
    ops.som_group_fits accepts — from the library's own mode query on this device."""
    from sonet_b200 import ops
    n_s = _last_true(lambda n: ops.som_group_mode(n, M, k, with_sn, DEV) == ops.SOM_GROUP_STAGED)
    n_u = _last_true(lambda n: ops.som_group_fits(n, M, k, DEV))
    return n_s, n_u


def _oracle(oracle_mod, task, opt, st, inp, S, sorted_slots=False):
    sl = {k: v[:S] for k, v in inp.items()}
    o = oracle_mod.encoder_forward(st["encoder"], opt, sl["pc"], sl["sn"], sl["node"],
                                   sl["node_knn_I"], sorted_slots=sorted_slots)
    if task == "classifier":
        o["score"] = oracle_mod.classifier_forward(st["head"], o["feature"])
    elif task == "segmenter":
        o["score_segmenter"] = oracle_mod.segmenter_forward(st["head"], opt, o, sl["pc"], sl["sn"],
                                                            sl["label"])
    return o


def _check_vs_oracle(m, task, opt, o, S):
    """The first S clouds of a CUDA run against the oracle."""
    from oracle import oracle
    enc, k = m.encoder, opt.k
    assert torch.equal(oracle.canon_sets(enc.min_idx[:S].cpu(), k),
                       oracle.canon_sets(o["min_idx"], k))
    mask = enc.mask[:S].cpu()
    assert torch.equal(torch.max(mask, dim=1)[0], o["mask_row_max"])
    assert torch.equal(torch.sum(mask, dim=1), o["mask_row_sum"])
    names = ["som_node", "first_pn_out_masked_max", "final_pn_out", "feature"]
    if opt.som_k >= 2:
        names += ["knn_center_1", "knn_feature_1"]
    for n in names:
        assert_close(getattr(enc, n)[:S], o[n], n)
    for n in ("centers", "x_decentered", "first_pn_out"):
        assert_close(to_slot_order(getattr(enc, n)[:S], enc.min_idx[:S], o["min_idx"], k), o[n], n)
    if task == "classifier":
        assert_close(m.score[:S], o["score"], "score")
    elif task == "segmenter":
        assert_close(m.score_segmenter[:S], o["score_segmenter"], "score_segmenter")


# ---- (a) against the reference's own fixtures at non-default options ---------------------------
@pytest.mark.parametrize("name", ["classifier_b2_n300_m121_k4", "classifier_b3_n150_m16_k1",
                                  "classifier_b1_n700_m256_k2"])
def test_classifier_options_vs_reference_golden(name):
    g = golden(name)
    opt, inp, seed = golden_case(g, "classifier")
    m = _model("classifier", opt, build_states("classifier", opt, seed))
    calls = _run(m, "classifier", inp)
    _assert_path(calls, must=("sonet_pointresnet_tc_pool_forward",))
    if opt.node_num * opt.som_k <= 2304 and opt.som_k >= 2:
        _assert_path(calls, must=("sonet_knn_assemble_pool_f32",))
    check_encoder_against_golden(g, m.encoder, opt)
    assert_golden(g, "score", m.score)


def test_segmenter_options_vs_reference_golden():
    g = golden("segmenter_b2_n200_m100_k2")
    opt, inp, seed = golden_case(g, "segmenter")
    m = _model("segmenter", opt, build_states("segmenter", opt, seed))
    calls = _run(m, "segmenter", inp)
    # the decomposed layer 1: a 9-channel point part (no normals), per-node addend over G=100
    assert _layer1_split(calls, 100) == 9
    enc = m.encoder
    check_encoder_against_golden(g, enc, opt)
    assert_golden(g, "centers", to_ref_slot_order(enc.centers, enc.min_idx, g, opt.k))
    assert_golden(g, "x_decentered", to_ref_slot_order(enc.x_decentered, enc.min_idx, g, opt.k))
    assert_golden(g, "score_segmenter", m.score_segmenter)


def test_autoencoder_conv4096_vs_reference_golden():
    g = golden("autoencoder_b2_n300_m36_conv4096")
    opt, inp, seed = golden_case(g, "autoencoder")
    m = _model("autoencoder", opt, build_states("autoencoder", opt, seed))
    calls = _run(m, "autoencoder", inp)
    assert m.predicted_pc.shape == (2, 3, 256 + 4096)
    assert [a[3] for a in _args(calls, "sonet_chamfer_f32")].count(256 + 4096) == 1
    check_encoder_against_golden(g, m.encoder, opt)
    assert_golden(g, "predicted_pc", m.predicted_pc)
    for n in ("conv_pc4", "conv_pc5", "conv_pc6"):
        assert_golden(g, n, getattr(m.decoder, n))
    for n in ("loss_chamfer", "loss_chamfer_conv4", "loss_chamfer_conv5", "loss"):
        assert_close(getattr(m, n), g[n], n)
    assert_close(m.chamfer_criteria.loss_array, g["loss_array"], "loss_array")


# ---- (b) dispatch boundaries against the oracle ------------------------------------------------
def _classifier_case(oracle_mod, B, N, S, seed, node_mode="sampled", sorted_slots=False, **over):
    from sonet_b200 import synth
    opt = synth.make_opt("classifier", batch_size=B, input_pc_num=N, **over)
    st = build_states("classifier", opt, seed)
    inp = synth.synth_inputs(B, N, opt.node_num, max(opt.som_k, 1), seed=seed, node_mode=node_mode)
    m = _model("classifier", opt, st)
    calls = _run(m, "classifier", inp)
    o = _oracle(oracle_mod, "classifier", opt, st, inp, S, sorted_slots)
    return m, opt, calls, o


@pytest.mark.parametrize("side", ["staged", "unstaged"])
def test_som_group_staging_boundary(oracle_mod, side):
    """M=64, k=3, normals: N = N_s (cloud staged in shared memory) and N_s + 1 (read from global
    memory); B=2, the first cloud against the oracle."""
    from sonet_b200 import ops
    n_s, _ = _group_limits(64, 3, True)
    N = n_s if side == "staged" else n_s + 1
    m, opt, calls, o = _classifier_case(oracle_mod, 2, N, 1, seed=101 + (side == "unstaged"))
    want = ops.SOM_GROUP_STAGED if side == "staged" else ops.SOM_GROUP_UNSTAGED
    _assert_path(calls, must=("sonet_som_group_decenter", "sonet_pointresnet_tc_pool_forward"),
                 must_not=("sonet_som_sort_decenter",))
    assert _group_mode_of_launch(calls) == want
    print("som_group %s at N=%d (N_s=%d)" % (side, N, n_s))
    _check_vs_oracle(m, "classifier", opt, o, 1)


@pytest.mark.parametrize("side", ["group", "sort"])
def test_som_group_fit_boundary(oracle_mod, side):
    """M=64, k=3, normals: N = N_u (the largest som_group takes, unstaged) and N_u + 1 (som_assign
    statistics + som_sort_decenter feed the fused pool); B=1."""
    from sonet_b200 import ops
    _, n_u = _group_limits(64, 3, True)
    N = n_u if side == "group" else n_u + 1
    m, opt, calls, o = _classifier_case(oracle_mod, 1, N, 1, seed=103 + (side == "sort"))
    if side == "group":
        _assert_path(calls, must=("sonet_som_group_decenter",), must_not=("sonet_som_sort_decenter",))
        assert _group_mode_of_launch(calls) == ops.SOM_GROUP_UNSTAGED
    else:
        _assert_path(calls, must=("sonet_som_sort_decenter", "sonet_pointresnet_tc_pool_forward"),
                     must_not=("sonet_som_group_decenter",))
        (a,) = _args(calls, "sonet_som_assign")
        assert a[8] is not None and a[10] is not None, "som_assign must compute the statistics"
    print("%s path at N=%d (N_u=%d)" % (side, N, n_u))
    _check_vs_oracle(m, "classifier", opt, o, 1)


def test_k4_without_normals_unstaged(oracle_mod):
    """k = 4 (the library's limit), surface_normal off, N one past its own staging limit."""
    from sonet_b200 import ops
    n_s, _ = _group_limits(64, 4, False)
    m, opt, calls, o = _classifier_case(oracle_mod, 1, n_s + 1, 1, seed=105, k=4,
                                        surface_normal=False)
    _assert_path(calls, must=("sonet_som_group_decenter", "sonet_pointresnet_tc_pool_forward"))
    (a,) = _args(calls, "sonet_som_group_decenter")
    assert a[1] is None and a[6] == 4
    assert _group_mode_of_launch(calls) == ops.SOM_GROUP_UNSTAGED
    (p,) = _args(calls, "sonet_pointresnet_tc_pool_forward")
    assert p[1] == 3, "Cin of the pool variant without normals"
    _check_vs_oracle(m, "classifier", opt, o, 1)


@pytest.mark.parametrize("som_k", [9, 10])
def test_knn_assemble_pool_limit(oracle_mod, som_k):
    """M=256 (every SOM kernel's limit): M*som_k = 2304 takes knn_assemble_pool, 2560 the
    pool_finalize + knn_assemble fallback."""
    m, opt, calls, o = _classifier_case(oracle_mod, 2, 1000, 2, seed=106 + som_k, node_num=256,
                                        som_k=som_k)
    if som_k * 256 <= 2304:
        _assert_path(calls, must=("sonet_knn_assemble_pool_f32",),
                     must_not=("sonet_pool_finalize", "sonet_knn_assemble_f32"))
    else:
        _assert_path(calls, must=("sonet_pool_finalize", "sonet_knn_assemble_f32"),
                     must_not=("sonet_knn_assemble_pool_f32",))
    _check_vs_oracle(m, "classifier", opt, o, 2)


def test_one_point_per_cloud(oracle_mod):
    """M=16, k=1, som_k=0, B=3, N=1: 15 empty nodes per cloud, a pool tile with one valid row."""
    m, opt, calls, o = _classifier_case(oracle_mod, 3, 1, 3, seed=120, sorted_slots=True,
                                        node_num=16, k=1, som_k=0)
    _assert_path(calls, must=("sonet_pointresnet_tc_pool_forward", "sonet_pool_finalize"))
    assert _args(calls, "sonet_pointresnet_tc_pool_forward")[0][3] == 1
    assert (o["mask_row_max"] == 0).sum(dim=1).tolist() == [15, 15, 15]
    _check_vs_oracle(m, "classifier", opt, o, 3)


@pytest.mark.parametrize("B,N,node_mode", [(2, 40, "uniform"), (1, 1023, "sampled")])
def test_fewer_points_than_nodes_and_odd_n(oracle_mod, B, N, node_mode):
    """N < M (most nodes empty) and N not a multiple of 4, M=64, through the fused path."""
    m, opt, calls, o = _classifier_case(oracle_mod, B, N, B, seed=121 + N, node_mode=node_mode,
                                        sorted_slots=(node_mode == "uniform"))
    _assert_path(calls, must=("sonet_som_group_decenter", "sonet_pointresnet_tc_pool_forward",
                              "sonet_knn_assemble_pool_f32"))
    if N < 64:
        assert int((o["mask_row_max"] == 0).sum()) > 0, "case must contain empty nodes"
    _check_vs_oracle(m, "classifier", opt, o, B)


def test_segmenter_m121_without_normals(oracle_mod):
    """k=3, M=121, normals off, B=3: decomposed layer 1 with a 9-channel point part and G=121."""
    from sonet_b200 import synth
    B, N = 3, 256
    opt = synth.make_opt("segmenter", batch_size=B, input_pc_num=N, node_num=121,
                         surface_normal=False)
    st = build_states("segmenter", opt, 131)
    inp = synth.synth_inputs(B, N, 121, opt.som_k, seed=131)
    m = _model("segmenter", opt, st)
    calls = _run(m, "segmenter", inp)
    assert _layer1_split(calls, 121) == 9
    _check_vs_oracle(m, "segmenter", opt, _oracle(oracle_mod, "segmenter", opt, st, inp, B), B)


def _decoder_fp64(opt, st):
    from sonet_b200 import networks
    cpu_opt = copy.copy(opt)
    cpu_opt.device = torch.device("cpu")
    ref = networks.Decoder(cpu_opt)
    ref.load_state_dict(st["head"])
    return ref.double().eval()          # CPU fp64: every layer takes the PyTorch path


def _check_autoencoder(oracle_mod, m, opt, st, inp, calls):
    pc = inp["pc"]
    with torch.no_grad():
        ref = _decoder_fp64(opt, st)
        want = ref(m.feature.cpu().double()).float()
    assert_close(m.predicted_pc, want, "predicted_pc")
    for n in ("conv_pc4", "conv_pc5", "conv_pc6"):
        assert_close(getattr(m.decoder, n), getattr(ref, n).float(), n)
    ch = {"loss_chamfer": oracle_mod.chamfer(m.predicted_pc.cpu(), pc),
          "loss_chamfer_conv4": oracle_mod.chamfer(m.decoder.conv_pc4.cpu(), pc),
          "loss_chamfer_conv5": oracle_mod.chamfer(m.decoder.conv_pc5.cpu(), pc)}
    for n, o in ch.items():
        assert_close(getattr(m, n), o["loss"], n)
    assert_close(m.loss, sum(o["loss"] for o in ch.values()), "loss")
    assert_close(m.chamfer_criteria.loss_array, ch["loss_chamfer"]["loss_array"], "loss_array")


def test_autoencoder_conv4096_without_fc_branch(oracle_mod):
    """output_fc_pc_num=0, output_conv_pc_num=4096: predicted_pc is conv_pc6 and the Chamfer
    kernels see 4096 predicted points."""
    from sonet_b200 import synth
    B, N = 2, 500
    opt = synth.make_opt("autoencoder", batch_size=B, input_pc_num=N, output_fc_pc_num=0,
                         output_conv_pc_num=4096)
    st = build_states("autoencoder", opt, 141)
    inp = synth.synth_inputs(B, N, seed=141)
    m = _model("autoencoder", opt, st)
    calls = _run(m, "autoencoder", inp)
    assert not hasattr(m.decoder, "fc_decoder")
    assert m.predicted_pc.shape == (B, 3, 4096)
    assert torch.equal(m.predicted_pc, m.decoder.conv_pc6)
    assert sorted(a[3] for a in _args(calls, "sonet_chamfer_f32")) == [256, 1024, 4096]
    _check_vs_oracle(m, "autoencoder", opt, _oracle(oracle_mod, "autoencoder", opt, st, inp, B), B)
    _check_autoencoder(oracle_mod, m, opt, st, inp, calls)


# ---- (c) one non-default configuration per task through every route ---------------------------
ROUTE_OPTS = {"classifier": dict(node_num=100, k=2, som_k=5, som_k_type="center",
                                 surface_normal=False),
              "segmenter": dict(node_num=100, k=2, som_k=9, som_k_type="avg",
                                surface_normal=False),
              "autoencoder": dict(node_num=36, k=4, som_k=5, output_conv_pc_num=4096)}
ROUTES = [(t, r) for t in ROUTE_OPTS for r in ("fused", "unfused", "cuda_core")] + \
    [("segmenter", "reference_signature")]


@pytest.mark.parametrize("task,route", ROUTES)
def test_every_route_vs_oracle(oracle_mod, monkeypatch, task, route):
    from sonet_b200 import synth
    B, N = 2, 333
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, **ROUTE_OPTS[task])
    st = build_states(task, opt, 151)
    inp = synth.synth_inputs(B, N, opt.node_num, opt.som_k, seed=151)
    if route == "cuda_core":
        monkeypatch.setenv("SONET_TC", "0")
    m = _model(task, opt, st)
    if route != "cuda_core":         # SONET_TC=0 must leave the fused pool on its own
        m.encoder.fuse_pool = route == "fused"
    calls = _run(m, task, inp)
    names = _names(calls)
    if route == "fused":
        _assert_path(calls, must=("sonet_som_group_decenter", "sonet_pointresnet_tc_pool_forward"))
    elif route in ("unfused", "reference_signature"):
        _assert_path(calls, must=("sonet_pointresnet_tc_forward", "sonet_index_max_f32"),
                     must_not=("sonet_pointresnet_tc_pool_forward",))
    else:
        assert not [n for n in names if "_tc_" in n], sorted(names)
        _assert_path(calls, must=("sonet_pointwise_layer_f32", "sonet_index_max_f32"))
    o = _oracle(oracle_mod, task, opt, st, inp, B)
    if route == "reference_signature":
        enc = m.encoder
        with torch.no_grad():
            kN = enc.min_idx.shape[1]
            idx = torch.max(enc.mask, dim=2)[1].unsqueeze(1)
            gat = lambda t: torch.gather(t, 2, idx.expand(B, t.shape[1], kN))  # noqa: E731
            s2 = m.segmenter(enc.x_decentered, m.pc, enc.centers, m.sn, m.input_label,
                             enc.first_pn_out, gat(enc.first_pn_out_masked_max),
                             gat(enc.knn_feature_1), gat(enc.final_pn_out), m.feature)
        assert_close(s2, o["score_segmenter"], "Segmenter.forward vs oracle")
        assert_close(s2, m.score_segmenter, "Segmenter.forward vs forward_nodes")
    _check_vs_oracle(m, task, opt, o, B)
    if task == "autoencoder":
        _check_autoencoder(oracle_mod, m, opt, st, inp, calls)


# ---- (d) outside the envelope -------------------------------------------------------------------
@pytest.mark.parametrize("task", ["classifier", "segmenter", "autoencoder"])
@pytest.mark.parametrize("over,limit", [(dict(node_num=289), r"M=289 out of range \[1,256\]"),
                                        (dict(k=5), r"k=5 out of range \[1,4\]")])
def test_options_beyond_the_limits_raise(task, over, limit):
    """The reference's scripts also run node_num = 289 (17x17) and k = 5; this library stops at
    M = 256 and k = 4 and must say so instead of returning numbers."""
    from sonet_b200 import synth
    B, N = 2, 400
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N, **over)
    st = build_states(task, opt, 161)
    inp = synth.synth_inputs(B, N, opt.node_num, opt.som_k, seed=161)
    m = _model(task, opt, st)
    with pytest.raises(RuntimeError, match=limit):
        _run(m, task, inp)
