"""How close the tensor-core path is to exact arithmetic, measured against an fp64 evaluation.

The parity bar (1e-4 relative, BASELINE.json north_star) is stated against the reference's fp32
results, which themselves carry rounding noise. These tests evaluate the same network in float64
(the oracle's value path follows the input dtype; index decisions stay fp32, oracle/oracle.py) and
compare BOTH the reference-equivalent fp32 CPU evaluation and the CUDA path with it: the CUDA
path's distance to the fp64 result must be of the same order as fp32's own — i.e. the fp16 hi/lo
split of the wgmma layers (csrc/tc_common.cuh) costs no more accuracy than plain fp32 arithmetic does,
also through the deepest chain the hot path has (segmenter: 13 chained layers).
"""
import pytest
import torch

from helpers import build_states
from sonet_b200 import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _err(a, ref):
    a = a.detach().double().cpu()
    ref = ref.double()
    return float(((a - ref).abs() / ref.abs().clamp(min=1.0)).max())


def _f64(st):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in st.items()}


def _gpu_opt(opt):
    opt.device = torch.device(DEV)
    opt.gpu_id = 0
    return opt


@pytest.mark.parametrize("task,B,N", [("classifier", 4, 5000), ("segmenter", 4, 1024)])
def test_cuda_path_error_vs_fp64_is_of_fp32_order(oracle_mod, task, B, N):
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N)
    st = build_states(task, opt, seed=77)
    inp = synth.synth_inputs(B, N, seed=77)
    cpu_opt = synth.make_opt(task, batch_size=B, input_pc_num=N)

    def cpu_eval(dt):
        enc_st = st["encoder"] if dt == torch.float32 else _f64(st["encoder"])
        head_st = st["head"] if dt == torch.float32 else _f64(st["head"])
        pc, sn, node = inp["pc"].to(dt), inp["sn"].to(dt), inp["node"].to(dt)
        o = oracle_mod.encoder_forward(enc_st, cpu_opt, pc, sn, node, inp["node_knn_I"])
        if task == "classifier":
            return oracle_mod.classifier_forward(head_st, o["feature"])
        return oracle_mod.segmenter_forward(head_st, cpu_opt, o, pc, sn, inp["label"])

    ref64 = cpu_eval(torch.float64)
    ref32 = cpu_eval(torch.float32)

    if task == "classifier":
        from sonet_b200 import classifier
        m = classifier.Model(_gpu_opt(opt))
        m.encoder.load_state_dict(st["encoder"])
        m.classifier.load_state_dict(st["head"])
        m.set_input(inp["pc"], inp["sn"], inp["label"], inp["node"], inp["node_knn_I"])
        m.test_model()
        ours = m.score
    else:
        from sonet_b200 import segmenter
        m = segmenter.Model(_gpu_opt(opt))
        m.encoder.load_state_dict(st["encoder"])
        m.segmenter.load_state_dict(st["head"])
        seg = torch.zeros(B, N, dtype=torch.int64)
        m.set_input(inp["pc"], inp["sn"], inp["label"], seg, inp["node"], inp["node_knn_I"])
        m.test_model()
        ours = m.score_segmenter

    e32 = _err(ref32, ref64)
    e_ours = _err(ours, ref64)
    e_par = _err(ours, ref32)
    print("\n[precision] %s B=%d N=%d: fp32 CPU vs fp64 %.2e | CUDA path vs fp64 %.2e | CUDA vs fp32 CPU %.2e"
          % (task, B, N, e32, e_ours, e_par))
    assert e_par <= 1e-4                       # the parity bar
    # same order as fp32's own rounding noise: a generous factor, with an absolute floor for
    # cases where the CPU result happens to be unusually close to fp64
    assert e_ours <= max(8.0 * e32, 2e-5), (e_ours, e32)


def _rel_to_max(a, ref):
    """max |a - ref| / max |ref| over the whole tensor (no unit floor)."""
    a = a.detach().double().cpu()
    ref = ref.double()
    return float((a - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("task,B,N", [("classifier", 4, 2048), ("segmenter", 2, 1024),
                                      ("autoencoder", 2, 1024)])
def test_trained_like_weights_error_vs_fp64_is_of_fp32_order(oracle_mod, task, B, N):
    """BatchNorm statistics spread like a trained network's (helpers.trained_like_state_dict):
    folded weight rows span many decades within one matrix, activations of single channels sit far
    below or above unit scale. Measured relative to each output tensor's maximum, with no floor:
    the CUDA path must meet the 1e-4 parity bar wherever fp32 CPU does, and stay of fp32's order."""
    from helpers import trained_like_state_dict
    from sonet_b200 import networks
    opt = synth.make_opt(task, batch_size=B, input_pc_num=N)
    st = build_states(task, opt, seed=91, make=trained_like_state_dict)
    inp = synth.synth_inputs(B, N, seed=91)
    cpu_opt = synth.make_opt(task, batch_size=B, input_pc_num=N)
    if task == "autoencoder":
        dec = networks.Decoder(cpu_opt)
        dec.load_state_dict(st["head"])
        dec.eval()

    def cpu_eval(dt):
        enc_st = st["encoder"] if dt == torch.float32 else _f64(st["encoder"])
        head_st = st["head"] if dt == torch.float32 else _f64(st["head"])
        pc, sn, node = inp["pc"].to(dt), inp["sn"].to(dt), inp["node"].to(dt)
        o = oracle_mod.encoder_forward(enc_st, cpu_opt, pc, sn, node, inp["node_knn_I"])
        if task == "classifier":
            return oracle_mod.classifier_forward(head_st, o["feature"])
        if task == "segmenter":
            return oracle_mod.segmenter_forward(head_st, cpu_opt, o, pc, sn, inp["label"])
        with torch.no_grad():
            return dec.to(dt)(o["feature"])

    ref64 = cpu_eval(torch.float64)
    ref32 = cpu_eval(torch.float32)
    keys = ("pc", "sn", "label", "node", "node_knn_I")
    if task == "classifier":
        from sonet_b200 import classifier
        m = classifier.Model(_gpu_opt(opt))
        m.classifier.load_state_dict(st["head"])
        m.set_input(*[inp[k] for k in keys])
    elif task == "segmenter":
        from sonet_b200 import segmenter
        m = segmenter.Model(_gpu_opt(opt))
        m.segmenter.load_state_dict(st["head"])
        m.set_input(inp["pc"], inp["sn"], inp["label"], torch.zeros(B, N, dtype=torch.int64),
                    inp["node"], inp["node_knn_I"])
    else:
        from sonet_b200 import autoencoder
        m = autoencoder.Model(_gpu_opt(opt))
        m.decoder.load_state_dict(st["head"])
        m.set_input(*[inp[k] for k in keys])
    m.encoder.load_state_dict(st["encoder"])
    m.test_model()
    ours = {"classifier": lambda: m.score, "segmenter": lambda: m.score_segmenter,
            "autoencoder": lambda: m.predicted_pc}[task]()

    e32 = _rel_to_max(ref32, ref64)
    e_ours = _rel_to_max(ours, ref64)
    e_par = _rel_to_max(ours, ref32)
    print("\n[precision] trained-like %s B=%d N=%d: fp32 CPU vs fp64 %.2e | CUDA path vs fp64 %.2e | "
          "CUDA vs fp32 CPU %.2e" % (task, B, N, e32, e_ours, e_par))
    assert bool(torch.isfinite(ours).all())
    if e32 <= 1e-5:
        assert e_par <= 1e-4
    assert e_ours <= max(8.0 * e32, 2e-5), (e_ours, e32)
