"""Shared test helpers: golden loading, model construction with the seeded synthetic weights."""
import os

import numpy as np
import torch

from sonet_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

# parity tolerance for floating-point tensors (BASELINE.json north_star: fp32 within 1e-4 rel):
#   |a - b| <= TOL * max(|b|, 1)
TOL = 1e-4


def golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)


def rel_err(a, b):
    a = torch.as_tensor(a, dtype=torch.float32).cpu()
    b = torch.as_tensor(b, dtype=torch.float32).cpu()
    return float(((a - b).abs() / b.abs().clamp(min=1.0)).max())


def assert_close(a, b, what, tol=TOL):
    e = rel_err(a, b)
    assert e <= tol, "%s: max |a-b|/max(|b|,1) = %.3e > %.1e" % (what, e, tol)


def sampled(g, name, t):
    """Compare-ready view of tensor t at the positions a golden strided sample was taken."""
    stride = int(g[name + "__stride"])
    assert tuple(g[name + "__shape"]) == tuple(t.shape), (name, tuple(g[name + "__shape"]), tuple(t.shape))
    return t.detach().cpu().contiguous().view(-1)[::stride]


def assert_golden(g, name, t, tol=TOL):
    assert_close(sampled(g, name, t), torch.from_numpy(g[name]), "golden " + name, tol)


def build_states(task, opt, seed):
    """State dicts (CPU tensors) for encoder and head, keyed like the reference's."""
    from sonet_b200 import networks
    cpu_opt = synth.make_opt(task, **{k: v for k, v in vars(opt).items()
                                      if k not in ("device",)})
    cpu_opt.device = torch.device("cpu")
    enc = networks.Encoder(cpu_opt)
    st = dict(encoder=synth.synth_state_dict(enc, seed=seed))
    if task == "classifier":
        st["head"] = synth.synth_state_dict(networks.Classifier(cpu_opt), seed=seed + 1)
    elif task == "segmenter":
        st["head"] = synth.synth_state_dict(networks.Segmenter(cpu_opt), seed=seed + 1)
    elif task == "autoencoder":
        st["head"] = synth.synth_state_dict(networks.Decoder(cpu_opt), seed=seed + 1)
    return st


def golden_options(g):
    """The non-default options a fixture was generated with (oracle/make_golden.py stores each
    one as opt_<name>)."""
    return {key[4:]: g[key].item() for key in g.files if key.startswith("opt_")}


def golden_case(g, task, **over):
    B, N, seed = int(g["B"]), int(g["N"]), int(g["seed"])
    som_k = int(g["som_k"])
    kw = dict(batch_size=B, input_pc_num=N, som_k=som_k)
    kw.update(golden_options(g))
    kw.update(over)
    opt = synth.make_opt(task, **kw)
    inp = synth.synth_inputs(B, N, opt.node_num, max(som_k, 1), seed=seed,
                             node_mode=str(g["node_mode"]))
    return opt, inp, seed


def check_encoder_against_golden(g, enc, opt):
    """Every cached encoder attribute of a CUDA run against a reference fixture: k-sets and mask
    statistics exact, node-level tensors and (in the reference's slot order) first_pn_out within
    TOL."""
    from oracle import oracle
    assert np.array_equal(oracle.canon_sets(enc.min_idx.cpu(), opt.k).numpy(), g["knn_sets"])
    mask = enc.mask
    assert mask.dtype == torch.int32
    assert np.array_equal(torch.max(mask, dim=1)[0].cpu().numpy(), g["mask_row_max"])
    assert np.array_equal(torch.sum(mask, dim=1).cpu().numpy(), g["mask_row_sum"])
    for n in ("som_node", "first_pn_out_masked_max", "final_pn_out", "feature"):
        assert_golden(g, n, getattr(enc, n))
    assert_golden(g, "first_pn_out", to_ref_slot_order(enc.first_pn_out, enc.min_idx, g, opt.k))
    if opt.som_k >= 2:
        assert_golden(g, "knn_center_1", enc.knn_center_1)
        assert_golden(g, "knn_feature_1", enc.knn_feature_1)


def to_ref_slot_order(t, our_min_idx, g, k):
    return to_slot_order(t, our_min_idx, torch.from_numpy(g["min_idx_ref"].astype(np.int64)), k)


def to_slot_order(t, our_min_idx, ref, k):
    """Reorder the k stacked copies of a [B,C,kN] tensor from OUR slot order (ascending distance)
    to the slot order the reference run used (its topk(sorted=False) order is implementation
    defined; parity for the assignment is per-point set equality — SURVEY.md Appendix C)."""
    ref = ref.detach().cpu().long()                                     # [B,kN]
    ours = our_min_idx.detach().cpu().long()
    B, kN = ours.shape
    N = kN // k
    ours_k = ours.view(B, k, N)
    ref_k = ref.view(B, k, N)
    # src_slot[b, s, n] = our slot holding the node the reference has in slot s
    match = ref_k.unsqueeze(2) == ours_k.unsqueeze(1)                   # [B, k_ref, k_ours, N]
    assert bool(match.any(dim=2).all()), "assignment sets differ"
    src_slot = match.float().argmax(dim=2)                              # [B,k,N]
    src = (src_slot * N + torch.arange(N).view(1, 1, N)).view(B, kN)
    tc = t.detach().cpu()
    return torch.gather(tc, 2, src.unsqueeze(1).expand(B, tc.shape[1], kN))
