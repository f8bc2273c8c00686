"""Host-side logic that needs no GPU: module API / state_dict parity with the reference,
BN folding arithmetic, synthetic generators, shard arithmetic."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import GOLDEN
from sonet_b200 import dist as sdist
from sonet_b200 import layers, networks, synth


@pytest.mark.parametrize("task,som_k,head", [("classifier", 9, "classifier"),
                                             ("classifier", 0, "classifier"),
                                             ("segmenter", 9, "segmenter"),
                                             ("autoencoder", 9, "decoder")])
def test_state_dict_keys_and_shapes_match_reference(task, som_k, head):
    _check_state_keys(task, som_k, True, head)


@pytest.mark.parametrize("task,som_k,sn,head", [("classifier", 1, True, "classifier"),
                                                ("segmenter", 1, True, "segmenter"),
                                                ("classifier", 9, False, "classifier"),
                                                ("segmenter", 9, False, "segmenter"),
                                                ("autoencoder", 9, False, "decoder")])
def test_state_dict_keys_match_reference_at_other_options(task, som_k, sn, head):
    """som_k=1 (the PointResNet final network, no KNN module) and surface_normal=False (3-channel
    first PointResNet, 9-channel segmenter point part): checkpoints of those networks load too."""
    _check_state_keys(task, som_k, sn, head)


def _check_state_keys(task, som_k, sn, head):
    want = json.load(open(os.path.join(GOLDEN, "state_keys.json")))
    opt = synth.make_opt(task, batch_size=2, input_pc_num=64, som_k=som_k, surface_normal=sn)
    mods = {"encoder": networks.Encoder(opt),
            head: getattr(networks, head.capitalize())(opt)}
    for name, m in mods.items():
        ref = want["%s/som_k=%d%s/%s" % (task, som_k, "" if sn else "/no_sn", name)]
        got = {k: list(v.shape) for k, v in m.state_dict().items()}
        assert got == ref, name


def test_bn_folding_matches_eval_batchnorm():
    torch.manual_seed(0)
    layer = layers.EquivariantLayer(7, 5, 'relu', 'batch')
    layer.load_state_dict(synth.synth_state_dict(layer, seed=3))
    layer.eval()
    wt, shift = layer.folded(transpose=True)
    assert wt.shape == (7, 5)
    x = torch.randn(2, 7, 11)
    with torch.no_grad():
        want = layer(x)                                     # PyTorch path on CPU tensors
        got = F.relu(torch.einsum("kc,bkp->bcp", wt, x) + shift[None, :, None])
    assert torch.allclose(got, want, atol=1e-5, rtol=1e-5)
    # re-packs when a parameter changes in place
    with torch.no_grad():
        layer.norm.running_mean.add_(1.0)
    wt2, shift2 = layer.folded(transpose=True)
    assert not torch.equal(shift, shift2)


def test_cpu_tensors_take_the_pytorch_path_and_encoder_refuses_cpu():
    opt = synth.make_opt("classifier", batch_size=2, input_pc_num=32)
    enc = networks.Encoder(opt).eval()
    inp = synth.synth_inputs(2, 32)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        enc(inp["pc"], inp["sn"], inp["node"], inp["node_knn_I"])
    cls = networks.Classifier(opt).eval()
    with torch.no_grad():
        assert cls(torch.randn(2, 1024)).shape == (2, 40)    # plain nn.Linear path on CPU


def test_synth_is_deterministic_and_well_formed():
    a, b = synth.synth_inputs(3, 100, seed=5), synth.synth_inputs(3, 100, seed=5)
    for k in a:
        assert torch.equal(a[k], b[k])
    assert torch.allclose((a["sn"] ** 2).sum(1), torch.ones(3, 100), atol=1e-5)
    assert torch.equal(a["node_knn_I"][:, :, 0], torch.arange(64).expand(3, 64))  # self first
    assert a["node_knn_I"].dtype == torch.int64 and a["node_knn_I"].shape == (3, 64, 9)


def test_shard_bounds_cover_batch():
    for total in (0, 1, 7, 64, 512):
        for world in (1, 2, 4, 8):
            spans = [sdist.shard_bounds(total, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == total
            assert all(spans[i][1] == spans[i + 1][0] for i in range(world - 1))
            sizes = [hi - lo for lo, hi in spans]
            assert max(sizes) - min(sizes) <= 1
