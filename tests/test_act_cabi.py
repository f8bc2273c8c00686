"""C-ABI of the activation codes (SONET_ACT_NONE / _RELU / _ELU), without a GPU: every layer entry
with an activation argument rejects an unknown code with a negative status and a message before any
CUDA call, and the explicit-activation entries of the fused kernels are exported and bound. The
train-mode BatchNorm entries' check is test_dp_train_host.test_rejects_unknown_activation."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ACT_ENTRIES = ("sonet_pointresnet_tc_forward_act", "sonet_pointresnet_tc_pool_forward_act",
               "sonet_knn_mlp_tc_forward_act")


def _calls(lib, act):
    """Each layer entry with an activation argument, called with `act` and otherwise plausible
    arguments (null pointers: the activation check must come first)."""
    n = None
    return {
        "sonet_pointwise_layer_f32": lambda: lib.sonet_pointwise_layer_f32(
            n, 8, n, 0, 2, 64, n, n, n, 16, act, n, n, 0, n, n),
        "sonet_linear_f32": lambda: lib.sonet_linear_f32(n, 2, 16, n, n, n, 8, act, n, n),
        "sonet_pointwise_tc_forward": lambda: lib.sonet_pointwise_tc_forward(
            n, 64, n, 0, 2, 256, n, 1.0, n, 64, act, n, n, 0, n, n),
        "sonet_pointwise_tc_forward_f16": lambda: lib.sonet_pointwise_tc_forward_f16(
            n, 64, n, 0, 2, 256, n, 1.0, n, 64, act, n, n, 0, n, n),
        "sonet_pointwise_tc_forward_rows": lambda: lib.sonet_pointwise_tc_forward_rows(
            n, 64, n, 0, 2, 256, n, 1.0, n, 64, act, n, n, 0, n, n),
        "sonet_pointwise_tc_forward_rows_f16": lambda: lib.sonet_pointwise_tc_forward_rows_f16(
            n, 64, n, 0, 2, 256, n, 1.0, n, 64, act, n, n, 0, n, n),
        "sonet_pointwise_tc_grouped_forward": lambda: lib.sonet_pointwise_tc_grouped_forward(
            n, 64, 2, 64, n, 0, 1.0, n, 64, act, 1, 1, 0, 0, 64, 0, n, n, n),
        "sonet_pointwise_tc_grouped_forward_f16": lambda: lib.sonet_pointwise_tc_grouped_forward_f16(
            n, 64, 2, 64, n, 0, 1.0, n, 64, act, 1, 1, 0, 0, 64, 0, n, n, n),
        "sonet_pointwise_tc_forward_dev": lambda: lib.sonet_pointwise_tc_forward_dev(
            n, 64, 2, 64, n, n, n, n, 64, act, 1, n, n, n),
        "sonet_pointresnet_tc_forward_act": lambda: lib.sonet_pointresnet_tc_forward_act(
            n, 6, 2, 256, n, n, act, 0, n, n),
        "sonet_pointresnet_tc_pool_forward_act": lambda: lib.sonet_pointresnet_tc_pool_forward_act(
            n, 6, 2, 256, n, n, n, n, 64, act, 0, n, n, n),
        "sonet_knn_mlp_tc_forward_act": lambda: lib.sonet_knn_mlp_tc_forward_act(
            n, n, n, 2, 64, 9, 9, n, 1, 512, n, n, 1.0, n, act, 0, n, n),
    }


@pytest.mark.parametrize("act", [3, -1])
def test_layer_entries_reject_unknown_activation_codes(lib_built, act):
    from sonet_b200 import _C
    lib = _C.lib()
    for name, call in _calls(lib, act).items():
        rc = call()
        assert rc < 0, "%s accepted activation code %d" % (name, act)
        msg = _C.last_error()
        assert "activation code %d" % act in msg, "%s: %r" % (name, msg)


def test_fused_act_entries_take_relu_or_elu_only(lib_built):
    """The fused kernels have no 'no activation' build: SONET_ACT_NONE is refused with a message."""
    from sonet_b200 import _C
    lib = _C.lib()
    for name, call in _calls(lib, 0).items():
        if name in ACT_ENTRIES:
            assert call() < 0 and "activation code 0" in _C.last_error(), name


def test_act_entries_exported_and_declared(lib_built):
    from sonet_b200 import _C
    h = ctypes.CDLL(lib_built)
    text = open(os.path.join(ROOT, "include", "sonet_b200.h")).read()
    for n in ACT_ENTRIES:
        assert hasattr(h, n), "library does not export %s" % n
        assert re.search(r"\b%s\s*\(" % n, text), "%s is not declared" % n
    assert tuple(_C.ACT_ENTRIES) == ACT_ENTRIES
    for code, name in ((0, "NONE"), (1, "RELU"), (2, "ELU")):
        assert re.search(r"#define SONET_ACT_%s %d\b" % (name, code), text)


def test_python_activation_codes():
    from sonet_b200 import layers, ops
    assert [ops.act_code(a) for a in (None, "relu", "elu", False, True, 2)] == [0, 1, 2, 0, 1, 2]
    with pytest.raises(RuntimeError, match="swish"):
        ops.act_code("swish")
    assert layers.KERNEL_ACTIVATIONS == (None, "relu", "elu")


@pytest.mark.parametrize("activation,fast", [("relu", True), ("elu", True), (None, True),
                                             ("swish", False), ("leakyrelu", False)])
def test_layer_eligibility_by_activation(activation, fast):
    """relu, elu and no activation are kernel epilogues; swish and leakyrelu stay PyTorch."""
    from sonet_b200 import layers
    lay = layers.EquivariantLayer(8, 16, activation=activation, normalization="batch")
    assert lay._fast_eligible() == fast
    lin = layers.MyLinear(8, 16, activation=activation, normalization="batch")
    assert (lin.activation in layers.KERNEL_ACTIVATIONS) == fast
    up = layers.UpConv(16, 64, activation=activation, normalization="batch")
    assert (up.activation in layers.KERNEL_ACTIVATIONS) == fast
