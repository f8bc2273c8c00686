"""C-ABI and dispatch of instance normalization, without a GPU: sonet_instance_norm_f32 is exported
and declared, and it rejects P < 2, an unknown activation or reduction code and a copy count or
group size that does not divide P with a negative status and a message before any CUDA call; the
layers route instance norm to the kernels except in MyLinear, where the reference raises."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "sonet_instance_norm_f32"


def _call(lib, P=16, act=1, reduce=0, k=1, out=None, B=2, C=8):
    """Null tensors: only the argument checks can run, and they must come first."""
    n = None
    return lib.sonet_instance_norm_f32(n, n, n, B, C, P, 1e-5, act, reduce, k, out, n, n, n)


def test_instance_norm_exported_and_declared(lib_built):
    from sonet_b200 import _C
    h = ctypes.CDLL(lib_built)
    assert hasattr(h, NAME), "library does not export %s" % NAME
    text = open(os.path.join(ROOT, "include", "sonet_b200.h")).read()
    assert re.search(r"\b%s\s*\(" % NAME, text)
    for code, name in ((0, "NONE"), (1, "KCOPY_MEAN"), (2, "GROUP_MAX")):
        assert re.search(r"#define SONET_REDUCE_%s %d\b" % (name, code), text)
    assert NAME in _C.EXPORTED_SYMBOLS


@pytest.mark.parametrize("P", [1, 0, -3])
def test_rejects_fewer_than_two_spatial_elements(lib_built, P):
    from sonet_b200 import _C
    assert _call(_C.lib(), P=P) < 0
    assert "Expected more than 1 spatial element" in _C.last_error()


@pytest.mark.parametrize("act", [3, -1])
def test_rejects_unknown_activation(lib_built, act):
    from sonet_b200 import _C
    assert _call(_C.lib(), act=act) < 0
    assert "activation code %d" % act in _C.last_error()


@pytest.mark.parametrize("reduce", [3, -1])
def test_rejects_unknown_reduction(lib_built, reduce):
    from sonet_b200 import _C
    assert _call(_C.lib(), reduce=reduce) < 0
    assert "reduction code %d" % reduce in _C.last_error()


@pytest.mark.parametrize("reduce,k,what", [(1, 3, "copy count"), (2, 5, "group size"),
                                           (1, 0, "copy count"), (2, -2, "group size")])
def test_rejects_non_dividing_k(lib_built, reduce, k, what):
    from sonet_b200 import _C
    assert _call(_C.lib(), P=16, reduce=reduce, k=k) < 0
    msg = _C.last_error()
    assert "not divisible" in msg and what in msg, msg


def test_rejects_null_and_aliased_reduction(lib_built):
    from sonet_b200 import _C
    lib = _C.lib()
    assert _call(lib) < 0 and "null pointer" in _C.last_error()
    buf = (ctypes.c_float * 64)()
    z = ctypes.addressof(buf)
    rc = lib.sonet_instance_norm_f32(z, None, None, 2, 2, 16, 1e-5, 1, 1, 2, z, None, None, None)
    assert rc < 0 and "alias" in _C.last_error()
    rc = lib.sonet_instance_norm_f32(z, None, None, 2, 2, 16, 1e-5, 1, 0, 1, z, z, None, None)
    assert rc < 0 and "together" in _C.last_error()


def test_kernel_normalizations_and_layer_routing():
    """batch and instance run on the kernels; MyLinear keeps instance on PyTorch; an instance norm
    with running statistics (eval would use them) stays PyTorch."""
    import torch
    from sonet_b200 import layers
    assert layers.KERNEL_NORMALIZATIONS == (None, "batch", "instance")
    for norm in (None, "batch", "instance"):
        assert layers.EquivariantLayer(8, 16, "relu", norm)._fast_eligible()
        assert layers.MyConv2d(8, 16, 1, activation="elu", normalization=norm)._fast_eligible()
    assert not layers.MyConv2d(8, 16, 3, padding=1, normalization="instance")._fast_eligible()
    lay = layers.EquivariantLayer(8, 16, "relu", "instance")
    lay.norm = torch.nn.InstanceNorm1d(16, affine=True, track_running_stats=True)
    assert not lay._fast_eligible()
    up = layers.UpConv(16, 64, activation="relu", normalization="instance")
    assert layers._norm_on_kernels(up.normalization, up.conv.norm)


def test_mylinear_instance_still_raises_like_the_reference():
    import torch
    from sonet_b200 import layers
    lin = layers.MyLinear(512, 256, activation="relu", normalization="instance").eval()
    with pytest.raises(ValueError, match="num_features"):
        lin(torch.randn(4, 512))


def test_forward_points_reductions_are_instance_only():
    import torch
    from sonet_b200 import layers
    lay = layers.EquivariantLayer(8, 16, "relu", "batch")
    with pytest.raises(RuntimeError, match="instance norm only"):
        lay.forward_points(torch.zeros(1, 8, 4), kcopy=2)
