"""The pybind11/ATen binding of INTEGRATION.md §3 (so-net_b200/bindings/index_max_pybind.cpp)
compiles against libsonet_b200.so with torch.utils.cpp_extension and behaves like the reference's
own plugin: same module surface; the host entry points are checked against the golden vectors the
reference BINARY produced, the CUDA entry point on the GPU box."""
import os

import numpy as np
import pytest
import torch

from helpers import golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def plugin(lib_built):
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils.cpp_extension import load
    libdir = os.path.dirname(lib_built)
    build_dir = os.path.join(ROOT, "so-net_b200", "build", "pybind_index_max")
    os.makedirs(build_dir, exist_ok=True)
    return load(name="index_max_sonet_b200",
                sources=[os.path.join(ROOT, "so-net_b200", "bindings", "index_max_pybind.cpp")],
                extra_include_paths=[os.path.join(ROOT, "include")],
                extra_ldflags=["-L" + libdir, "-lsonet_b200", "-Wl,-rpath," + libdir],
                build_directory=build_dir, with_cuda=True, verbose=False)


def test_binding_surface_and_host_path_vs_reference_binary_goldens(plugin):
    for name in ("forward_cpu", "forward_multi_thread_cpu", "forward_cuda", "forward_cuda_shared_mem"):
        assert callable(getattr(plugin, name))           # models/index_max_ext/index_max.cpp:154-159
    g = golden("index_max")
    out = plugin.forward_cpu(torch.from_numpy(g["kat_data"]), torch.from_numpy(g["kat_index"]), 5)
    assert out.dtype == torch.int32 and out.tolist() == [[[0, 1, 0, 4, 0]]]
    for tag in ("a", "b"):
        d, i = torch.from_numpy(g[tag + "_data"]), torch.from_numpy(g[tag + "_index"])
        assert np.array_equal(plugin.forward_cpu(d, i, int(g[tag + "_K"])).numpy(), g[tag + "_out"])
        assert np.array_equal(plugin.forward_multi_thread_cpu(d, i, int(g[tag + "_K"]), 3).numpy(),
                              g[tag + "_out"])
    with pytest.raises(RuntimeError):                    # CHECK_INPUT behaviour (index_max.cpp:119-121)
        plugin.forward_cuda(torch.from_numpy(g["a_data"]), torch.from_numpy(g["a_index"]), 4)


@pytest.mark.gpu
def test_binding_cuda_entry_vs_goldens(plugin):
    g = golden("index_max")
    for tag in ("a", "b"):
        d, i = torch.from_numpy(g[tag + "_data"]).cuda(), torch.from_numpy(g[tag + "_index"]).cuda()
        for fn in (plugin.forward_cuda, plugin.forward_cuda_shared_mem):
            assert np.array_equal(fn(d, i, int(g[tag + "_K"])).cpu().numpy(), g[tag + "_out"])
