import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "so-net_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def lib_built():
    """libsonet_b200.so must exist (built by __graft_entry__.build()); build it if stale."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("sonet_build", os.path.join(ROOT, "so-net_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    if not os.path.exists(mod.LIB):
        mod.build()
    return mod.LIB


@pytest.fixture(scope="session")
def oracle_mod():
    from oracle import build as obuild
    obuild.build_c()
    from oracle import oracle
    return oracle
