"""The opt-in fp16 mode without a GPU: SONET_TC parsing, and the six `_f16` C-ABI entries declared
in include/sonet_b200.h, bound in _C.py with their split twins' signatures and exported."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPLIT_ENTRIES = ("sonet_pointresnet_tc_forward", "sonet_pointresnet_tc_pool_forward",
                 "sonet_pointwise_tc_forward", "sonet_pointwise_tc_forward_rows",
                 "sonet_pointwise_tc_grouped_forward", "sonet_knn_mlp_tc_forward")
F16_ENTRIES = tuple(n + "_f16" for n in SPLIT_ENTRIES)


@pytest.mark.parametrize("value,mode", [(None, "split"), ("1", "split"), ("0", "fp32"),
                                        ("fp16", "fp16"), ("bf16", "split"), ("", "split"),
                                        ("FP16", "split")])
def test_tc_mode_parsing(monkeypatch, value, mode):
    from sonet_b200 import layers
    if value is None:
        monkeypatch.delenv("SONET_TC", raising=False)
    else:
        monkeypatch.setenv("SONET_TC", value)
    assert layers.tc_mode() == mode
    assert layers.tc_enabled() == (mode != "fp32")
    assert layers.tc_f16() == (mode == "fp16")


def test_tc_mode_is_read_at_call_time(monkeypatch):
    from sonet_b200 import layers
    monkeypatch.setenv("SONET_TC", "fp16")
    assert layers.tc_mode() == "fp16"
    monkeypatch.setenv("SONET_TC", "0")
    assert layers.tc_mode() == "fp32"


def _prototypes():
    text = open(os.path.join(ROOT, "include", "sonet_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    return {n: " ".join(p.split()) for n, p in
            re.findall(r"\b(sonet_\w+)\s*\(([^;{]*?)\)\s*;", text, flags=re.S)}


def test_f16_entries_declared_with_the_split_signatures():
    protos = _prototypes()
    for split, f16 in zip(SPLIT_ENTRIES, F16_ENTRIES):
        assert f16 in protos, f16
        assert protos[f16] == protos[split], f16


def test_f16_entries_bound_and_exported(lib_built):
    from sonet_b200 import _C
    assert sorted(_C.F16_ENTRIES) == sorted(F16_ENTRIES)
    for split, f16 in zip(SPLIT_ENTRIES, F16_ENTRIES):
        assert _C._SIGNATURES[f16] == _C._SIGNATURES[split]
    h = ctypes.CDLL(lib_built)
    for n in F16_ENTRIES:
        assert hasattr(h, n), "library does not export %s" % n


def test_ops_entry_names():
    from sonet_b200 import ops
    for n in SPLIT_ENTRIES:
        assert ops._entry(n, False) == n
        assert ops._entry(n, True) == n + "_f16"


def test_f16_entries_validate_arguments_before_launching(lib_built):
    """Bad arguments come back as error codes, as from the split entries, without a device."""
    from sonet_b200 import _C
    lib = _C.lib()
    assert lib.sonet_pointresnet_tc_forward_f16(None, 7, 1, 1, None, None, None, None) == -1
    assert "Cin=7" in _C.last_error()
    assert lib.sonet_knn_mlp_tc_forward_f16(None, None, None, 1, 4, 1, 1, None, 4, 1, None, None,
                                            1.0, None, None, None) == -1
    assert "K=1" in _C.last_error()
    assert lib.sonet_pointwise_tc_forward_f16(None, 0, None, 0, 1, 1, None, 1.0, None, 1, 1, None,
                                              None, 0, None, None) == -1
    assert lib.sonet_pointwise_tc_grouped_forward_f16(None, 64, 1, 1, None, 0, 1.0, None, 64, 1, 0,
                                                      1, 0, 0, 0, 0, None, None, None) == -1
