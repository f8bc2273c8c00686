"""C-ABI: the shared library loads and exports exactly what include/sonet_b200.h declares;
argument validation and the host (CPU) plugin entry points work without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "sonet_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sonet_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(lib_built):
    h = ctypes.CDLL(lib_built)
    names = declared_symbols()
    assert len(names) >= 15
    for n in names:
        assert hasattr(h, n), "library does not export %s" % n


def test_python_binding_covers_header(lib_built):
    from sonet_b200 import _C
    assert sorted(_C.EXPORTED_SYMBOLS) == declared_symbols()
    lib = _C.lib()
    assert b"sm_90a" in lib.sonet_version()


def test_library_has_no_torch_dependency(lib_built):
    import subprocess
    out = subprocess.run(["ldd", lib_built], capture_output=True, text=True).stdout
    assert "libtorch" not in out and "libc10" not in out


def test_bad_arguments_return_error_codes(lib_built):
    from sonet_b200 import _C
    lib = _C.lib()
    # K out of range is rejected before any CUDA call
    rc = lib.sonet_index_max_f32(None, None, 1, 1, 1, 0, None, None, None)
    assert rc == -1 and "K=0" in _C.last_error()
    rc = lib.sonet_index_max_f32(None, None, 1, 1, 4, 64, None, None, None)
    assert rc == -1 and "null" in _C.last_error()
    rc = lib.sonet_som_assign(None, None, 1, 8, 500, 3, None, None, None, None, None, None)
    assert rc == -1 and "M=500" in _C.last_error()
    rc = lib.sonet_som_assign(None, None, 1, 8, 64, 7, None, None, None, None, None, None)
    assert rc == -1
    rc = lib.sonet_chamfer_f32(None, None, 0, 1, 1, None, None, None, None, None, None, None, None)
    assert rc == -1
    with pytest.raises(RuntimeError):
        _C.check(rc, "chamfer")
    # entry points added in round 2: argument checks come before any CUDA call
    assert lib.sonet_seg_loss_f32(None, None, 2, 50, 1024, 1, None, None, None) == -1
    assert "null" in _C.last_error()
    assert lib.sonet_seg_loss_f32(None, None, 0, 50, 1024, 1, None, None, None) == -1
    assert lib.sonet_seg_loss_scratch_bytes(32, 1024) >= 32 * 4 * 12
    assert lib.sonet_seg_loss_scratch_bytes(-1, 4) == -1
    assert lib.sonet_linear_f32(None, 4, 0, None, None, None, 8, 0, None, None) == -1
    assert lib.sonet_linear_f32(None, 4, 16, None, None, None, 8, 0, None, None) == -1
    assert "null" in _C.last_error()
    assert lib.sonet_som_train(None, None, 0, None, None, 4, 2, 100, 300, None, None, None) == -1
    assert "M=300" in _C.last_error()
    assert lib.sonet_pointwise_tc_grouped_forward(None, 64, 2, 64, None, 0, 1.0, None, 64, 1, 4, 2, 0, 0,
                                                  64, 0, None, None, None) == -1      # split-K, no scratch
    # empty batches are a no-op success
    assert lib.sonet_linear_f32(None, 0, 16, None, None, None, 8, 0, None, None) == 0
    assert lib.sonet_index_max_f32(None, None, 0, 4, 4, 8, None, None, None) == 0
    assert lib.sonet_pointwise_layer_f32(None, 4, None, 0, 0, 16, None, None, None, 8, 1, None,
                                         None, 0, None, None) == 0


def test_som_group_mode_arithmetic(lib_built):
    """sonet_som_group_mode on an H100's 232448 B of opt-in shared memory: at M=64, k=3 the cloud
    (with normals) is staged up to N=6200 and som_group runs at all up to N=18601; one more point
    changes the mode. Host-only: the capacity is an argument."""
    from sonet_b200 import _C, ops
    lib = _C.lib()
    cap = 232448
    mode = lambda N, M=64, k=3, sn=1: lib.sonet_som_group_mode(N, M, k, sn, cap)  # noqa: E731
    assert (mode(6200), mode(6201)) == (ops.SOM_GROUP_STAGED, ops.SOM_GROUP_UNSTAGED)
    assert (mode(18601), mode(18602)) == (ops.SOM_GROUP_UNSTAGED, ops.SOM_GROUP_NONE)
    assert mode(6201, sn=0) == ops.SOM_GROUP_STAGED         # without normals: 3 channels staged
    for N in (6200, 6201, 18601, 18602):
        fits = lib.sonet_som_group_smem_bytes(N, 64, 3) <= cap
        assert (mode(N) != ops.SOM_GROUP_NONE) == fits
    assert mode(1, M=256, k=4) == ops.SOM_GROUP_STAGED
    assert mode(1, M=257) == ops.SOM_GROUP_NONE              # every SOM kernel stops at M=256
    assert mode(1 << 24, k=1) == ops.SOM_GROUP_NONE          # node ids share 32 bits with n
    assert lib.sonet_som_group_mode(1 << 24, 64, 1, 1, 1 << 40) == ops.SOM_GROUP_NONE
    assert mode(10, k=0) < 0 and "k=0" in _C.last_error()


def test_cuda_entry_points_reject_host_tensors():
    from sonet_b200 import index_max
    data = torch.zeros(1, 2, 8)
    idx = torch.zeros(1, 8, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="CUDA"):
        index_max.forward_cuda(data, idx, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        index_max.forward_cuda_shared_mem(data, idx, 4)


def test_plugin_cpu_entry_points_known_answer(oracle_mod):
    """SURVEY.md §8c known-answer fact, verified on the reference binary."""
    from sonet_b200 import index_max
    d = torch.tensor([[[1, 5, 5, -2000, 3, 3]]], dtype=torch.float32)
    i = torch.tensor([[0, 1, 1, 2, 3, 3]], dtype=torch.int32)
    assert index_max.forward_cpu(d, i, 5).tolist() == [[[0, 1, 0, 4, 0]]]
    assert index_max.forward_multi_thread_cpu(d, i, 5, 3).tolist() == [[[0, 1, 0, 4, 0]]]
    rs = np.random.RandomState(0)
    data = torch.from_numpy(rs.normal(size=(3, 21, 257)).astype(np.float32))
    index = torch.from_numpy(rs.randint(0, 13, size=(3, 257)).astype(np.int32))
    want = oracle_mod.index_max(data, index, 13)
    assert torch.equal(index_max.forward_cpu(data, index, 13), want)
    assert torch.equal(index_max.forward_multi_thread_cpu(data, index, 13, 4), want)
    with pytest.raises(RuntimeError):
        index_max.forward_cpu(data, index.clamp(min=0) + 100, 13)


def test_every_wrapper_call_names_a_bound_symbol_with_the_right_arity():
    """Static check (no GPU): each `_call("sonet_...", args...)` / `_C.lib().sonet_...(args...)` in the
    Python layer names a symbol of the ctypes table and passes as many arguments as it declares —
    a typo here would otherwise only surface on a GPU box."""
    import ast
    import glob
    import os

    from sonet_b200 import _C
    pkg = os.path.dirname(_C.__file__)
    seen = set()
    for path in sorted(glob.glob(os.path.join(pkg, "*.py"))):
        tree = ast.parse(open(path).read(), path)
        for node in ast.walk(tree):
            if not isinstance(node, ast.Call):
                continue
            name, nargs = None, None
            f = node.func
            if isinstance(f, ast.Name) and f.id == "_call" and node.args and \
                    isinstance(node.args[0], ast.Constant) and isinstance(node.args[0].value, str):
                name, nargs = node.args[0].value, len(node.args) - 1
            elif isinstance(f, ast.Attribute) and f.attr.startswith("sonet_"):
                name, nargs = f.attr, len(node.args)
            if name is None:
                continue
            where = "%s:%d" % (os.path.basename(path), node.lineno)
            assert name in _C._SIGNATURES, "%s calls unknown symbol %s" % (where, name)
            if not any(isinstance(x, ast.Starred) for x in node.args):
                assert nargs == len(_C._SIGNATURES[name]), \
                    "%s passes %d args to %s (declared %d)" % (where, nargs, name,
                                                               len(_C._SIGNATURES[name]))
            seen.add(name)
    assert len(seen) >= 25, sorted(seen)


def _header_text():
    text = open(os.path.join(ROOT, "include", "sonet_b200.h")).read()
    return re.sub(r"/\*.*?\*/", " ", text, flags=re.S)          # strip comments


def _header_prototypes():
    """name -> (return type, parameter list) of every prototype in include/sonet_b200.h: this
    test's own reading of the header, independent of the binding's parser."""
    protos = {}
    for ret, name, params in re.findall(r"^[ \t]*(\w[\w \t*]*?)\s*\b(sonet_\w+)\s*\(([^;{]*?)\)\s*;",
                                        _header_text(), flags=re.M):
        params = " ".join(params.split())
        protos[name] = (" ".join(ret.split()),
                        [] if params in ("", "void") else [q.strip() for q in params.split(",")])
    return protos


def _machine_type(name, q):
    """The ctypes type a C declaration `q` (a parameter, or a return type) passes as."""
    if re.fullmatch(r"const char\s*\*", q):
        return ctypes.c_char_p
    if "*" in q or "sonet_stream_t" in q:
        return ctypes.c_void_p
    if "unsigned long long" in q:
        return ctypes.c_ulonglong
    if "long long" in q:
        return ctypes.c_longlong
    if re.match(r"(const\s+)?double\b", q):
        return ctypes.c_double
    if re.match(r"(const\s+)?float\b", q):
        return ctypes.c_float
    assert re.match(r"(const\s+)?int\b", q), "%s: unhandled type %r" % (name, q)
    return ctypes.c_int


def test_ctypes_arity_matches_the_header_prototypes():
    """The ctypes argtypes of every symbol have as many entries as its prototype in
    include/sonet_b200.h has parameters (a mismatch corrupts the call frame silently)."""
    from sonet_b200 import _C
    protos = _header_prototypes()
    assert set(protos) == set(_C._SIGNATURES) == set(declared_symbols())
    for name, (_, plist) in protos.items():
        sig = _C._SIGNATURES[name]
        assert len(plist) == len(sig), "%s: header %d parameters, ctypes %d" % (name, len(plist),
                                                                              len(sig))
        for q, ct in zip(plist, sig):           # and the same machine type, parameter by parameter
            want = _machine_type(name, q)
            assert ct is want, "%s: parameter %r is bound as %s" % (name, q, ct.__name__)


def test_ctypes_restypes_match_the_header_prototypes(lib_built):
    """Every bound entry returns the type its prototype declares: a `long long` size query read
    as a C int would come back truncated, a `const char*` as a number."""
    from sonet_b200 import _C
    lib = _C.lib()
    for name, (ret, _) in _header_prototypes().items():
        restype = getattr(lib, name).restype
        assert restype is _machine_type(name, ret), "%s: returns %r, bound as %s" % (
            name, ret, restype.__name__)
    assert lib.sonet_wgrad_kpad(1 << 16, 1 << 16, 1) == 1 << 32         # not truncated to 32 bits


def test_header_constants():
    """Every `#define SONET_<NAME> <int>` of the header is in _C.CONSTANTS with its value, and the
    Python names of the codes ops.py passes to the library hold the header's values."""
    from sonet_b200 import _C, ops
    defines = re.findall(r"^\s*#define\s+(SONET_\w+)\s+\(?\s*(-?\d+)\s*\)?\s*$", _header_text(),
                         flags=re.M)
    want = {n: int(v) for n, v in defines}
    assert len(want) >= 17 and want["SONET_ERR_BAD_ARG"] == -1
    assert _C.CONSTANTS == want
    for group, names in (("ACT", ("NONE", "RELU", "ELU")), ("SAMPLE", ("SUBSET", "FILL", "MAX_P")),
                         ("REDUCE", ("NONE", "KCOPY_MEAN", "GROUP_MAX")),
                         ("SOM_GROUP", ("NONE", "UNSTAGED", "STAGED"))):
        for n in names:
            assert getattr(ops, "%s_%s" % (group, n)) == want["SONET_%s_%s" % (group, n)], (group, n)


def test_binding_parser_refuses_unknown_types():
    """The binding's header parser binds only types with an exact ctypes twin: anything else
    raises naming the entry and the parameter; `(void)` and `()` take no arguments."""
    from sonet_b200 import _C
    with pytest.raises(RuntimeError, match=r"sonet_x: parameter 'size_t n'"):
        _C.parse_header("int sonet_x(const float* a,\n            size_t n, sonet_stream_t s);")
    with pytest.raises(RuntimeError, match=r"sonet_y: return type 'unsigned'"):
        _C.parse_header("unsigned sonet_y(int n);")
    sigs, res, consts = _C.parse_header(
        "typedef void* sonet_stream_t; /* sonet_w(x) */\n#define SONET_A (-4)\n#define SONET_B 7\n"
        "long long sonet_v(void);\nint sonet_u();\nconst char* sonet_t(unsigned long long s,\n"
        "                  double d, float f, int** p);\n")
    assert sigs == {"sonet_v": [], "sonet_u": [],
                    "sonet_t": [ctypes.c_ulonglong, ctypes.c_double, ctypes.c_float, ctypes.c_void_p]}
    assert res == {"sonet_v": ctypes.c_longlong, "sonet_u": ctypes.c_int, "sonet_t": ctypes.c_char_p}
    assert consts == {"SONET_A": -4, "SONET_B": 7}
