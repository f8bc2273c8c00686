"""ctypes binding of libsonet_b200.so (the C-ABI declared in include/sonet_b200.h).

The library is the product: if it is missing, importing any op raises — there is NO Python/CPU
fallback for the CUDA entry points. Tensors cross the boundary as raw device pointers; outputs
are allocated by the caller (here, by the thin wrappers in ops.py with torch.empty).

The header is the one statement of the ABI: the ctypes argument and return types of every entry
and the SONET_* constants are read from it at import, without loading the library.
"""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(_HERE))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libsonet_b200.so")
HEADER_PATH = os.path.join(ROOT, "include", "sonet_b200.h")

_lib = None

_SCALARS = {"int": ctypes.c_int, "long long": ctypes.c_longlong,
            "unsigned long long": ctypes.c_ulonglong, "float": ctypes.c_float,
            "double": ctypes.c_double}
# `<return type> sonet_<name>(<parameters, possibly over several lines>);` at the start of a line
_PROTOTYPE = re.compile(r"^[ \t]*(\w[\w \t*]*?)\s*\b(sonet_\w+)\s*\(([^;]*?)\)\s*;", re.M)
_DEFINE = re.compile(r"^#define\s+(SONET_\w+)\s+\(?(-?\d+)\)?\s*$", re.M)


def _ctype(entry, decl, param=True):
    """The ctypes type of a parameter declaration `type name` of `entry` (param) or of its return
    type. Pointers and streams pass as void*; a type with no exact ctypes twin raises, so that a new
    entry is never bound as something it is not."""
    if not param and re.fullmatch(r"const\s+char\s*\*", decl):
        return ctypes.c_char_p
    if "*" in decl or "sonet_stream_t" in decl.split():
        return ctypes.c_void_p
    m = re.fullmatch(r"(?:const\s+)?(\w+(?:\s+\w+)*?)" + (r"\s+\w+" if param else ""), decl)
    scalar = m and " ".join(m.group(1).split())
    if scalar in _SCALARS:
        return _SCALARS[scalar]
    raise RuntimeError("%s: %s %r has no ctypes binding" % (
        entry, "parameter" if param else "return type", decl))


def parse_header(text):
    """(argtypes, restypes, constants) of the C-ABI declared in the header text `text`: entry name
    -> list of ctypes argument types and -> ctypes return type, both in declaration order, and
    every `#define SONET_<NAME> <int>` as {"SONET_<NAME>": int}."""
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)    # comments hold call-like text
    argtypes, restypes = {}, {}
    for ret, name, params in _PROTOTYPE.findall(text):
        params = " ".join(params.split())
        argtypes[name] = [] if params in ("", "void") else \
            [_ctype(name, p.strip()) for p in params.split(",")]
        restypes[name] = _ctype(name, ret.strip(), param=False)
    constants = {n: int(v) for n, v in _DEFINE.findall(text)}
    return argtypes, restypes, constants


with open(HEADER_PATH) as _f:
    _SIGNATURES, _RESTYPE, CONSTANTS = parse_header(_f.read())

EXPORTED_SYMBOLS = tuple(_SIGNATURES)
# the one-product twins of the train-mode GEMM entries (SONET_TRAIN_TC=fp16)
TRAIN_F16_ENTRIES = ("sonet_pointwise_tc_forward_dev_f16", "sonet_pointwise_tc_grouped_forward_dev_f16",
                     "sonet_wgrad_tc_f16")
# the opt-in fp16 mode's twins of the eval wgmma entries (same arguments as the split entry)
F16_ENTRIES = tuple(n for n in _SIGNATURES if n.endswith("_f16") and n not in TRAIN_F16_ENTRIES)
# the fused kernels with an explicit activation code (SONET_ACT_RELU / _ELU) and f16 flag
ACT_ENTRIES = tuple(n for n in _SIGNATURES if n.endswith("_act"))


def lib():
    """Load (once) and return the ctypes handle. Raises if the library has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libsonet_b200.so not found at %s — build it with `python so-net_b200/build.py` "
                "(there is no fallback path)" % LIB_PATH)
        handle = ctypes.CDLL(LIB_PATH)
        for name, argtypes in _SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if a declared symbol is not exported
            fn.argtypes = argtypes
            fn.restype = _RESTYPE[name]
        _lib = handle
    return _lib


def last_error():
    return lib().sonet_last_error_string().decode("utf-8", "replace")


def check(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (what, rc, last_error()))


def ptr(t):
    """Device/host pointer of a tensor as an integer (None -> NULL)."""
    return None if t is None else t.data_ptr()
