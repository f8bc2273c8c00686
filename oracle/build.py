"""Build the oracle's native pieces (TEST INFRASTRUCTURE — see oracle/oracle_c.c header).

  oracle/_build/liboracle_c.so   gcc -O2 -ffp-contract=off oracle_c.c        (always)
  oracle/_ref/index_max*.so  the REFERENCE's own plugin, compiled from the sources where they
                                 lie under /root/reference/models/index_max_ext (read-only, never
                                 copied), with torch.utils.cpp_extension — only when /root/reference
                                 exists (this container). The GPU box uses the prebuilt file.
  oracle/_ref/pyref/{models,util}/*.pyc   the REFERENCE's own Python modules compiled to CPython
                                 bytecode (py_compile) from the sources where they lie — binary
                                 build products like the .so above, never the sources. Python imports
                                 sourceless .pyc files, so the unmodified reference Model classes
                                 (models/{classifier,segmenter,autoencoder}.py) can run on the GPU
                                 box, where /root/reference does not exist: (a) as the CPU arm of
                                 bench.py ("kind": "reference") and (b) on top of sonet_b200's
                                 networks in the drop-in GPU test. Same interpreter image on both
                                 sides, so the bytecode magic matches; if it ever does not, the
                                 importers fall back to the oracle port and say so.
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
BUILD = os.path.join(HERE, "_build")
REFDIR = os.path.join(HERE, "_ref")
LIB = os.path.join(BUILD, "liboracle_c.so")
REF_SRC = "/root/reference/models/index_max_ext"


def build_c(force=False):
    os.makedirs(BUILD, exist_ok=True)
    src = os.path.join(HERE, "oracle_c.c")
    if force or not os.path.exists(LIB) or os.path.getmtime(src) > os.path.getmtime(LIB):
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", LIB,
                               src, "-lm"])
        print("[oracle] built", os.path.relpath(LIB, HERE))
    return LIB


def ref_plugin_path():
    hits = sorted(glob.glob(os.path.join(REFDIR, "index_max*.so")))
    return hits[0] if hits else None


def build_ref(force=False):
    """Compile the reference plugin in place (sources are only read). ~2-3 minutes, once."""
    if ref_plugin_path() and not force:
        return ref_plugin_path()
    if not os.path.isdir(REF_SRC):
        return None
    os.makedirs(REFDIR, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils.cpp_extension import load
    scratch = os.path.join(REFDIR, "_scratch")
    os.makedirs(scratch, exist_ok=True)
    load(name="index_max",
         sources=[os.path.join(REF_SRC, "index_max.cpp"), os.path.join(REF_SRC, "index_max_cuda.cu")],
         build_directory=scratch, verbose=False)
    built = glob.glob(os.path.join(scratch, "index_max*.so"))
    for b in built:
        os.replace(b, os.path.join(REFDIR, os.path.basename(b)))
    # keep only the shared object (objects/ninja files are scratch)
    for f in glob.glob(os.path.join(scratch, "*")):
        try:
            os.remove(f)
        except OSError:
            pass
    try:
        os.rmdir(scratch)
    except OSError:
        pass
    print("[oracle] built reference plugin ->", ref_plugin_path())
    return ref_plugin_path()


PYREF = os.path.join(REFDIR, "pyref")
REF_ROOT = "/root/reference"
_PYREF_PKGS = ("models", "util")


def pyref_root():
    """Directory holding the bytecode-compiled reference packages, or None if not built / stale
    for this interpreter."""
    import importlib.util
    probe = os.path.join(PYREF, "models", "classifier.pyc")
    if not os.path.exists(probe):
        return None
    with open(probe, "rb") as f:
        if f.read(4) != importlib.util.MAGIC_NUMBER:
            return None
    return PYREF


def build_pyref(force=False):
    """py_compile every top-level module of the reference's `models` and `util` packages into
    oracle/_ref/pyref (sourceless .pyc). Only possible where /root/reference exists."""
    import py_compile
    if not os.path.isdir(os.path.join(REF_ROOT, "models")):
        return pyref_root()
    if pyref_root() and not force:
        return PYREF
    n = 0
    for pkg in _PYREF_PKGS:
        src_dir = os.path.join(REF_ROOT, pkg)
        dst_dir = os.path.join(PYREF, pkg)
        os.makedirs(dst_dir, exist_ok=True)
        for f in sorted(os.listdir(src_dir)):
            if not f.endswith(".py"):
                continue
            py_compile.compile(os.path.join(src_dir, f), cfile=os.path.join(dst_dir, f + "c"),
                               dfile="%s/%s" % (pkg, f), doraise=True)
            n += 1
    print("[oracle] compiled %d reference modules to bytecode -> %s" % (n, os.path.relpath(PYREF, HERE)))
    return PYREF


if __name__ == "__main__":
    build_c(force="--force" in sys.argv)
    if "--no-ref" not in sys.argv:
        build_ref(force="--force-ref" in sys.argv)
        build_pyref(force="--force-ref" in sys.argv)
