"""Build libsonet_b200.so (C-ABI, no libtorch dependency) with nvcc for sm_90a, in-tree.

    python so-net_b200/build.py [--force] [--verbose]

The shared library lands in so-net_b200/lib/ (git-ignored, but it travels with gpurun snapshots).
Objects are rebuilt only when a source or header is newer than the object.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "libsonet_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--use_fast_math=false",
          "-Xptxas", "-v", "-I", INCLUDE]
# --use_fast_math is NOT used: parity needs IEEE division/sqrt and no FMA contraction surprises
CFLAGS = [f for f in CFLAGS if not f.startswith("--use_fast_math")]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs += [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    return hs


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    hdr_mtime = max(os.path.getmtime(h) for h in headers())
    jobs = []
    objs = []
    for src in sources():
        obj = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        stale = force or _newer(src, obj) or hdr_mtime > os.path.getmtime(obj)
        if stale:
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [NVCC, *ARCH, *CFLAGS, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = r.stdout + r.stderr
        with open(obj + ".log", "w") as f:
            f.write(" ".join(cmd) + "\n" + log)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, log))
        if verbose:
            print(log)
        return src

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            for s in ex.map(compile_one, jobs):
                print("[build] compiled", os.path.relpath(s, HERE))
    if jobs or not os.path.exists(LIB):
        cmd = [NVCC, *ARCH, "-shared", "-o", LIB, *objs, "-lcudart", "-lpthread", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
        print("[build] linked", os.path.relpath(LIB, HERE))
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
