"""Builds libvalle_b200.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc.

    python -m valle_b200.build [--force]

The shared object lands in valle_b200/lib/ (git-ignored).  No torch / pybind dependency: the ABI is plain C (include/valle_b200.h).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libvalle_b200.so")
OBJDIR = os.path.join(HERE, "build")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest() -> str:
    h = hashlib.sha256()
    files = sorted(os.listdir(CSRC)) + ["../../include/valle_b200.h"]
    for f in files:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p):
            h.update(f.encode())
            with open(p, "rb") as fh:
                h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False, trace: bool = False) -> str:
    """trace=True builds the profiling variant libvalle_b200_trace.so (-DVB_TRACE: device timeline stamps in the
    AR decode-step kernels, tools/trace_ar_step.py); the product library carries no tracing code."""
    lib = LIB.replace(".so", "_trace.so") if trace else LIB
    objdir = OBJDIR + ("_trace" if trace else "")
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(objdir, exist_ok=True)
    stamp = lib[:-3] + ".stamp"
    dig = _digest()
    if not force and os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == dig:
        return lib
    nvcc = _nvcc()
    extra = (["-Xptxas", "-v"] if verbose else []) + (["-DVB_TRACE"] if trace else [])

    def compile_one(src):
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *extra, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(sources()))) as ex:
        objs = list(ex.map(compile_one, sources()))
    cmd = [nvcc, "-shared", "-o", lib, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, trace="--trace" in sys.argv))
