"""In-tree build of the native libraries (nvcc for sm_90a, g++ for the host mirror).

  libmtg_b200.so   CUDA kernels + the C-ABI of include/mtg_b200.h          (csrc/*.cu)
  libmtg_host.so   C++ mirror of the reference's Vertex/Segment/Polynomial/
                   PolynomialOptimization<N> API on top of the C-ABI       (host/src/*.cpp)

Everything is compiled with explicit commands (no JIT cache) so the .so files travel with the
repository snapshot to the GPU box.
"""
import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
HOST = os.path.join(PKG, "host")
LIB_CUDA = os.path.join(PKG, "libmtg_b200.so")
LIB_HOST = os.path.join(PKG, "libmtg_host.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-shared", "-Wall"]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the CUDA extension cannot be built")


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _sources(d, exts):
    out = []
    for base, _, files in os.walk(d):
        for f in files:
            if f.endswith(exts):
                out.append(os.path.join(base, f))
    return sorted(out)


def build_cuda(force=False, verbose=False):
    deps = _sources(CSRC, (".cu", ".cuh", ".h")) + [os.path.join(ROOT, "include", "mtg_b200.h")]
    if force or _newer(LIB_CUDA, deps):
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
              ["-o", LIB_CUDA, os.path.join(CSRC, "mtg_capi.cu")]
        subprocess.check_call(cmd)
    return LIB_CUDA


def build_host(force=False):
    srcs = _sources(os.path.join(HOST, "src"), (".cpp",))
    if not srcs:
        return None
    deps = srcs + _sources(os.path.join(HOST, "include"), (".h",)) + [os.path.join(ROOT, "include", "mtg_b200.h")]
    if force or _newer(LIB_HOST, deps + [LIB_CUDA]):
        cxx = os.environ.get("CXX", "g++")
        cmd = [cxx] + CXX_FLAGS + ["-I", os.path.join(HOST, "include"), "-I", os.path.join(ROOT, "include"),
                                   "-o", LIB_HOST] + srcs + \
              ["-L", PKG, "-lmtg_b200", "-Wl,-rpath,$ORIGIN"]
        subprocess.check_call(cmd)
    return LIB_HOST


def build_all(force=False, verbose=False):
    build_cuda(force=force, verbose=verbose)
    build_host(force=force)
