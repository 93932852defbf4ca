"""ctypes binding of tests/extrema_exact.cpp: the binary128 maximum of |p^(k)(t)| over a trajectory.

TEST INFRASTRUCTURE ONLY: imported by tests/test_time_objective.py and tools/extrema_bench.py."""
import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_DIR, "extrema_exact.cpp")
_SO = os.path.join(_DIR, "libextrema_exact.so")
_lib = None

_dp = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_ip = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")


def build():
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread",
                               "-Wall", "-o", _SO, _SRC])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        L.exact_max_magnitude.restype = C.c_int
        L.exact_max_magnitude.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int64, _dp, _dp, C.c_int, _dp, _dp, _ip, _dp,
                                          _dp, C.c_int]
        _lib = L
    return _lib


def max_magnitude(times, coeffs, k, n_threads=None):
    """times [B][K], coeffs [B][K][D][N] -> dict(value, time, segment, runner_up, scale), each [B]."""
    times = np.ascontiguousarray(times, dtype=np.float64)
    coeffs = np.ascontiguousarray(coeffs, dtype=np.float64)
    B, K, D, N = coeffs.shape
    out = {n: np.zeros(B) for n in ("value", "time", "runner_up", "scale")}
    seg = np.zeros(B, dtype=np.int32)
    rc = lib().exact_max_magnitude(N, K, D, B, times, coeffs, int(k), out["value"], out["time"], seg, out["runner_up"],
                                   out["scale"], int(n_threads or os.cpu_count() or 1))
    if rc != 0:
        raise ValueError(f"exact_max_magnitude rc={rc}")
    out["segment"] = seg
    return out
