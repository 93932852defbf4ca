"""ctypes binding of tests/feasibility_sampling_exact.cpp: the binary128 replay of FeasibilitySampling over B
trajectories.

TEST INFRASTRUCTURE ONLY: imported by tests/test_input_feasibility_sampling.py."""
import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_DIR, "feasibility_sampling_exact.cpp")
_SO = os.path.join(_DIR, "libfeasibility_sampling_exact.so")
_lib = None

_dp = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_ip = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")

LIMITS = ("f_min", "f_max", "v_max", "omega_xy_max", "omega_z_max", "omega_z_dot_max")


def build():
    # -ffp-contract=off: the running sum of sample times must be the reference's fp64 additions
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC",
                               "-shared", "-pthread", "-Wall", "-o", _SO, _SRC])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        L.exact_input_feasibility_sampling.restype = C.c_int
        L.exact_input_feasibility_sampling.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int64, _dp, _dp, C.c_uint32,
                                                       _dp, C.c_double, C.c_double, _ip, _ip, _ip, _dp, C.c_int]
        _lib = L
    return _lib


def input_feasibility_sampling(times, coeffs, limits, sampling_interval, gravity, n_threads=None):
    """times [B][K], coeffs [B][K][D][N], limits {name: value} -> dict(result, segment, status, margin), each [B]:
    margin is the smallest relative gap |q - limit| / limit of any comparison made up to the deciding one."""
    times = np.ascontiguousarray(times, dtype=np.float64)
    coeffs = np.ascontiguousarray(coeffs, dtype=np.float64)
    B, K, D, N = coeffs.shape
    present = 0
    lim = np.zeros(6)
    for q, n in enumerate(LIMITS):
        if n in limits:
            present |= 1 << q
            lim[q] = float(limits[n])
    out = dict(result=np.zeros(B, dtype=np.int32), segment=np.zeros(B, dtype=np.int32),
               status=np.zeros(B, dtype=np.int32), margin=np.zeros(B))
    rc = lib().exact_input_feasibility_sampling(N, K, D, B, times, coeffs, present, lim, float(gravity),
                                                float(sampling_interval), out["result"], out["segment"],
                                                out["status"], out["margin"], int(n_threads or os.cpu_count() or 1))
    if rc != 0:
        raise ValueError(f"exact_input_feasibility_sampling rc={rc}")
    return out
