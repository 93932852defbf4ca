"""ctypes binding of tests/half_plane_exact.cpp: the binary128 replay of FeasibilityBase::checkHalfPlaneFeasibility
over B trajectories, and the exact check of the GPU shortcut's bound.

TEST INFRASTRUCTURE ONLY: imported by tests/test_half_plane_feasibility.py."""
import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_DIR, "half_plane_exact.cpp")
_DEPS = (_SRC, os.path.join(_DIR, "extrema_exact.cpp"))
_SO = os.path.join(_DIR, "libhalf_plane_exact.so")
_lib = None
PATH_END_POINT, PATH_SHORTCUT, PATH_ISOLATION = 1, 2, 4

_dp = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")
_ip = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")


def build():
    if not os.path.exists(_SO) or any(os.path.getmtime(_SO) < os.path.getmtime(d) for d in _DEPS):
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread",
                               "-ffp-contract=off", "-Wall", "-o", _SO, _SRC])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        L.exact_half_plane.restype = C.c_int
        L.exact_half_plane.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int64, _dp, _dp, C.c_int, _dp, _ip, _ip, _ip,
                                       _dp, _ip, C.c_int]
        L.exact_half_plane_bound.restype = None
        L.exact_half_plane_bound.argtypes = [C.c_int, C.c_double, _dp, _dp, C.c_int, _dp, _dp]
        _lib = L
    return _lib


def half_plane_feasibility(times, coeffs, planes, n_threads=None):
    """times [B][K], coeffs [B][K][D][N], planes [P][6] -> dict(feasible, segment, plane, margin, paths), each [B]:
    margin is the smallest relative |minimum distance| over the visited (segment, plane) pairs, less the fp64
    evaluation's forward-error factor; paths is the OR over those pairs of the kernel step that decides them
    (PATH_END_POINT, PATH_SHORTCUT, PATH_ISOLATION)."""
    times = np.ascontiguousarray(times, dtype=np.float64)
    coeffs = np.ascontiguousarray(coeffs, dtype=np.float64)
    planes = np.ascontiguousarray(np.asarray(planes, dtype=np.float64).reshape(-1, 6))
    B, K, D, N = coeffs.shape
    out = dict(feasible=np.zeros(B, dtype=np.int32), segment=np.zeros(B, dtype=np.int32),
               plane=np.zeros(B, dtype=np.int32), margin=np.zeros(B),
               paths=np.zeros(B, dtype=np.int32))
    rc = lib().exact_half_plane(N, K, D, B, times, coeffs, len(planes), planes if len(planes) else np.zeros(6),
                                out["feasible"], out["segment"], out["plane"], out["margin"], out["paths"],
                                int(n_threads or os.cpu_count() or 1))
    if rc != 0:
        raise ValueError(f"exact_half_plane rc={rc}")
    return out


def shortcut_bound(coeffs, T, plane, ts):
    """One segment (coeffs [D][N]) and plane: dict(bmin, E, exact_min, eval_err, bern_err) -- the kernel's fp64
    Bernstein minimum and bound, the exact minimum distance on [0, T], and the largest fp64 evaluation error at the
    times ts and Bernstein-coefficient error, both measured in binary128."""
    c = np.ascontiguousarray(coeffs, dtype=np.float64)
    N = c.shape[1]
    out = np.zeros(5)
    ts = np.ascontiguousarray(ts, dtype=np.float64)
    lib().exact_half_plane_bound(N, float(T), c, np.ascontiguousarray(plane, dtype=np.float64), len(ts), ts, out)
    return dict(zip(("bmin", "E", "exact_min", "eval_err", "bern_err"), out))
