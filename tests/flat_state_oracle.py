"""ctypes binding of tests/flat_state_exact.cpp: the attitude of a flat state (yaw or rotation vector) in binary128.

TEST INFRASTRUCTURE ONLY: imported by tests/test_flat_state_sampling.py."""
import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_DIR, "flat_state_exact.cpp")
_SO = os.path.join(_DIR, "libflat_state_exact.so")
_lib = None

_dp = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")


def build():
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o",
                               _SO, _SRC])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        for name in ("exact_rotation_vector_state", "exact_yaw_state"):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = [C.c_int64, _dp, _dp, _dp, _dp, _dp, _dp]
        L.exact_jacobian_coefficients.restype = C.c_int
        L.exact_jacobian_coefficients.argtypes = [C.c_double, _dp]
        _lib = L
    return _lib


def _run(fn, a, da, dda, width):
    a, da, dda = (np.ascontiguousarray(x, dtype=np.float64).reshape(-1, width) for x in (a, da, dda))
    M = a.shape[0]
    q, w, wd = np.zeros((M, 4)), np.zeros((M, 3)), np.zeros((M, 3))
    fn(M, a.ravel(), da.ravel(), dda.ravel(), q, w, wd)
    return q, w, wd


def rotation_vector_state(phi, dphi, ddphi):
    """phi, dphi, ddphi [M][3] -> (q [M][4] (w, x, y, z), omega [M][3], omega_dot [M][3]), binary128 rounded once."""
    return _run(lib().exact_rotation_vector_state, phi, dphi, ddphi, 3)


def yaw_state(yaw, yaw_rate, yaw_acc):
    """yaw, yaw_rate, yaw_acc [M] -> (q [M][4], omega [M][3], omega_dot [M][3])."""
    return _run(lib().exact_yaw_state, yaw, yaw_rate, yaw_acc, 1)


def jacobian_coefficients(t):
    """(a, b, a'/t, b'/t) of the left Jacobian of SO(3) at angle t."""
    out = np.zeros(4)
    lib().exact_jacobian_coefficients(float(t), out)
    return out
