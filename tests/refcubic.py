"""ctypes wrapper of oracle/_ref/libref_cubic.so: the REFERENCE's own inversion-filter code (get_feasible_steps.cpp: the quadratic and
cubic smallest-positive-root finders and the absolute-coordinate coefficient lines of computeInjectiveStepSize_3d) compiled from
/root/reference by oracle/build_ref.sh.  Used to pin the reference's formula to tests/golden/inversion_regimes_golden.npz.  Test
infrastructure only."""
import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_cubic.so")
_dp = C.POINTER(C.c_double)


def available():
    return os.path.exists(PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(PATH)
        _lib.ref_quad_root.restype = _lib.ref_cubic_root.restype = C.c_double
        _lib.ref_quad_root.argtypes = [C.c_double] * 4
        _lib.ref_cubic_root.argtypes = [C.c_double] * 5
        _lib.ref_inversion_coefs.argtypes = [_dp, _dp, C.c_double, _dp]
    return _lib


def quad_root(a, b, c, tol=1e-6):
    return lib().ref_quad_root(a, b, c, tol)


def cubic_root(a, b, c, d, tol=1e-6):
    return lib().ref_cubic_root(a, b, c, d, tol)


def coefs(X, P, slack):
    """(a, b, c, d) as the reference expands them from the four vertices X (4,3) and their directions P (4,3)"""
    X = np.ascontiguousarray(X, dtype=np.float64).ravel()
    P = np.ascontiguousarray(P, dtype=np.float64).ravel()
    out = np.empty(4)
    lib().ref_inversion_coefs(X.ctypes.data_as(_dp), P.ctypes.data_as(_dp), slack, out.ctypes.data_as(_dp))
    return out
