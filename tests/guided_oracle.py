"""ctypes binding of tests/guided_oracle.c (the CPU statement of cs_match_knn2_guided and of its predicate) and a numpy
float32 statement of the predicate.

TEST INFRASTRUCTURE ONLY: imported by tests/ and scripts/guided_bench.py, never by the cudasift_b200 package."""
import ctypes

import numpy as np

from cudasift_b200 import build
from cudasift_b200.records import SIFT_DTYPE

H, F = 1, 2          # CS_GEOM_HOMOGRAPHY, CS_GEOM_FUNDAMENTAL
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build.build_guided_oracle())
        L.guided_oracle_match_knn2.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                               ctypes.c_int, ctypes.c_void_p, ctypes.c_float, ctypes.c_int,
                                               ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        L.guided_oracle_match_knn2.restype = None
        L.guided_oracle_admissible.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_float] + \
            [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_void_p]
        L.guided_oracle_admissible.restype = None
        _lib = L
    return _lib


def _model(M):
    return np.ascontiguousarray(np.asarray(M, np.float64).reshape(9))


def match_knn2_guided(s1, s2, model, M, thresh, reverse=False, threads=8):
    """(idx int32 [rows, 2], score float32 [rows, 2]): the two nearest admissible neighbours of every row of s1 in s2,
    or (reverse) of every row of s2 in s1, under the model M (set-1 pixels to set-2 pixels) and thresh."""
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE)
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE)
    nr = len(s2) if reverse else len(s1)
    idx, score = np.full((nr, 2), -1, np.int32), np.zeros((nr, 2), np.float32)
    m = _model(M)
    if len(s1) and len(s2):
        lib().guided_oracle_match_knn2(s1.ctypes.data, len(s1), s2.ctypes.data, len(s2), int(model), m.ctypes.data,
                                       float(thresh), int(bool(reverse)), idx.ctypes.data, score.ctypes.data,
                                       int(threads))
    return idx, score


def admissible_c(model, M, thresh, x, y, u, v):
    """The C statement of the predicate, element by element."""
    x, y, u, v = (np.ascontiguousarray(a, np.float32) for a in (x, y, u, v))
    out = np.zeros(len(x), np.uint8)
    m = _model(M)
    lib().guided_oracle_admissible(int(model), m.ctypes.data, float(thresh), x.ctypes.data, y.ctypes.data,
                                   u.ctypes.data, v.ctypes.data, len(x), out.ctypes.data)
    return out.astype(bool)


def guided_model(M, thresh):
    """(f float32 [9], t2 float32): the model at unit Frobenius norm (sum of squares in index order, in double), rounded
    to float, and fl(thresh * thresh)."""
    m = _model(M)
    s = 0.0
    for v in m:
        s += float(v) * float(v)
    s = s ** 0.5
    return np.array([float(v) / s for v in m], np.float64).astype(np.float32), np.float32(thresh) * np.float32(thresh)


def admissible_np(model, M, thresh, x, y, u, v):
    """The predicate in numpy float32 (every operation one rounding), broadcasting over x, y, u, v."""
    f, t2 = guided_model(M, thresh)
    x, y, u, v = (np.asarray(a, np.float32) for a in (x, y, u, v))
    with np.errstate(all="ignore"):
        if model == F:
            l0 = (f[0] * x + f[1] * y) + f[2]
            l1 = (f[3] * x + f[4] * y) + f[5]
            l2 = (f[6] * x + f[7] * y) + f[8]
            a = l0 * l0 + l1 * l1
            m0 = (f[0] * u + f[3] * v) + f[6]
            m1 = (f[1] * u + f[4] * v) + f[7]
            b = m0 * m0 + m1 * m1
            num = (l0 * u + l1 * v) + l2
            ok = num * num < t2 * (a + b)
        else:
            px = (f[0] * x + f[1] * y) + f[2]
            py = (f[3] * x + f[4] * y) + f[5]
            pw = (f[6] * x + f[7] * y) + f[8]
            dx = u * pw - px
            dy = v * pw - py
            ok = dx * dx + dy * dy < t2 * (pw * pw)
    return ok & np.isfinite(x) & np.isfinite(y) & np.isfinite(u) & np.isfinite(v)
