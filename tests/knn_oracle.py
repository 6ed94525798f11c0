"""ctypes binding of tests/knn_oracle.c (the CPU statement of cs_match_knn2) and a numpy statement of the ratio test.

TEST INFRASTRUCTURE ONLY: imported by tests/ and scripts/knn_bench.py, never by the cudasift_b200 package."""
import ctypes

import numpy as np

from cudasift_b200 import build
from cudasift_b200.records import SIFT_DTYPE

_lib = None


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build.build_knn_oracle())
        L.knn_oracle_match_knn2.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_int]
        L.knn_oracle_match_knn2.restype = None
        _lib = L
    return _lib


def match_knn2(s1, s2, threads=8):
    """(idx int32 [n1, 2], score float32 [n1, 2]): the two nearest neighbours of every row of s1 among all rows of s2."""
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE)
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE)
    idx, score = np.full((len(s1), 2), -1, np.int32), np.zeros((len(s1), 2), np.float32)
    if len(s1) and len(s2):
        lib().knn_oracle_match_knn2(s1.ctypes.data, len(s1), s2.ctypes.data, len(s2), idx.ctypes.data, score.ctypes.data,
                                    int(threads))
    return idx, score


def ratio_keep(idx, score, maxRatio, maxDistance):
    """COLMAP's one-way test per row, in float64: d = arccos(min(score, 1)); j1 >= 0, d1 <= maxDistance and
    d1 < maxRatio * d2 (a missing second neighbour has score 0: d2 = pi / 2).  Also returns the smaller of the two
    margins, so that callers can exclude rows a last-bit difference in arccos could flip."""
    d = np.arccos(np.minimum(score.astype(np.float64), 1.0))
    r, m = float(np.float32(maxRatio)), float(np.float32(maxDistance))
    keep = (idx[:, 0] >= 0) & (d[:, 0] <= m) & (d[:, 0] < r * d[:, 1])
    margin = np.minimum(np.abs(d[:, 0] - m), np.abs(d[:, 0] - r * d[:, 1]))
    margin[idx[:, 0] < 0] = np.inf
    return keep, margin


def ratio_pairs(idx1, score1, idx2, score2, maxRatio, maxDistance, crossCheck):
    """(pairs int32 [k, 2] in increasing i, smallest margin of the rows that decide them)."""
    keep, margin = ratio_keep(idx1, score1, maxRatio, maxDistance)
    i = np.arange(len(idx1))
    j = idx1[:, 0]
    if crossCheck:
        k2, m2 = ratio_keep(idx2, score2, maxRatio, maxDistance)
        jj = np.where(j >= 0, j, 0)
        keep &= (j >= 0) & k2[jj] & (idx2[jj, 0] == i)
        margin = np.where(j >= 0, np.minimum(margin, m2[jj]), margin)
    return np.stack([i[keep], j[keep]], axis=1).astype(np.int32), float(margin.min()) if len(margin) else np.inf
