"""cudasift_b200 -- H100-native (sm_90a) SIFT extraction + brute-force matching.

Python mirror of the reference's C++ interface (cudaSift.h / cudaImage.h of
Celebrandil/CudaSift): InitCuda, CudaImage, SiftData, ExtractSift, MatchSiftData keep their
names, argument meaning and defaults, and run through the C ABI of libcudasift_b200.so
(include/cudasift_b200.h).  There is no CPU fallback: without the CUDA library or without a
GPU every call raises.
"""
import ctypes
import os

import numpy as np

from . import build as _build

__all__ = ["SIFT_DTYPE", "lib", "set_tuning", "InitCuda", "CudaImage", "SiftData", "InitSiftData", "FreeSiftData",
           "AllocSiftTempMemory", "FreeSiftTempMemory", "ExtractSift", "MatchSiftData", "FindHomography", "Extractor",
           "CudaSiftError", "extract_host", "match_host", "rank_records", "MatchSiftDataMutual", "match_mutual_host",
           "match_knn2", "MatchSiftDataRatio", "match_ratio_host", "VerifyPairs", "verify_pairs_host", "verify_stats",
           "GEOM_MODELS"]

from .records import SIFT_DTYPE   # cudaSift.h:6-22 -- 576-byte record, descriptor at byte 64
assert SIFT_DTYPE.itemsize == 576


class CudaSiftError(RuntimeError):
    pass


_lib = None


def lib():
    """The loaded C-ABI library (built on first use when a toolkit is present)."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("CUDASIFT_B200_LIB") or _build.LIB     # override: kernel experiments (scripts/expbuild.sh)
    if not os.path.exists(path):
        path = _build.build_library()
    L = ctypes.CDLL(path)
    c = ctypes
    vp, ip, fp = c.c_void_p, c.c_int, c.c_float
    sig = {
        "cs_last_error": (c.c_char_p, []),
        "cs_version": (c.c_char_p, []),
        "cs_init": (ip, [ip]),
        "cs_launch_count": (c.c_ulonglong, []),
        "cs_set_tuning": (ip, [c.c_char_p, ip]),
        "cs_extract_launches_per_image": (ip, [ip, ip]),
        "cs_device_alloc": (vp, [c.c_size_t]),
        "cs_device_free": (ip, [vp]),
        "cs_memcpy_h2d": (ip, [vp, vp, c.c_size_t]),
        "cs_memcpy_d2h": (ip, [vp, vp, c.c_size_t]),
        "cs_memset_d": (ip, [vp, ip, c.c_size_t]),
        "cs_host_alloc_pinned": (vp, [c.c_size_t]),
        "cs_host_free_pinned": (ip, [vp]),
        "cs_device_sync": (ip, []),
        "cs_alloc_temp": (vp, [ip, ip, ip, ip]),
        "cs_free_temp": (ip, [vp]),
        "cs_temp_floats": (c.c_size_t, [ip, ip, ip, ip]),
        "cs_extract": (ip, [vp, ip, ip, ip, ip, c.c_double, fp, fp, ip, vp, vp, vp, ip]),
        "cs_extract_host": (ip, [vp, ip, ip, ip, c.c_double, fp, fp, ip, vp, ip]),
        "cs_match": (ip, [vp, ip, vp, ip, vp, ip, c.POINTER(c.c_double)]),
        "cs_match_host": (ip, [vp, ip, vp, ip, ip, c.POINTER(c.c_double)]),
        "cs_match_stats": (ip, [c.POINTER(c.c_ulonglong)]),
        "cs_match_mutual": (ip, [vp, ip, vp, ip, fp, fp, vp, ip, ip, c.POINTER(c.c_double)]),
        "cs_match_mutual_host": (ip, [vp, ip, vp, ip, fp, fp, vp, ip, ip, c.POINTER(c.c_double)]),
        "cs_match_knn2": (ip, [vp, ip, vp, ip, vp, vp, ip, c.POINTER(c.c_double)]),
        "cs_match_ratio": (ip, [vp, ip, vp, ip, fp, fp, ip, vp, ip, ip, c.POINTER(c.c_double)]),
        "cs_match_ratio_host": (ip, [vp, ip, vp, ip, fp, fp, ip, vp, ip, ip, c.POINTER(c.c_double)]),
        "cs_verify_pairs": (ip, [vp, ip, vp, ip, vp, ip, ip, ip, fp, c.c_ulonglong, vp, vp, ip, c.POINTER(c.c_double)]),
        "cs_verify_pairs_host": (ip, [vp, ip, vp, ip, vp, ip, ip, ip, fp, c.c_ulonglong, vp, vp, ip,
                                      c.POINTER(c.c_double)]),
        "cs_verify_stats": (ip, [c.POINTER(c.c_longlong)]),
        "cs_verify_models": (ip, [vp, ip, vp, ip, vp, ip, ip, ip, fp, c.c_ulonglong, vp, vp, vp]),
        "cs_find_homography": (ip, [vp, ip, vp, c.POINTER(c.c_int), ip, fp, fp, fp, c.POINTER(c.c_double)]),
        "cs_improve_homography": (ip, [vp, ip, vp, ip, fp, fp, fp, c.POINTER(c.c_int)]),
        "cs_lowpass": (ip, [vp, vp, ip, ip, ip, fp]),
        "cs_scaledown": (ip, [vp, vp, ip, ip, ip, ip]),
        "cs_scaleup": (ip, [vp, vp, ip, ip, ip, ip]),
        "cs_laplace_taps": (ip, [ip, fp, vp]),
        "cs_dog_planes": (ip, [vp, vp, ip, ip, ip, ip, ip]),
        "cs_tex_probe": (ip, [vp, ip, ip, ip, vp, vp, ip, vp]),
        "cs_describe_points": (ip, [vp, ip, ip, ip, vp, ip, ip, fp]),
        "cs_extractor_create": (vp, [ip, ip, ip, ip, ip]),
        "cs_extractor_destroy": (ip, [vp]),
        "cs_extractor_submit_device": (ip, [vp, vp, ip, c.c_double, fp, fp]),
        "cs_extractor_submit_host": (ip, [vp, vp, c.c_double, fp, fp]),
        "cs_extractor_submit_host_u8": (ip, [vp, vp, c.c_double, fp, fp]),
        "cs_extractor_wait": (ip, [vp]),
        "cs_event_create": (vp, []),
        "cs_event_destroy": (ip, [vp]),
        "cs_event_record": (ip, [vp, vp]),
        "cs_event_elapsed_ms": (c.c_double, [vp, vp]),
        "cs_extractor_profile": (ip, [vp, vp, ip, c.c_double, fp, fp, c.POINTER(c.c_float)]),
        "cs_max_batch": (ip, []),
        "cs_detector_items": (ip, [ip, ip, ip, ip, ip, ip, vp, ip]),
        "cs_extractor_create_batch": (vp, [ip, ip, ip, ip, ip, ip]),
        "cs_extractor_submit_device_batch": (ip, [vp, ip, vp, ip, c.c_double, fp, fp]),
        "cs_extractor_submit_host_batch": (ip, [vp, ip, vp, c.c_double, fp, fp]),
        "cs_extractor_wait_batch": (ip, [vp, vp]),
        "cs_extractor_count": (ip, [vp, ip]),
        "cs_extractor_device_points_at": (vp, [vp, ip]),
        "cs_extractor_host_points_at": (vp, [vp, ip]),
        "cs_extractor_host_image_at": (vp, [vp, ip]),
        "cs_extractor_profile_batch": (ip, [vp, ip, vp, ip, c.c_double, fp, fp, c.POINTER(c.c_float)]),
        "cs_extractor_read_level": (ip, [vp, ip, ip, vp]),
        "cs_extractor_device_points": (vp, [vp]),
        "cs_extractor_host_points": (vp, [vp]),
        "cs_extractor_host_image": (vp, [vp]),
        "cs_extractor_create_ranked": (vp, [ip, ip, ip, ip, ip, ip, ip]),
        "cs_extractor_candidates": (ip, [vp, ip]),
        "cs_rank_records": (ip, [vp, ip, vp, ip]),
    }
    for name, (res, args) in sig.items():
        f = getattr(L, name)
        f.restype, f.argtypes = res, args
    _lib = L
    return L


def _check(r, what):
    if r is None or (isinstance(r, int) and r < 0):
        raise CudaSiftError("%s failed: %s" % (what, lib().cs_last_error().decode()))
    return r


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def iAlignUp(a, b):
    return a if a % b == 0 else a - a % b + b


def InitCuda(devNum=0):
    """cudaSiftH.cu:19-37."""
    return _check(lib().cs_init(int(devNum)), "InitCuda")


class DeviceBuffer:
    """Raw device allocation (cudaMalloc) with host<->device copies."""

    def __init__(self, nbytes):
        self.nbytes = int(nbytes)
        self.ptr = _check(lib().cs_device_alloc(self.nbytes), "cudaMalloc")

    def upload(self, arr):
        arr = np.ascontiguousarray(arr)
        assert arr.nbytes <= self.nbytes
        _check(lib().cs_memcpy_h2d(self.ptr, _ptr(arr), arr.nbytes), "memcpy H2D")

    def download(self, dtype, count):
        out = np.empty(count, dtype=dtype)
        assert out.nbytes <= self.nbytes
        _check(lib().cs_memcpy_d2h(_ptr(out), self.ptr, out.nbytes), "memcpy D2H")
        return out

    def zero(self):
        _check(lib().cs_memset_d(self.ptr, 0, self.nbytes), "memset")

    def free(self):
        if self.ptr:
            lib().cs_device_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class CudaImage:
    """cudaImage.h:8-25: pitched float image on the device (+ optional host pixels)."""

    def __init__(self):
        self.width = self.height = self.pitch = 0
        self.h_data = None
        self._buf = None

    @property
    def d_data(self):
        return self._buf.ptr if self._buf else None

    def Allocate(self, width, height, pitch=None, withHost=False, devMem=None, hostMem=None):
        self.width, self.height = int(width), int(height)
        self.pitch = int(pitch) if pitch else iAlignUp(self.width, 128)
        self._buf = DeviceBuffer(self.pitch * self.height * 4)
        if hostMem is not None:
            self.h_data = np.ascontiguousarray(hostMem, dtype=np.float32).reshape(self.height, self.width)
        elif withHost:
            self.h_data = np.zeros((self.height, self.width), np.float32)
        return self

    def Download(self):
        padded = np.zeros((self.height, self.pitch), np.float32)
        padded[:, :self.width] = self.h_data
        self._buf.upload(padded)

    def Readback(self):
        a = self._buf.download(np.float32, self.pitch * self.height).reshape(self.height, self.pitch)
        self.h_data = a[:, :self.width].copy()
        return self.h_data

    def device_array(self):
        return self._buf.download(np.float32, self.pitch * self.height).reshape(self.height, self.pitch)


class SiftData:
    """cudaSift.h:24-33."""

    def __init__(self):
        self.numPts = 0
        self.maxPts = 0
        self.h_data = None
        self._buf = None

    @property
    def d_data(self):
        return self._buf.ptr if self._buf else None


def InitSiftData(data, num=1024, host=False, dev=True):
    """cudaSiftH.cu:234-249."""
    data.numPts, data.maxPts = 0, int(num)
    data.h_data = np.zeros(num, SIFT_DTYPE) if host else None
    data._buf = DeviceBuffer(num * SIFT_DTYPE.itemsize) if dev else None
    return data


def FreeSiftData(data):
    if data._buf:
        data._buf.free()
    data._buf, data.h_data, data.numPts, data.maxPts = None, None, 0, 0


def AllocSiftTempMemory(width, height, numOctaves, scaleUp=False):
    return _check(lib().cs_alloc_temp(width, height, numOctaves, int(scaleUp)), "AllocSiftTempMemory")


def FreeSiftTempMemory(ptr):
    lib().cs_free_temp(ptr)


def ExtractSift(siftData, img, numOctaves, initBlur, thresh, lowestScale=0.0, scaleUp=False, tempMemory=None):
    """cudaSiftH.cu:72-144; on return numPts, d_data and (if allocated) h_data are valid."""
    n = _check(lib().cs_extract(img.d_data, img.width, img.height, img.pitch, int(numOctaves), float(initBlur),
                                float(thresh), float(lowestScale), int(bool(scaleUp)), tempMemory, siftData.d_data,
                                _ptr(siftData.h_data) if siftData.h_data is not None else None, siftData.maxPts),
               "ExtractSift")
    siftData.numPts = n
    return n


def MatchSiftData(data1, data2, mode=0):
    """matching.cu:1090-1206; returns milliseconds."""
    ms = ctypes.c_double(0.0)
    _check(lib().cs_match(data1.d_data, data1.numPts, data2.d_data, data2.numPts,
                          _ptr(data1.h_data) if data1.h_data is not None else None, int(mode), ctypes.byref(ms)),
           "MatchSiftData")
    return ms.value


MATCH_FIELDS = ("score", "ambiguity", "match", "match_xpos", "match_ypos")


def MatchSiftDataMutual(data1, data2, minScore=0.0, maxAmbiguity=float("inf"), mode=0):
    """Both directions of MatchSiftData in one call, cross-checked (cs_match_mutual).  data1's match fields become
    those of MatchSiftData(data1, data2), data2's those of MatchSiftData(data2, data1); the h_data of a set that has
    one receives its five match fields.  Returns (pairs, ms): int32 [k, 2] rows (i, j) with data1 row i and data2
    row j each other's match, score > minScore and ambiguity < maxAmbiguity, in increasing i."""
    n1, n2 = data1.numPts, data2.numPts
    room = min(n1, n2)
    ms = ctypes.c_double(0.0)
    d_pairs = DeviceBuffer(max(room, 1) * 8)
    try:
        k = _check(lib().cs_match_mutual(data1.d_data, n1, data2.d_data, n2, float(minScore), float(maxAmbiguity),
                                         d_pairs.ptr if room else None, room, int(mode), ctypes.byref(ms)),
                   "MatchSiftDataMutual")
        pairs = d_pairs.download(np.int32, 2 * k).reshape(k, 2) if k else np.zeros((0, 2), np.int32)
    finally:
        d_pairs.free()
    for d, n in ((data1, n1), (data2, n2)):
        if d.h_data is not None and n:
            recs = d._buf.download(SIFT_DTYPE, n)
            for f in MATCH_FIELDS:
                d.h_data[f][:n] = recs[f]
    return pairs, ms.value


def match_knn2(s1, s2, mode=0):
    """The two nearest neighbours of every row of s1 among all rows of s2 (cs_match_knn2), on host record arrays.
    Returns (idx int32 [n1, 2], score float32 [n1, 2], ms): j1 is the lowest index with the largest positive score, j2
    the lowest other index with the largest remaining one; a missing neighbour is (-1, 0.0).  The records are only read."""
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE)
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE)
    n1, n2 = len(s1), len(s2)
    idx, score = np.full((n1, 2), -1, np.int32), np.zeros((n1, 2), np.float32)
    ms = ctypes.c_double(0.0)
    if n1 == 0 or n2 == 0:                   # no neighbours: nothing to compute
        return idx, score, ms.value
    bufs = [DeviceBuffer(s1.nbytes), DeviceBuffer(s2.nbytes), DeviceBuffer(idx.nbytes), DeviceBuffer(score.nbytes)]
    try:
        bufs[0].upload(s1)
        bufs[1].upload(s2)
        _check(lib().cs_match_knn2(bufs[0].ptr, n1, bufs[1].ptr, n2, bufs[2].ptr, bufs[3].ptr, int(mode), ctypes.byref(ms)),
               "cs_match_knn2")
        idx = bufs[2].download(np.int32, 2 * n1).reshape(n1, 2)
        score = bufs[3].download(np.float32, 2 * n1).reshape(n1, 2)
    finally:
        for b in bufs:
            b.free()
    return idx, score, ms.value


def MatchSiftDataRatio(data1, data2, maxRatio=0.8, maxDistance=0.7, crossCheck=True, mode=0):
    """Lowe's ratio test on the true two nearest neighbours (cs_match_ratio; the defaults are COLMAP's).  Returns
    (pairs, ms): int32 [k, 2] rows (i, j), data1 row i matched to data2 row j, in increasing i.  The records are only
    read."""
    n1, n2 = data1.numPts, data2.numPts
    room = min(n1, n2) if crossCheck else n1
    ms = ctypes.c_double(0.0)
    d_pairs = DeviceBuffer(max(room, 1) * 8)
    try:
        k = _check(lib().cs_match_ratio(data1.d_data, n1, data2.d_data, n2, float(maxRatio), float(maxDistance),
                                        int(bool(crossCheck)), d_pairs.ptr if room else None, room, int(mode),
                                        ctypes.byref(ms)), "MatchSiftDataRatio")
        pairs = d_pairs.download(np.int32, 2 * k).reshape(k, 2) if k else np.zeros((0, 2), np.int32)
    finally:
        d_pairs.free()
    return pairs, ms.value


def match_ratio_host(s1, s2, maxRatio=0.8, maxDistance=0.7, crossCheck=True, mode=0):
    """MatchSiftDataRatio on host record arrays (cs_match_ratio_host); returns (pairs[k, 2] int32, ms)."""
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE)
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE)
    pairs = np.zeros((min(len(s1), len(s2)) if crossCheck else len(s1), 2), np.int32)
    ms = ctypes.c_double(0.0)
    k = _check(lib().cs_match_ratio_host(_ptr(s1), len(s1), _ptr(s2), len(s2), float(maxRatio), float(maxDistance),
                                         int(bool(crossCheck)), _ptr(pairs), len(pairs), int(mode), ctypes.byref(ms)),
               "cs_match_ratio_host")
    return pairs[:k].copy(), ms.value


GEOM_MODELS = {"homography": 1, "fundamental": 2}     # CS_GEOM_HOMOGRAPHY, CS_GEOM_FUNDAMENTAL


def _geom_model(model):
    if isinstance(model, str):
        if model not in GEOM_MODELS:
            raise ValueError("model must be 'homography' or 'fundamental', not %r" % model)
        return GEOM_MODELS[model]
    return int(model)


def _pair_array(pairs):
    return np.ascontiguousarray(np.asarray(pairs, np.int32).reshape(-1, 2))


def VerifyPairs(data1, data2, pairs, model="fundamental", numLoops=4096, thresh=4.0, seed=0):
    """RANSAC verification of a correspondence list on the device (cs_verify_pairs): pairs is the int32 [k, 2] array of
    (data1 row, data2 row) that MatchSiftDataMutual and MatchSiftDataRatio return.  model: "fundamental" (7-point) or
    "homography" (4-point); thresh in pixels (COLMAP's max_error = 4 by default; Sampson error for F, transfer error
    for H).  Returns (model 3x3 float64 in pixel coordinates, inliers int32 [m, 2] in input order, ms)."""
    pairs = _pair_array(pairs)
    k = len(pairs)
    out = np.zeros(9, np.float64)
    ms = ctypes.c_double(0.0)
    bufs = [DeviceBuffer(max(k, 1) * 8), DeviceBuffer(max(k, 1) * 8)]
    try:
        if k:
            bufs[0].upload(pairs)
        m = _check(lib().cs_verify_pairs(data1.d_data, data1.numPts, data2.d_data, data2.numPts, bufs[0].ptr if k else None,
                                         k, _geom_model(model), int(numLoops), float(thresh), int(seed), _ptr(out),
                                         bufs[1].ptr if k else None, k, ctypes.byref(ms)), "VerifyPairs")
        inliers = bufs[1].download(np.int32, 2 * m).reshape(m, 2) if m else np.zeros((0, 2), np.int32)
    finally:
        for b in bufs:
            b.free()
    return out.reshape(3, 3), inliers, ms.value


def verify_pairs_host(s1, s2, pairs, model="fundamental", numLoops=4096, thresh=4.0, seed=0):
    """VerifyPairs on host record arrays (cs_verify_pairs_host); returns (model 3x3 float64, inliers [m, 2] int32, ms)."""
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE)
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE)
    pairs = _pair_array(pairs)
    out = np.zeros(9, np.float64)
    inliers = np.zeros((len(pairs), 2), np.int32)
    ms = ctypes.c_double(0.0)
    m = _check(lib().cs_verify_pairs_host(_ptr(s1), len(s1), _ptr(s2), len(s2), _ptr(pairs), len(pairs),
                                          _geom_model(model), int(numLoops), float(thresh), int(seed), _ptr(out),
                                          _ptr(inliers), len(inliers), ctypes.byref(ms)), "cs_verify_pairs_host")
    return out.reshape(3, 3), inliers[:m].copy(), ms.value


def verify_stats():
    """The last verify call: [valid pairs, invalid pairs, non-degenerate samples, models scored, winning slot
    (sample*3 + root, -1 if none), its inlier count, refit kept (0/1), final inlier count]."""
    out = (ctypes.c_longlong * 8)()
    _check(lib().cs_verify_stats(out), "cs_verify_stats")
    return list(out)


def FindHomography(data, numLoops=1000, minScore=0.85, maxAmbiguity=0.95, thresh=5.0, seed=None):
    """matching.cu:1000-1087; returns (3x3 homography, numMatches, ms).  seed: srand() value."""
    H = np.zeros(9, np.float32)
    n, ms = ctypes.c_int(0), ctypes.c_double(0.0)
    if seed is not None:
        ctypes.CDLL(None).srand(int(seed))
    _check(lib().cs_find_homography(data.d_data, data.numPts, _ptr(H), ctypes.byref(n), int(numLoops), float(minScore),
                                    float(maxAmbiguity), float(thresh), ctypes.byref(ms)), "FindHomography")
    return H.reshape(3, 3), n.value, ms.value


def ImproveHomography(records, homography, numLoops=5, minScore=0.0, maxAmbiguity=0.80, thresh=3.0):
    """geomFuncs.cpp:6-72 on a host record array (modified in place: match_error).  Returns
    (refined 3x3 homography, numFit).  Defaults are the demo's (mainSift.cpp:78)."""
    assert records.dtype == SIFT_DTYPE and records.flags.c_contiguous
    H = np.ascontiguousarray(np.asarray(homography, np.float32).reshape(9)).copy()
    n = ctypes.c_int(0)
    _check(lib().cs_improve_homography(_ptr(records), len(records), _ptr(H), int(numLoops), float(minScore),
                                       float(maxAmbiguity), float(thresh), ctypes.byref(n)), "ImproveHomography")
    return H.reshape(3, 3), n.value


def match_stats():
    out = (ctypes.c_ulonglong * 4)()
    _check(lib().cs_match_stats(out), "cs_match_stats")
    return list(out)


def extract_host(img, numOctaves=5, initBlur=1.0, thresh=3.0, lowestScale=0.0, scaleUp=False, maxPts=32768):
    """Download + ExtractSift + readback from a host float image; returns the records."""
    img = np.ascontiguousarray(img, np.float32)
    h, w = img.shape
    pts = np.zeros(maxPts, SIFT_DTYPE)
    n = _check(lib().cs_extract_host(_ptr(img), w, h, int(numOctaves), float(initBlur), float(thresh),
                                     float(lowestScale), int(bool(scaleUp)), _ptr(pts), maxPts), "cs_extract_host")
    return pts[:n].copy()


def match_host(s1, s2, mode=0):
    """MatchSiftData on host record arrays; returns (updated copy of s1, ms)."""
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE).copy()
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE)
    ms = ctypes.c_double(0.0)
    _check(lib().cs_match_host(_ptr(s1), len(s1), _ptr(s2), len(s2), int(mode), ctypes.byref(ms)), "cs_match_host")
    return s1, ms.value


def match_mutual_host(s1, s2, minScore=0.0, maxAmbiguity=float("inf"), mode=0):
    """MatchSiftDataMutual on host record arrays; returns (updated copy of s1, updated copy of s2, pairs[k, 2] int32,
    ms)."""
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE).copy()
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE).copy()
    pairs = np.zeros((min(len(s1), len(s2)), 2), np.int32)
    ms = ctypes.c_double(0.0)
    k = _check(lib().cs_match_mutual_host(_ptr(s1), len(s1), _ptr(s2), len(s2), float(minScore), float(maxAmbiguity),
                                          _ptr(pairs), len(pairs), int(mode), ctypes.byref(ms)), "cs_match_mutual_host")
    return s1, s2, pairs[:k].copy(), ms.value


def rank_records(records, n):
    """The ranking stage on host records: the min(n, len(records)) records with the largest |sharpness|, sorted by
    (|sharpness| descending, subsampling, ypos, xpos, scale, orientation); ranked on the device."""
    records = np.ascontiguousarray(records, SIFT_DTYPE)
    n = int(n)
    if n < 1:
        raise ValueError("n must be >= 1")
    if len(records) == 0:
        return records.copy()
    d_in, d_out = DeviceBuffer(records.nbytes), DeviceBuffer(min(n, len(records)) * SIFT_DTYPE.itemsize)
    try:
        d_in.upload(records)
        k = _check(lib().cs_rank_records(d_in.ptr, len(records), d_out.ptr, n), "cs_rank_records")
        return d_out.download(SIFT_DTYPE, k)
    finally:
        d_in.free()
        d_out.free()


def set_tuning(key, value):
    return _check(lib().cs_set_tuning(key.encode(), int(value)), "cs_set_tuning")


class Extractor:
    """Pipelined extractor (one CUDA stream + arena + result buffers for up to `batch` images per submit);
    see cudasift_b200.h.  maxCandidates=None: plain extractor (slot = the first maxPts records found, in no set
    order).  An integer >= maxPts: ranked extractor, each slot holds the maxPts records with the largest |sharpness|
    out of up to maxCandidates found, in a fixed order (cs_extractor_create_ranked)."""

    def __init__(self, width, height, numOctaves=5, maxPts=32768, scaleUp=False, batch=1, maxCandidates=None):
        self.handle = None
        self.w, self.h, self.maxPts, self.batch, self.maxCandidates = width, height, maxPts, batch, maxCandidates
        if maxCandidates is None:
            self.handle = _check(lib().cs_extractor_create_batch(width, height, numOctaves, maxPts, int(scaleUp), batch),
                                 "cs_extractor_create_batch")
        else:
            self.handle = _check(lib().cs_extractor_create_ranked(width, height, numOctaves, maxPts, int(scaleUp), batch,
                                                                  int(maxCandidates)), "cs_extractor_create_ranked")

    def candidates(self, slot):
        """Records found for image `slot` in the last wait; == maxCandidates: the candidate area overflowed."""
        return lib().cs_extractor_candidates(self.handle, slot)

    # ---- batches: one launch per stage for n images ----
    def submit_device_batch(self, d_imgs, pitch, initBlur=1.0, thresh=3.0, lowestScale=0.0):
        arr = (ctypes.c_void_p * len(d_imgs))(*d_imgs)
        _check(lib().cs_extractor_submit_device_batch(self.handle, len(d_imgs), arr, pitch, initBlur, thresh, lowestScale),
               "submit_device_batch")

    def submit_host_batch(self, h_img_ptrs, initBlur=1.0, thresh=3.0, lowestScale=0.0):
        arr = (ctypes.c_void_p * len(h_img_ptrs))(*h_img_ptrs)
        _check(lib().cs_extractor_submit_host_batch(self.handle, len(h_img_ptrs), arr, initBlur, thresh, lowestScale),
               "submit_host_batch")

    def wait_batch(self, n):
        counts = (ctypes.c_int * n)()
        _check(lib().cs_extractor_wait_batch(self.handle, counts), "wait_batch")
        return list(counts)

    def profile_batch(self, d_imgs, pitch, initBlur=1.0, thresh=3.0, lowestScale=0.0):
        arr = (ctypes.c_void_p * len(d_imgs))(*d_imgs)
        out = (ctypes.c_float * 5)()
        n = _check(lib().cs_extractor_profile_batch(self.handle, len(d_imgs), arr, pitch, initBlur, thresh, lowestScale, out),
                   "profile_batch")
        return n, list(out)

    def host_points_at(self, slot, n):
        p = lib().cs_extractor_host_points_at(self.handle, slot)
        buf = (ctypes.c_char * (n * SIFT_DTYPE.itemsize)).from_address(p)
        return np.frombuffer(buf, dtype=SIFT_DTYPE, count=n)

    def device_points_at(self, slot, n):
        """Copy of the first n records of image slot `slot` (device -> host)."""
        out = np.empty(n, SIFT_DTYPE)
        if n:
            _check(lib().cs_memcpy_d2h(_ptr(out), lib().cs_extractor_device_points_at(self.handle, slot), out.nbytes), "d2h")
        return out

    def read_level(self, slot, level):
        wh = _check(lib().cs_extractor_read_level(self.handle, slot, level, None), "read_level")
        w, h = wh & 0xffff, wh >> 16
        out = np.empty((h, w), np.float32)
        _check(lib().cs_extractor_read_level(self.handle, slot, level, _ptr(out)), "read_level")
        return out

    def host_image(self):
        p = lib().cs_extractor_host_image(self.handle)
        return np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctypes.c_float)), shape=(self.h, self.w))

    def submit_device(self, d_img, pitch, initBlur=1.0, thresh=3.0, lowestScale=0.0):
        _check(lib().cs_extractor_submit_device(self.handle, d_img, pitch, initBlur, thresh, lowestScale), "submit")

    def submit_host(self, h_img_ptr, initBlur=1.0, thresh=3.0, lowestScale=0.0):
        _check(lib().cs_extractor_submit_host(self.handle, h_img_ptr, initBlur, thresh, lowestScale), "submit")

    def submit_host_u8(self, h_img_ptr, initBlur=1.0, thresh=3.0, lowestScale=0.0):
        _check(lib().cs_extractor_submit_host_u8(self.handle, h_img_ptr, initBlur, thresh, lowestScale), "submit")

    def wait(self):
        return _check(lib().cs_extractor_wait(self.handle), "wait")

    def profile(self, d_img, pitch, initBlur=1.0, thresh=3.0, lowestScale=0.0):
        """(numPts, [ms LowPass, ScaleDown chain, detect, describe, total]) for one image."""
        out = (ctypes.c_float * 5)()
        n = _check(lib().cs_extractor_profile(self.handle, d_img, pitch, initBlur, thresh, lowestScale, out), "profile")
        return n, list(out)

    def host_points(self, n):
        p = lib().cs_extractor_host_points(self.handle)
        buf = (ctypes.c_char * (n * SIFT_DTYPE.itemsize)).from_address(p)
        return np.frombuffer(buf, dtype=SIFT_DTYPE, count=n)

    def device_points(self):
        return lib().cs_extractor_device_points(self.handle)

    def close(self):
        if self.handle:
            lib().cs_extractor_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
