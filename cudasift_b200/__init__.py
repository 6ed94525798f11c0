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
           "GEOM_MODELS", "match_knn2_guided", "MatchSiftDataGuided", "match_guided_host", "guided_stats",
           "VerifyEssential", "verify_essential_host", "essential_stats", "essential_to_fundamental", "VerifyJob",
           "VerifyPairsBatch", "VerifyEssentialBatch", "MatchSet", "MatchJob", "MatchSiftDataRatioBatch",
           "MatchSiftDataGuidedBatch", "TrackList", "BuildTracks", "TriangulateTracks", "PoseJob", "AbsolutePoseBatch",
           "BundleAdjust", "BundleAdjustIntrinsics", "UndistortRecords", "TrainVocabulary", "AssignWords",
           "RetrievePairs", "RotationAveraging", "GlobalPositioning", "UndistortImages", "PatchMatchStereo",
           "PatchMatchStereoGeometric", "FuseDepthMaps", "SelectStereoViews", "PoissonMesh",
           "PoissonMeshScreened", "SimplifyMesh", "RefineMesh", "CleanMesh"]

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
    path = os.environ.get("CUDASIFT_B200_LIB") or _build.LIB     # override: a library built some other way
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
        "cs_match_knn2_guided": (ip, [vp, ip, vp, ip, ip, vp, fp, vp, vp, c.POINTER(c.c_double)]),
        "cs_match_guided": (ip, [vp, ip, vp, ip, ip, vp, fp, fp, fp, ip, vp, ip, c.POINTER(c.c_double)]),
        "cs_match_guided_host": (ip, [vp, ip, vp, ip, ip, vp, fp, fp, fp, ip, vp, ip, c.POINTER(c.c_double)]),
        "cs_match_guided_stats": (ip, [c.POINTER(c.c_ulonglong)]),
        "cs_verify_models": (ip, [vp, ip, vp, ip, vp, ip, ip, ip, fp, c.c_ulonglong, vp, vp, vp]),
        "cs_verify_essential": (ip, [vp, ip, vp, ip, vp, ip, vp, vp, ip, fp, c.c_ulonglong, vp, vp, vp, vp, ip,
                                     c.POINTER(c.c_double)]),
        "cs_verify_essential_host": (ip, [vp, ip, vp, ip, vp, ip, vp, vp, ip, fp, c.c_ulonglong, vp, vp, vp, vp, ip,
                                          c.POINTER(c.c_double)]),
        "cs_verify_essential_stats": (ip, [c.POINTER(c.c_longlong)]),
        "cs_verify_essential_models": (ip, [vp, ip, vp, ip, vp, ip, vp, vp, ip, fp, c.c_ulonglong, vp, vp, vp]),
        "cs_verify_pairs_batch": (ip, [vp, ip, ip, ip, fp, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_verify_essential_batch": (ip, [vp, ip, vp, vp, ip, fp, vp, vp, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_match_ratio_batch": (ip, [vp, ip, vp, ip, fp, fp, ip, vp, vp, c.POINTER(c.c_double)]),
        "cs_match_guided_batch": (ip, [vp, ip, vp, ip, vp, vp, fp, fp, fp, ip, vp, vp, c.POINTER(c.c_double)]),
        "cs_build_tracks": (ip, [vp, ip, vp, ip, ip, ip, vp, vp, ip, vp, ip, vp, c.POINTER(c.c_double)]),
        "cs_vocab_assign": (ip, [vp, ip, vp, ip, vp, vp, c.POINTER(c.c_double)]),
        "cs_vocab_train": (ip, [vp, ip, ip, ip, c.c_ulonglong, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_retrieve_pairs": (ip, [vp, ip, vp, ip, ip, vp, vp, vp, vp, ip, vp, c.POINTER(c.c_double)]),
        "cs_triangulate_tracks": (ip, [vp, ip, vp, vp, vp, vp, ip, vp, ip, ip, c.c_double, c.c_double, c.c_ulonglong,
                                       vp, vp, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_bundle_adjust": (ip, [vp, ip, vp, vp, vp, vp, vp, ip, vp, ip, vp, vp, ip, ip, c.c_double, c.c_double,
                                  vp, vp, vp, vp, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_bundle_adjust_intrinsics": (ip, [vp, ip, vp, vp, vp, ip, c.c_double, vp, vp, vp, vp, ip, vp, ip, vp, vp,
                                             ip, ip, c.c_double, c.c_double, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                             c.POINTER(c.c_double)]),
        "cs_undistort_records": (ip, [vp, ip, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_global_positioning": (ip, [vp, ip, vp, vp, vp, ip, vp, ip, vp, ip, c.c_ulonglong, ip, c.c_double, ip, ip,
                                       c.c_double, vp, vp, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_rotation_averaging": (ip, [ip, vp, ip, vp, vp, ip, ip, ip, c.c_double, c.c_double, c.c_double, vp, vp, vp,
                                       vp, vp, vp, vp]),
        "cs_undistort_images": (ip, [vp, ip, vp, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_patch_match_stereo": (ip, [vp, ip, vp, vp, vp, vp, ip, ip, ip, ip, ip, c.c_ulonglong, vp,
                                       c.POINTER(c.c_double)]),
        "cs_patch_match_stereo_geometric": (ip, [vp, ip, vp, vp, vp, vp, vp, ip, ip, ip, ip, ip, c.c_double,
                                                 c.c_double, c.c_ulonglong, vp, c.POINTER(c.c_double)]),
        "cs_fuse_depth_maps": (ip, [vp, ip, vp, vp, vp, vp, ip, fp, ip, c.c_double, c.c_double, c.c_double, vp, vp, vp,
                                    vp, ip, vp, c.POINTER(c.c_double)]),
        "cs_poisson_mesh": (ip, [vp, vp, vp, ip, ip, c.c_double, ip, c.c_double, c.c_double, vp, vp, ip, vp, ip, vp,
                                 vp, vp, c.POINTER(c.c_double)]),
        "cs_poisson_mesh_screened": (ip, [vp, vp, vp, ip, ip, c.c_double, c.c_double, ip, c.c_double, c.c_double, vp,
                                          vp, ip, vp, ip, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_simplify_mesh": (ip, [vp, vp, ip, vp, ip, ip, c.c_double, c.c_double, vp, vp, ip, vp, ip, vp, vp,
                                  c.POINTER(c.c_double)]),
        "cs_clean_mesh": (ip, [vp, vp, ip, vp, ip, ip, c.c_double, ip, ip, c.c_double, ip, ip, c.c_double, c.c_double,
                               vp, vp, ip, vp, ip, vp, vp, c.POINTER(c.c_double)]),
        "cs_texture_mesh": (ip, [vp, ip, vp, vp, vp, vp, ip, vp, ip, c.c_double, c.c_double, c.c_double, ip, ip, ip,
                                 vp, ip, vp, vp, vp, vp, ip, vp, vp, c.POINTER(c.c_double)]),
        "cs_texture_mesh_photo": (ip, [vp, ip, vp, vp, vp, vp, ip, vp, ip, ip, c.c_double, c.c_double, c.c_double,
                                       c.c_double, c.c_double, ip, ip, ip, vp, ip, vp, vp, vp, vp, ip, vp, vp,
                                       c.POINTER(c.c_double)]),
        "cs_texture_mesh_bp": (ip, [vp, ip, vp, vp, vp, vp, ip, vp, ip, ip, c.c_double, c.c_double, ip, c.c_double,
                                    c.c_double, c.c_double, ip, ip, ip, vp, ip, vp, vp, vp, vp, ip, vp, vp,
                                    c.POINTER(c.c_double)]),
        "cs_mesh_refine": (ip, [vp, ip, vp, vp, vp, vp, ip, vp, ip, vp, ip, ip, c.c_double, c.c_double, ip,
                                c.c_double, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_level_texture_seams": (ip, [vp, ip, vp, ip, vp, vp, vp, ip, vp, ip, ip, ip, c.c_double, c.c_double, ip,
                                        c.c_double, vp, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_level_texture_seams_local": (ip, [vp, ip, vp, ip, vp, vp, vp, ip, vp, ip, ip, ip, ip, ip, c.c_double, vp,
                                              vp, vp, c.POINTER(c.c_double)]),
        "cs_absolute_pose_batch": (ip, [vp, ip, vp, ip, vp, ip, c.c_double, vp, vp, vp, vp, c.POINTER(c.c_double)]),
        "cs_absolute_pose_models": (ip, [vp, ip, vp, vp, ip, c.c_double, vp, vp, vp]),
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


class MatchSet(ctypes.Structure):
    """cs_match_set: one image's device records in a batched ratio match."""
    _fields_ = [("pts", ctypes.c_void_p), ("n", ctypes.c_int)]


class MatchJob(ctypes.Structure):
    """cs_match_job: two set indices and the job's device pair buffer."""
    _fields_ = [("set1", ctypes.c_int), ("set2", ctypes.c_int), ("pairs", ctypes.c_void_p), ("maxPairs", ctypes.c_int)]


def _match_batch(datas, jobs, crossCheck, call):
    """The set and job tables of a batched match over SiftData datas and (a, b) jobs, every pair list in one device
    buffer with room for each job's largest count; call(sets, numSets, jobs, numJobs, counts, stats, ms) runs the
    batch.  Returns (pairs: a list of int32 [k, 2], stats uint64 [J, 4], ms)."""
    sets = (MatchSet * max(len(datas), 1))()
    for s, d in enumerate(datas):
        sets[s] = MatchSet(d.d_data, d.numPts)
    rooms = []
    for a, b in jobs:
        n1, n2 = datas[a].numPts, datas[b].numPts
        rooms.append(min(n1, n2) if crossCheck else n1)
    offsets = np.concatenate([[0], np.cumsum(rooms, dtype=np.int64)]).astype(np.int64)
    total = int(offsets[-1])
    J = len(jobs)
    counts, stats = np.zeros(J, np.int32), np.zeros((J, 4), np.uint64)
    ms = ctypes.c_double(0.0)
    buf = DeviceBuffer(max(total, 1) * 8)
    try:
        table = (MatchJob * max(J, 1))()
        for q, (a, b) in enumerate(jobs):
            table[q] = MatchJob(int(a), int(b), buf.ptr + 8 * int(offsets[q]) if rooms[q] else None, rooms[q])
        call(ctypes.addressof(sets) if datas else None, len(datas), ctypes.addressof(table) if J else None, J,
             _ptr(counts), _ptr(stats), ctypes.byref(ms))
        flat = buf.download(np.int32, 2 * total).reshape(-1, 2) if total else np.zeros((0, 2), np.int32)
    finally:
        buf.free()
    pairs = [flat[offsets[q]:offsets[q] + int(counts[q])].copy() for q in range(J)]
    return pairs, stats, ms.value


def MatchSiftDataRatioBatch(datas, jobs, maxRatio=0.8, maxDistance=0.7, crossCheck=True):
    """MatchSiftDataRatio over many image pairs in one call (cs_match_ratio_batch): datas is a list of SiftData, jobs a
    list of (a, b) indices into it.  Job p's pairs equal MatchSiftDataRatio(datas[a], datas[b], maxRatio, maxDistance,
    crossCheck) bit for bit.  Every pair list lives in one device buffer, room for each job's largest count.  Returns
    (pairs: a list of int32 [k, 2], stats uint64 [J, 4] as match_stats after a mode-2 call, ms)."""
    def call(sets, S, table, J, counts, stats, ms):
        _check(lib().cs_match_ratio_batch(sets, S, table, J, float(maxRatio), float(maxDistance), int(bool(crossCheck)),
                                          counts, stats, ms), "MatchSiftDataRatioBatch")
    return _match_batch(datas, jobs, crossCheck, call)


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


def _verify_device(pairs, call):
    """The shared path of VerifyPairs and VerifyEssential: the pairs in one device buffer, room for as many inliers in
    another; call(d_pairs, k, d_inliers) makes the library call and returns the inlier count.  Returns the inliers,
    int32 [m, 2]."""
    k = len(pairs)
    bufs = [DeviceBuffer(max(k, 1) * 8), DeviceBuffer(max(k, 1) * 8)]
    try:
        if k:
            bufs[0].upload(pairs)
        m = call(bufs[0].ptr if k else None, k, bufs[1].ptr if k else None)
        return bufs[1].download(np.int32, 2 * m).reshape(m, 2) if m else np.zeros((0, 2), np.int32)
    finally:
        for b in bufs:
            b.free()


def _verify_host(s1, s2, pairs, call):
    """The shared path of verify_pairs_host and verify_essential_host: contiguous records and pairs, room for every pair
    as an inlier; call(s1, s2, pairs, inliers) makes the library call and returns the inlier count.  Returns the
    inliers, int32 [m, 2]."""
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE)
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE)
    pairs = _pair_array(pairs)
    inliers = np.zeros((len(pairs), 2), np.int32)
    m = call(s1, s2, pairs, inliers)
    return inliers[:m].copy()


def VerifyPairs(data1, data2, pairs, model="fundamental", numLoops=4096, thresh=4.0, seed=0):
    """RANSAC verification of a correspondence list on the device (cs_verify_pairs): pairs is the int32 [k, 2] array of
    (data1 row, data2 row) that MatchSiftDataMutual and MatchSiftDataRatio return.  model: "fundamental" (7-point) or
    "homography" (4-point); thresh in pixels (COLMAP's max_error = 4 by default; Sampson error for F, transfer error
    for H).  Returns (model 3x3 float64 in pixel coordinates, inliers int32 [m, 2] in input order, ms)."""
    out = np.zeros(9, np.float64)
    ms = ctypes.c_double(0.0)
    inliers = _verify_device(_pair_array(pairs), lambda d_pairs, k, d_inliers: _check(lib().cs_verify_pairs(
        data1.d_data, data1.numPts, data2.d_data, data2.numPts, d_pairs, k, _geom_model(model), int(numLoops),
        float(thresh), int(seed), _ptr(out), d_inliers, k, ctypes.byref(ms)), "VerifyPairs"))
    return out.reshape(3, 3), inliers, ms.value


def verify_pairs_host(s1, s2, pairs, model="fundamental", numLoops=4096, thresh=4.0, seed=0):
    """VerifyPairs on host record arrays (cs_verify_pairs_host); returns (model 3x3 float64, inliers [m, 2] int32, ms)."""
    out = np.zeros(9, np.float64)
    ms = ctypes.c_double(0.0)
    inliers = _verify_host(s1, s2, pairs, lambda s1, s2, pairs, inliers: _check(lib().cs_verify_pairs_host(
        _ptr(s1), len(s1), _ptr(s2), len(s2), _ptr(pairs), len(pairs), _geom_model(model), int(numLoops),
        float(thresh), int(seed), _ptr(out), _ptr(inliers), len(inliers), ctypes.byref(ms)), "cs_verify_pairs_host"))
    return out.reshape(3, 3), inliers, ms.value


def verify_stats():
    """The last verify call: [valid pairs, invalid pairs, non-degenerate samples, models scored, winning slot
    (sample*3 + root, -1 if none), its inlier count, refit kept (0/1), final inlier count]."""
    out = (ctypes.c_longlong * 8)()
    _check(lib().cs_verify_stats(out), "cs_verify_stats")
    return list(out)


def _intrinsics(K):
    return np.ascontiguousarray(np.asarray(K, np.float64).reshape(9))


class VerifyJob(ctypes.Structure):
    """cs_verify_job: one image pair of a batched verification (device records, pairs and inlier buffer)."""
    _fields_ = [("s1", ctypes.c_void_p), ("n1", ctypes.c_int), ("s2", ctypes.c_void_p), ("n2", ctypes.c_int),
                ("pairs", ctypes.c_void_p), ("numPairs", ctypes.c_int), ("seed", ctypes.c_ulonglong),
                ("inliers", ctypes.c_void_p), ("maxInliers", ctypes.c_int)]


class _BatchJobs:
    """The job table of a batch call for [(data1, data2, pairs) or (data1, data2, pairs, seed)]: every pair list in one
    device buffer and every inlier list in another, each job's pointers into them (room for all its pairs)."""

    def __init__(self, jobs):
        parsed = []
        for j in jobs:
            if len(j) not in (3, 4):
                raise ValueError("a job is (data1, data2, pairs) or (data1, data2, pairs, seed)")
            parsed.append((j[0], j[1], _pair_array(j[2]), int(j[3]) if len(j) == 4 else 0))
        self.sizes = [len(p[2]) for p in parsed]
        self.offsets = np.concatenate([[0], np.cumsum(self.sizes, dtype=np.int64)]).astype(np.int64)
        total = int(self.offsets[-1])
        self.bufs = [DeviceBuffer(max(total, 1) * 8), DeviceBuffer(max(total, 1) * 8)]
        if total:
            self.bufs[0].upload(np.concatenate([p[2] for p in parsed]))
        self.table = (VerifyJob * max(len(parsed), 1))()
        for q, (d1, d2, pairs, seed) in enumerate(parsed):
            k, o = self.sizes[q], 8 * int(self.offsets[q])
            self.table[q] = VerifyJob(d1.d_data, d1.numPts, d2.d_data, d2.numPts, self.bufs[0].ptr + o if k else None, k,
                                      seed, self.bufs[1].ptr + o if k else None, k)
        self.count = len(parsed)

    def ptr(self):
        return ctypes.addressof(self.table) if self.count else None

    def inliers(self, counts):
        """Each job's inlier list, int32 [m, 2], from the shared inlier buffer."""
        total = int(self.offsets[-1])
        flat = self.bufs[1].download(np.int32, 2 * total).reshape(-1, 2) if total else np.zeros((0, 2), np.int32)
        return [flat[self.offsets[q]:self.offsets[q] + int(counts[q])].copy() for q in range(self.count)]

    def free(self):
        for b in self.bufs:
            b.free()


def VerifyPairsBatch(jobs, model="fundamental", numLoops=4096, thresh=4.0):
    """VerifyPairs over many image pairs in one call (cs_verify_pairs_batch): jobs is a list of (data1, data2, pairs)
    or (data1, data2, pairs, seed), the seed 0 when not given; model, numLoops and thresh are common.  Job p's results
    equal VerifyPairs(data1, data2, pairs, model, numLoops, thresh, seed) bit for bit.  Returns (models [J, 3, 3]
    float64, inliers: a list of int32 [m, 2], stats int64 [J, 8] as verify_stats, ms)."""
    code = _geom_model(model)
    J = len(jobs)
    models, counts, stats = np.zeros((J, 9)), np.zeros(J, np.int32), np.zeros((J, 8), np.int64)
    ms = ctypes.c_double(0.0)
    b = _BatchJobs(jobs)
    try:
        _check(lib().cs_verify_pairs_batch(b.ptr(), J, code, int(numLoops), float(thresh), _ptr(models), _ptr(counts),
                                           _ptr(stats), ctypes.byref(ms)), "VerifyPairsBatch")
        inliers = b.inliers(counts)
    finally:
        b.free()
    return models.reshape(J, 3, 3), inliers, stats, ms.value


def VerifyEssentialBatch(jobs, K1s, K2s, numLoops=4096, thresh=4.0):
    """VerifyEssential over many image pairs in one call (cs_verify_essential_batch): jobs as for VerifyPairsBatch,
    K1s and K2s the intrinsics per job ([J, 3, 3], or one 3x3 for all jobs).  Job p's results equal
    VerifyEssential(data1, data2, pairs, K1s[p], K2s[p], numLoops, thresh, seed) bit for bit.  Returns (E [J, 3, 3],
    R [J, 3, 3], t [J, 3], inliers: a list of int32 [m, 2], stats int64 [J, 10] as essential_stats, ms)."""
    J = len(jobs)
    k1 = np.ascontiguousarray(np.broadcast_to(np.asarray(K1s, np.float64).reshape(-1, 9), (J, 9)))
    k2 = np.ascontiguousarray(np.broadcast_to(np.asarray(K2s, np.float64).reshape(-1, 9), (J, 9)))
    E, R, t = np.zeros((J, 9)), np.zeros((J, 9)), np.zeros((J, 3))
    counts, stats = np.zeros(J, np.int32), np.zeros((J, 10), np.int64)
    ms = ctypes.c_double(0.0)
    b = _BatchJobs(jobs)
    try:
        _check(lib().cs_verify_essential_batch(b.ptr(), J, _ptr(k1), _ptr(k2), int(numLoops), float(thresh), _ptr(E),
                                               _ptr(R), _ptr(t), _ptr(counts), _ptr(stats), ctypes.byref(ms)),
               "VerifyEssentialBatch")
        inliers = b.inliers(counts)
    finally:
        b.free()
    return E.reshape(J, 3, 3), R.reshape(J, 3, 3), t, inliers, stats, ms.value


def VerifyEssential(data1, data2, pairs, K1, K2, numLoops=4096, thresh=4.0, seed=0):
    """Calibrated verification on the device (cs_verify_essential): RANSAC for the essential matrix with the 5-point
    solver, then the relative pose.  pairs as for VerifyPairs; K1, K2 the 3x3 pinhole intrinsics of the two images
    (skew allowed); thresh in pixels (the Sampson error of F = K2^-T E K1^-1, as VerifyPairs' "fundamental").
    Returns (E 3x3, R 3x3, t [3], inliers int32 [m, 2] in input order, ms): E at unit Frobenius norm, X2 = R X1 + t
    with |t| = 1."""
    E, R, t = np.zeros(9), np.zeros(9), np.zeros(3)
    k1, k2 = _intrinsics(K1), _intrinsics(K2)
    ms = ctypes.c_double(0.0)
    inliers = _verify_device(_pair_array(pairs), lambda d_pairs, k, d_inliers: _check(lib().cs_verify_essential(
        data1.d_data, data1.numPts, data2.d_data, data2.numPts, d_pairs, k, _ptr(k1), _ptr(k2), int(numLoops),
        float(thresh), int(seed), _ptr(E), _ptr(R), _ptr(t), d_inliers, k, ctypes.byref(ms)), "VerifyEssential"))
    return E.reshape(3, 3), R.reshape(3, 3), t, inliers, ms.value


def verify_essential_host(s1, s2, pairs, K1, K2, numLoops=4096, thresh=4.0, seed=0):
    """VerifyEssential on host record arrays (cs_verify_essential_host); returns (E, R, t, inliers [m, 2] int32, ms)."""
    E, R, t = np.zeros(9), np.zeros(9), np.zeros(3)
    k1, k2 = _intrinsics(K1), _intrinsics(K2)
    ms = ctypes.c_double(0.0)
    inliers = _verify_host(s1, s2, pairs, lambda s1, s2, pairs, inliers: _check(lib().cs_verify_essential_host(
        _ptr(s1), len(s1), _ptr(s2), len(s2), _ptr(pairs), len(pairs), _ptr(k1), _ptr(k2), int(numLoops),
        float(thresh), int(seed), _ptr(E), _ptr(R), _ptr(t), _ptr(inliers), len(inliers), ctypes.byref(ms)),
        "cs_verify_essential_host"))
    return E.reshape(3, 3), R.reshape(3, 3), t, inliers, ms.value


def essential_stats():
    """The last essential call: the eight fields of verify_stats (winning slot sample*10 + root), then the final
    inliers in front of the chosen pose and the runner-up pose candidate's count."""
    out = (ctypes.c_longlong * 10)()
    _check(lib().cs_verify_essential_stats(out), "cs_verify_essential_stats")
    return list(out)


def essential_to_fundamental(E, K1, K2):
    """F = K2^-T E K1^-1 at unit Frobenius norm with its largest-magnitude entry positive: the pixel model of an
    essential matrix, for MatchSiftDataGuided(..., "fundamental", F)."""
    E = np.asarray(E, np.float64).reshape(3, 3)
    K1, K2 = np.asarray(K1, np.float64).reshape(3, 3), np.asarray(K2, np.float64).reshape(3, 3)
    F = np.linalg.inv(K2).T @ E @ np.linalg.inv(K1)
    n = np.linalg.norm(F)
    if not n > 0:
        return np.zeros((3, 3))
    flat = F.reshape(-1)
    return F * (np.copysign(1.0, flat[int(np.argmax(np.abs(flat)))]) / n)


def _guided_model(M):
    return np.ascontiguousarray(np.asarray(M, np.float64).reshape(9))


def match_knn2_guided(s1, s2, model, M, thresh=4.0):
    """Guided two nearest neighbours (cs_match_knn2_guided) on host record arrays: match_knn2, with row i of s1 only
    considering the rows j of s2 that the model M (3x3, set-1 pixels to set-2 pixels, as VerifyPairs returns it)
    admits within thresh pixels (Sampson error for "fundamental", forward transfer error for "homography").  Returns
    (idx int32 [n1, 2], score float32 [n1, 2], ms)."""
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE)
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE)
    n1, n2 = len(s1), len(s2)
    m = _guided_model(M)
    idx, score = np.full((n1, 2), -1, np.int32), np.zeros((n1, 2), np.float32)
    ms = ctypes.c_double(0.0)
    if n1 == 0 or n2 == 0:
        _check(lib().cs_match_knn2_guided(None, 0, None, 0, _geom_model(model), _ptr(m), float(thresh), None, None,
                                          None), "cs_match_knn2_guided")
        return idx, score, ms.value
    bufs = [DeviceBuffer(s1.nbytes), DeviceBuffer(s2.nbytes), DeviceBuffer(idx.nbytes), DeviceBuffer(score.nbytes)]
    try:
        bufs[0].upload(s1)
        bufs[1].upload(s2)
        _check(lib().cs_match_knn2_guided(bufs[0].ptr, n1, bufs[1].ptr, n2, _geom_model(model), _ptr(m), float(thresh),
                                          bufs[2].ptr, bufs[3].ptr, ctypes.byref(ms)), "cs_match_knn2_guided")
        idx = bufs[2].download(np.int32, 2 * n1).reshape(n1, 2)
        score = bufs[3].download(np.float32, 2 * n1).reshape(n1, 2)
    finally:
        for b in bufs:
            b.free()
    return idx, score, ms.value


def MatchSiftDataGuided(data1, data2, model, M, thresh=4.0, maxRatio=0.8, maxDistance=0.7, crossCheck=True):
    """Guided matching (cs_match_guided, COLMAP's guided_matching): MatchSiftDataRatio restricted to the pairs the model
    M admits within thresh pixels; model and M as VerifyPairs returns them.  Returns (pairs int32 [k, 2], ms)."""
    n1, n2 = data1.numPts, data2.numPts
    m = _guided_model(M)
    room = min(n1, n2) if crossCheck else n1
    ms = ctypes.c_double(0.0)
    d_pairs = DeviceBuffer(max(room, 1) * 8)
    try:
        k = _check(lib().cs_match_guided(data1.d_data, n1, data2.d_data, n2, _geom_model(model), _ptr(m), float(thresh),
                                         float(maxRatio), float(maxDistance), int(bool(crossCheck)),
                                         d_pairs.ptr if room else None, room, ctypes.byref(ms)), "MatchSiftDataGuided")
        pairs = d_pairs.download(np.int32, 2 * k).reshape(k, 2) if k else np.zeros((0, 2), np.int32)
    finally:
        d_pairs.free()
    return pairs, ms.value


def match_guided_host(s1, s2, model, M, thresh=4.0, maxRatio=0.8, maxDistance=0.7, crossCheck=True):
    """MatchSiftDataGuided on host record arrays (cs_match_guided_host); returns (pairs[k, 2] int32, ms)."""
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE)
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE)
    m = _guided_model(M)
    pairs = np.zeros((min(len(s1), len(s2)) if crossCheck else len(s1), 2), np.int32)
    ms = ctypes.c_double(0.0)
    k = _check(lib().cs_match_guided_host(_ptr(s1), len(s1), _ptr(s2), len(s2), _geom_model(model), _ptr(m),
                                          float(thresh), float(maxRatio), float(maxDistance), int(bool(crossCheck)),
                                          _ptr(pairs), len(pairs), ctypes.byref(ms)), "cs_match_guided_host")
    return pairs[:k].copy(), ms.value


def guided_stats():
    """The last guided call: [predicate evaluations, admissible pairs (exact chains run), rows of set 1 with an
    admissible candidate, the same for set 2 in a cross-checked call (else 0)]."""
    out = (ctypes.c_ulonglong * 4)()
    _check(lib().cs_match_guided_stats(out), "cs_match_guided_stats")
    return list(out)


def MatchSiftDataGuidedBatch(datas, jobs, model, Ms, thresh=4.0, maxRatio=0.8, maxDistance=0.7, crossCheck=True):
    """MatchSiftDataGuided over many image pairs in one call (cs_match_guided_batch): datas and jobs as for
    MatchSiftDataRatioBatch; model one name or code for every job, or a list with one per job; Ms [J, 3, 3], for example
    the models VerifyPairsBatch returns (leave out the jobs whose verification failed: a zero model is an error).  Job
    p's pairs equal MatchSiftDataGuided(datas[a], datas[b], model[p], Ms[p], thresh, maxRatio, maxDistance, crossCheck)
    bit for bit.  Returns (pairs: a list of int32 [k, 2], stats uint64 [J, 4] as guided_stats after that call, ms)."""
    J = len(jobs)
    names = list(model) if isinstance(model, (list, tuple, np.ndarray)) else [model] * J
    if len(names) != J:
        raise ValueError("model: one for every job, or a list of %d, not %d" % (J, len(names)))
    codes = np.array([_geom_model(m) for m in names], np.int32)
    m = np.ascontiguousarray(np.asarray(Ms, np.float64).reshape(J, 9))

    def call(sets, S, table, J, counts, stats, ms):
        _check(lib().cs_match_guided_batch(sets, S, table, J, _ptr(codes), _ptr(m), float(thresh), float(maxRatio),
                                           float(maxDistance), int(bool(crossCheck)), counts, stats, ms),
               "MatchSiftDataGuidedBatch")
    return _match_batch(datas, jobs, crossCheck, call)


class TrackList(ctypes.Structure):
    """cs_track_list: the device pair list of one image pair, for BuildTracks."""
    _fields_ = [("image1", ctypes.c_int), ("image2", ctypes.c_int), ("pairs", ctypes.c_void_p),
                ("numPairs", ctypes.c_int)]


def BuildTracks(imageSizes, lists, minLength=2, dropConflicting=True):
    """Feature tracks over many image pairs in one call (cs_build_tracks): imageSizes[a] is the feature count of image
    a, lists a sequence of (a, b, pairs) with pairs int32 [k, 2] of {feature of a, feature of b}, for example
    zip(jobs, pairs) from MatchSiftDataGuidedBatch or MatchSiftDataRatioBatch.  The lists go up in one device buffer;
    the outputs are sized from the pair count (no track has fewer than minLength of the at most 2 k features the
    pairs touch), so one call returns them whole.  Returns (offsets int32 [T + 1], members int32 [M, 2] of {image,
    feature}, trackOf int32 [N], stats int64 [8] as the header describes them, ms)."""
    sizes = np.ascontiguousarray(np.asarray(imageSizes, np.int64).reshape(-1).astype(np.int32))
    parsed = [(int(a), int(b), _pair_array(p)) for a, b, p in lists]
    counts = [len(p) for _, _, p in parsed]
    offs = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int64)
    P, N = int(offs[-1]), int(sizes.sum(dtype=np.int64))
    maxMembers = min(N, 2 * P)
    maxTracks = maxMembers // max(int(minLength), 2)
    table = (TrackList * max(len(parsed), 1))()
    stats, ms = np.zeros(8, np.int64), ctypes.c_double(0.0)
    bufs = [DeviceBuffer(max(P, 1) * 8), DeviceBuffer(max(N, 1) * 4), DeviceBuffer((maxTracks + 1) * 4),
            DeviceBuffer(max(maxMembers, 1) * 8)]
    try:
        if P:
            bufs[0].upload(np.concatenate([p for _, _, p in parsed]))
        for q, (a, b, p) in enumerate(parsed):
            table[q] = TrackList(a, b, bufs[0].ptr + 8 * int(offs[q]) if counts[q] else None, counts[q])
        T = _check(lib().cs_build_tracks(_ptr(sizes), len(sizes), ctypes.addressof(table) if parsed else None,
                                         len(parsed), int(minLength), int(bool(dropConflicting)),
                                         bufs[1].ptr if N else None, bufs[2].ptr, maxTracks,
                                         bufs[3].ptr if maxMembers else None, maxMembers, _ptr(stats),
                                         ctypes.byref(ms)), "BuildTracks")
        M = int(stats[7])
        offsets = bufs[2].download(np.int32, T + 1)
        members = bufs[3].download(np.int32, 2 * M).reshape(M, 2) if M else np.zeros((0, 2), np.int32)
        trackOf = bufs[1].download(np.int32, N) if N else np.zeros(0, np.int32)
    finally:
        for buf in bufs:
            buf.free()
    return offsets, members, trackOf, stats, ms.value


def _set_table(datas):
    return (MatchSet * max(len(datas), 1))(*[MatchSet(d.d_data, d.numPts) for d in datas])


def TrainVocabulary(datas, numWords, maxIterations=10, seed=0):
    """A visual vocabulary of numWords unit-length words by spherical k-means over every feature of datas, in one call
    (cs_vocab_train).  Returns (vocab: a SiftData of numWords records whose descriptors are the words, trace float64
    [iterations run, 4] of {changed assignments, words without members, fallback rows, mean best score}, stats int64
    [4] as the header describes them, ms)."""
    vocab = InitSiftData(SiftData(), int(numWords))
    trace = np.zeros((max(int(maxIterations), 0), 4))
    stats, ms = np.zeros(4, np.int64), ctypes.c_double(0.0)
    try:
        _check(lib().cs_vocab_train(_set_table(datas) if datas else None, len(datas), int(numWords),
                                    int(maxIterations), int(seed), vocab.d_data, _ptr(trace) if len(trace) else None,
                                    _ptr(stats), ctypes.byref(ms)), "TrainVocabulary")
    except Exception:
        FreeSiftData(vocab)
        raise
    vocab.numPts = int(numWords)
    return vocab, trace[:int(stats[0])].copy(), stats, ms.value


def AssignWords(datas, vocab):
    """The word of every feature of datas in one call (cs_vocab_assign): j1 of match_knn2 against vocab's records, or
    -1.  Returns (wordOf int32 [sum of numPts], feature g = numPts of the earlier sets + i as in BuildTracks, stats
    uint64 [5] as the header describes them, ms)."""
    N = sum(int(d.numPts) for d in datas)
    stats, ms = np.zeros(5, np.uint64), ctypes.c_double(0.0)
    wordOf = np.zeros(N, np.int32)
    buf = DeviceBuffer(max(N, 1) * 4)
    try:
        _check(lib().cs_vocab_assign(_set_table(datas) if datas else None, len(datas), vocab.d_data, int(vocab.numPts),
                                     buf.ptr if N else None, _ptr(stats), ctypes.byref(ms)), "AssignWords")
        if N:
            wordOf = buf.download(np.int32, N)
    finally:
        buf.free()
    return wordOf, stats, ms.value


def RetrievePairs(imageSizes, wordOf, numWords, topK=50):
    """Every image's topK neighbours by tf-idf and the deduplicated pair table in one call (cs_retrieve_pairs):
    imageSizes[a] is image a's feature count and wordOf (int32 [sum of the sizes]) AssignWords' output.  Returns
    (neighbours int32 [N, topK] (-1: none), scores float64 [N, topK] (cosine of the fixed-point tf-idf vectors), pairs
    int32 [P, 2] of {a < b} in ascending order, ready as MatchSiftDataRatioBatch's jobs, stats int64 [7], ms)."""
    sizes = np.ascontiguousarray(np.asarray(imageSizes, np.int64).reshape(-1).astype(np.int32))
    words = np.ascontiguousarray(np.asarray(wordOf, np.int32).reshape(-1))
    I, N, K = len(sizes), int(sizes.sum(dtype=np.int64)), int(topK)
    if len(words) != N:
        raise ValueError("wordOf: one per feature, %d, not %d" % (N, len(words)))
    maxPairs = I * K
    neighbours, scores = np.full((I, K), -1, np.int32), np.zeros((I, K))
    stats, ms = np.zeros(7, np.int64), ctypes.c_double(0.0)
    bufs = [DeviceBuffer(max(N, 1) * 4), DeviceBuffer(max(I * K, 1) * 4), DeviceBuffer(max(I * K, 1) * 8),
            DeviceBuffer(max(maxPairs, 1) * 8)]
    try:
        if N:
            bufs[0].upload(words)
        P = _check(lib().cs_retrieve_pairs(_ptr(sizes) if I else None, I, bufs[0].ptr, int(numWords), K, bufs[1].ptr,
                                           bufs[2].ptr, None, bufs[3].ptr, maxPairs, _ptr(stats), ctypes.byref(ms)),
                   "RetrievePairs")
        if N and I:
            neighbours = bufs[1].download(np.int32, I * K).reshape(I, K)
            scores = bufs[2].download(np.float64, I * K).reshape(I, K)
        pairs = bufs[3].download(np.int32, 2 * P).reshape(P, 2) if P else np.zeros((0, 2), np.int32)
    finally:
        for buf in bufs:
            buf.free()
    return neighbours, scores, pairs, stats, ms.value


def _per_image(x, shape, n, what):
    """x as float64 [n, *shape]: one array per image, or one for every image."""
    x = np.asarray(x, np.float64)
    if x.shape == shape:
        x = np.broadcast_to(x, (n,) + shape)
    if x.shape != (n,) + shape:
        raise ValueError("%s: shape %s or (%d, %s), not %s" % (what, shape, n, ", ".join(map(str, shape)), x.shape))
    return np.ascontiguousarray(x)


def _tracks(offsets, members):
    """BuildTracks' offsets and members as contiguous int32 arrays, with the track and member counts."""
    off = np.ascontiguousarray(np.asarray(offsets, np.int64).reshape(-1).astype(np.int32))
    mem = np.ascontiguousarray(np.asarray(members, np.int64).reshape(-1, 2).astype(np.int32))
    return off, mem, max(len(off) - 1, 0), len(mem)


def TriangulateTracks(datas, Ks, Rs, ts, offsets, members, numTrials=256, maxError=4.0, minTriAngle=1.5, seed=0):
    """A 3-D point per feature track with known cameras, in one call (cs_triangulate_tracks): RANSAC over two-view DLT
    points, inliers by reprojection error below maxError pixels, one multi-view refit.  datas[a] holds image a's
    records; Ks, Rs ([3, 3] each) and ts ([3]) are per image or one for every image, camera a mapping a world point X to
    R_a X + t_a; offsets and members are BuildTracks' outputs.  Returns (points float64 [T, 3] (NaN without a point),
    counts int32 [T], errors float32 [M], inlier bool [M], stats int64 [8] as the header describes them, ms)."""
    S = len(datas)
    K, R, t = _per_image(Ks, (3, 3), S, "Ks"), _per_image(Rs, (3, 3), S, "Rs"), _per_image(ts, (3,), S, "ts")
    off, mem, T, M = _tracks(offsets, members)
    sets = _set_table(datas)
    points, counts = np.full((T, 3), np.nan), np.zeros(T, np.int32)
    errors, inlier = np.full(M, np.nan, np.float32), np.zeros(M, bool)
    stats, ms = np.zeros(8, np.int64), ctypes.c_double(0.0)
    bufs = [DeviceBuffer(max(off.nbytes, 4)), DeviceBuffer(max(mem.nbytes, 8)), DeviceBuffer(max(points.nbytes, 8)),
            DeviceBuffer(max(counts.nbytes, 4)), DeviceBuffer(max(errors.nbytes, 4)), DeviceBuffer(max(M, 1))]
    try:
        if T:
            bufs[0].upload(off)
        if M:
            bufs[1].upload(mem)
        _check(lib().cs_triangulate_tracks(sets if S else None, S, _ptr(K), _ptr(R), _ptr(t), bufs[0].ptr, T,
                                           bufs[1].ptr, M, int(numTrials), float(maxError), float(minTriAngle),
                                           int(seed), bufs[2].ptr, bufs[3].ptr, bufs[4].ptr, bufs[5].ptr, _ptr(stats),
                                           ctypes.byref(ms)), "TriangulateTracks")
        if T:
            points = bufs[2].download(np.float64, 3 * T).reshape(T, 3)
            counts = bufs[3].download(np.int32, T)
        if M:
            errors = bufs[4].download(np.float32, M)
            inlier = bufs[5].download(np.uint8, M).astype(bool)
    finally:
        for buf in bufs:
            buf.free()
    return points, counts, errors, inlier, stats, ms.value


def BundleAdjust(datas, Ks, Rs, ts, offsets, members, points, use=None, fixed=None, maxIterations=50,
                 maxLinearIterations=100, linearTol=1e-6, maxError=4.0):
    """Bundle adjustment of every camera and track point in one call (cs_bundle_adjust): Levenberg-Marquardt with the
    points eliminated by the Schur complement and the camera system solved by preconditioned CG on the device.  datas,
    Ks, Rs, ts, offsets and members as for TriangulateTracks; points [T, 3] its points (NaN: no point); use (bool [M],
    for example TriangulateTracks' inlier) selects the members to adjust on, None every valid one.  fixed (uint8 per
    image: 0 free, 1 held, 2..4 t[fixed - 2] held); None is COLMAP's gauge: image 0 held and image 1's largest |t|
    component held.  Returns (R [S, 3, 3], t [S, 3], points [T, 3], errors float32 [M], inlier bool [M] under the final
    parameters, cost (initial, final), trace float64 [iterations run, 4] of {candidate cost, lambda, CG iterations,
    accepted}, stats int64 [8] as the header describes them, ms)."""
    S = len(datas)
    K, R, t = _per_image(Ks, (3, 3), S, "Ks"), _per_image(Rs, (3, 3), S, "Rs"), _per_image(ts, (3,), S, "ts")

    def call(args):
        return lib().cs_bundle_adjust(args[0], S, _ptr(K), _ptr(R), _ptr(t), *args[1:])
    R_out, t_out, rest = _bundle_call(call, datas, R, t, offsets, members, points, use, fixed, maxIterations,
                                      maxLinearIterations, linearTol, maxError, "BundleAdjust")
    return (R_out, t_out) + rest


def _bundle_call(call, datas, R, t, offsets, members, points, use, fixed, maxIterations, maxLinearIterations,
                 linearTol, maxError, what):
    """The common arguments of BundleAdjust and BundleAdjustIntrinsics: call(args) makes the C call with args =
    (sets, fixed, d_offsets, numTracks, d_members, numMembers, d_use, d_points, maxIterations, maxLinearIterations,
    linearTol, maxError, R_out, t_out, d_errors, d_inlier, cost_out, trace_out, stats_out, ms) (the intrinsics' call
    puts its K_out and dist_out before R_out).  Returns (R_out, t_out, (points, errors, inlier, cost, trace, stats,
    ms))."""
    S = len(datas)
    off, mem, T, M = _tracks(offsets, members)
    pts = np.ascontiguousarray(np.asarray(points, np.float64).reshape(-1, 3))
    if len(pts) != T:
        raise ValueError("points: one per track, %d, not %d" % (T, len(pts)))
    if fixed is None:
        fixed = np.zeros(S, np.uint8)
        if S > 0:
            fixed[0] = 1
        if S > 1:
            fixed[1] = 2 + int(np.argmax(np.abs(t[1])))
    fix = np.ascontiguousarray(np.asarray(fixed).reshape(-1).astype(np.uint8))
    if len(fix) != S:
        raise ValueError("fixed: one per image, %d, not %d" % (S, len(fix)))
    u = None if use is None else np.ascontiguousarray(np.asarray(use).reshape(-1).astype(np.uint8))
    if u is not None and len(u) != M:
        raise ValueError("use: one per member, %d, not %d" % (M, len(u)))
    sets = _set_table(datas)
    R_out, t_out = np.zeros((S, 3, 3)), np.zeros((S, 3))
    errors, inlier = np.full(M, np.nan, np.float32), np.zeros(M, bool)
    cost, trace = np.zeros(2), np.zeros((max(int(maxIterations), 0), 4))
    stats, ms = np.zeros(8, np.int64), ctypes.c_double(0.0)
    bufs = [DeviceBuffer(max(off.nbytes, 4)), DeviceBuffer(max(mem.nbytes, 8)), DeviceBuffer(max(pts.nbytes, 8)),
            DeviceBuffer(max(4 * M, 4)), DeviceBuffer(max(M, 1)), DeviceBuffer(max(M, 1))]
    try:
        if T:
            bufs[0].upload(off)
            bufs[2].upload(pts)
        if M:
            bufs[1].upload(mem)
            if u is not None:
                bufs[5].upload(u)
        _check(call((sets if S else None, _ptr(fix) if S else None, bufs[0].ptr, T, bufs[1].ptr, M,
                     bufs[5].ptr if u is not None else None, bufs[2].ptr, int(maxIterations),
                     int(maxLinearIterations), float(linearTol), float(maxError), _ptr(R_out), _ptr(t_out),
                     bufs[3].ptr, bufs[4].ptr, _ptr(cost), _ptr(trace) if len(trace) else None, _ptr(stats),
                     ctypes.byref(ms))), what)
        if T:
            pts = bufs[2].download(np.float64, 3 * T).reshape(T, 3)
        if M and T:
            errors = bufs[3].download(np.float32, M)
            inlier = bufs[4].download(np.uint8, M).astype(bool)
    finally:
        for buf in bufs:
            buf.free()
    return R_out, t_out, (pts, errors, inlier, (cost[0], cost[1]), trace[:int(stats[6])].copy(), stats, ms.value)


LOSSES = {"trivial": 0, "soft_l1": 1, "cauchy": 2}


def BundleAdjustIntrinsics(datas, Ks, Rs, ts, offsets, members, points, dists=None, refine=3, loss="trivial",
                           lossScale=1.0, use=None, fixed=None, maxIterations=50, maxLinearIterations=100,
                           linearTol=1e-6, maxError=4.0):
    """Self-calibrating bundle adjustment in one call (cs_bundle_adjust_intrinsics): BundleAdjust with each image's
    focal length and radial distortion (k1, k2) refined and a robust loss.  dists ([2] per image or one for every image;
    None: zero) start the distortion; refine is one mask for every image or one per image (bit 0 focal, 1 k1, 2 k2;
    the default 3, focal and k1, is COLMAP's mapper default); loss is "trivial", "soft_l1" or "cauchy" with scale
    lossScale pixels.  The other arguments as BundleAdjust.  Returns (K [S, 3, 3], dists [S, 2], R [S, 3, 3], t [S, 3],
    points [T, 3], errors float32 [M], inlier bool [M] under the final parameters, cost (initial, final), trace,
    stats int64 [8], ms)."""
    S = len(datas)
    K, R, t = _per_image(Ks, (3, 3), S, "Ks"), _per_image(Rs, (3, 3), S, "Rs"), _per_image(ts, (3,), S, "ts")
    dist = np.zeros((S, 2)) if dists is None else _per_image(dists, (2,), S, "dists")
    ref = np.asarray(refine).reshape(-1)
    if ref.size == 1:
        ref = np.full(S, int(ref[0]))
    if len(ref) != S:
        raise ValueError("refine: one mask, or one per image, %d, not %d" % (S, len(ref)))
    if (ref < 0).any() or (ref > 7).any():
        raise ValueError("refine: masks of bits 0 (focal), 1 (k1) and 2 (k2)")
    ref = np.ascontiguousarray(ref.astype(np.uint8))
    if loss not in LOSSES:
        raise ValueError("loss: one of %s, not %r" % (", ".join(LOSSES), loss))
    K_out, dist_out = np.zeros((S, 3, 3)), np.zeros((S, 2))

    def call(args):
        return lib().cs_bundle_adjust_intrinsics(args[0], S, _ptr(K), _ptr(dist) if S else None,
                                                 _ptr(ref) if S else None, LOSSES[loss], float(lossScale), _ptr(R),
                                                 _ptr(t), *args[1:12], _ptr(K_out), _ptr(dist_out), *args[12:])
    R_out, t_out, rest = _bundle_call(call, datas, R, t, offsets, members, points, use, fixed, maxIterations,
                                      maxLinearIterations, linearTol, maxError, "BundleAdjustIntrinsics")
    return (K_out, dist_out, R_out, t_out) + rest


def UndistortRecords(datas, Ks, dists):
    """The records of every image with their positions undistorted under Ks and dists (cs_undistort_records), in new
    device SiftData (the caller frees them); every other field is copied, orientation and scale are not corrected.  A
    record whose inverse does not exist gets NaN positions (an invalid track member).  Ks [3, 3] and dists [2] per image
    or one for every image."""
    S = len(datas)
    K, dist = _per_image(Ks, (3, 3), S, "Ks"), _per_image(dists, (2,), S, "dists")
    outs = []
    try:
        for d in datas:
            o = InitSiftData(SiftData(), max(int(d.numPts), 1))
            o.numPts = int(d.numPts)
            outs.append(o)
        ptrs = (ctypes.c_void_p * max(S, 1))(*[o.d_data for o in outs])
        ms = ctypes.c_double(0.0)
        _check(lib().cs_undistort_records(_set_table(datas) if S else None, S, _ptr(K), _ptr(dist),
                                          ptrs if S else None, ctypes.byref(ms)), "UndistortRecords")
    except BaseException:
        for o in outs:
            FreeSiftData(o)
        raise
    return outs


def RotationAveraging(numImages, edges, Rrel, weights, refImage=0, maxIterations=50, maxLinearIterations=200,
                      linearTol=1e-8, sigmaDeg=5.0, maxAngleDeg=5.0):
    """Every image's absolute rotation from the relative rotations of verified pairs (cs_rotation_averaging): a maximum
    spanning tree by weight for the start, then IRLS under the Geman-McClure loss at sigmaDeg degrees (0: the squared
    loss), each iteration a Laplacian system solved by CG on the device.  edges [E, 2] are image pairs {i, j}, Rrel
    [E, 3, 3] VerifyEssentialBatch's R for them (X_j = R X_i + t) and weights [E] (for example its inlier counts), all
    > 0.  Returns (R [N, 3, 3] (NaN for an image not joined to refImage), residual angles in degrees [E] (NaN for an
    edge outside refImage's component), inlier bool [E] (angle < maxAngleDeg), cost (start, final), trace float64
    [iterations run, 3] of {cost, CG iterations, largest step}, stats int64 [6] as the header describes them,
    ms (spanning tree on the host, device))."""
    N = int(numImages)
    ed = np.ascontiguousarray(np.asarray(edges, np.int64).reshape(-1, 2).astype(np.int32))
    E = len(ed)
    Q = np.ascontiguousarray(np.asarray(Rrel, np.float64).reshape(-1, 9))
    w = np.ascontiguousarray(np.asarray(weights, np.float64).reshape(-1))
    if len(Q) != E or len(w) != E:
        raise ValueError("Rrel and weights: one per edge, %d, not %d and %d" % (E, len(Q), len(w)))
    R = np.zeros((max(N, 0), 9))
    residuals, inlier = np.full(E, np.nan), np.zeros(E, np.uint8)
    cost, trace = np.zeros(2), np.zeros((max(int(maxIterations), 0), 3))
    stats, ms = np.zeros(6, np.int64), np.zeros(2)
    p = (lambda a: _ptr(a) if a.size else None)
    _check(lib().cs_rotation_averaging(N, p(ed), E, p(Q), p(w), int(refImage), int(maxIterations),
                                       int(maxLinearIterations), float(linearTol), float(sigmaDeg),
                                       float(maxAngleDeg), p(R), p(residuals), p(inlier), _ptr(cost), p(trace),
                                       _ptr(stats), _ptr(ms)), "RotationAveraging")
    return (R.reshape(-1, 3, 3), residuals, inlier.astype(bool), (cost[0], cost[1]), trace[:int(stats[3])].copy(),
            stats, (ms[0], ms[1]))


def GlobalPositioning(datas, Ks, Rs, offsets, members, use=None, refImage=0, seed=0, loss="trivial", lossScale=1.0,
                      maxIterations=100, maxLinearIterations=100, linearTol=1e-6):
    """Every camera centre and track point from known rotations, in one call (cs_global_positioning): GLOMAP's BATA
    residual v - s (X - c) on every used observation, from random starts, by Levenberg-Marquardt on the device.  datas,
    Ks, offsets and members as for BundleAdjust; Rs [S, 3, 3] RotationAveraging's rotations (NaN: the image takes no
    part); use (bool [M]) selects members, None every valid one; loss "trivial", "soft_l1" or "cauchy" with scale
    lossScale (on unit rays).  Returns (t [S, 3] (NaN without a used observation), points [T, 3] (NaN for a track with
    fewer than 2), cost (start, final), trace float64 [iterations run, 4] as BundleAdjust's, stats int64 [8] as the
    header describes them, ms), at the header's scale: the RMS distance of the positioned centres from refImage's."""
    S = len(datas)
    K = _per_image(Ks, (3, 3), S, "Ks")
    R = _per_image(Rs, (3, 3), S, "Rs")
    off, mem, T, M = _tracks(offsets, members)
    u = None if use is None else np.ascontiguousarray(np.asarray(use).reshape(-1).astype(np.uint8))
    if u is not None and len(u) != M:
        raise ValueError("use: one per member, %d, not %d" % (M, len(u)))
    if loss not in LOSSES:
        raise ValueError("loss: one of %s, not %r" % (", ".join(LOSSES), loss))
    t = np.zeros((S, 3))
    points = np.full((T, 3), np.nan)
    cost, trace = np.zeros(2), np.zeros((max(int(maxIterations), 0), 4))
    stats, ms = np.zeros(8, np.int64), ctypes.c_double(0.0)
    bufs = [DeviceBuffer(max(off.nbytes, 4)), DeviceBuffer(max(mem.nbytes, 8)), DeviceBuffer(max(points.nbytes, 8)),
            DeviceBuffer(max(M, 1))]
    try:
        if T:
            bufs[0].upload(off)
        if M:
            bufs[1].upload(mem)
            if u is not None:
                bufs[3].upload(u)
        _check(lib().cs_global_positioning(_set_table(datas) if S else None, S, _ptr(K), _ptr(R), bufs[0].ptr, T,
                                           bufs[1].ptr, M, bufs[3].ptr if u is not None else None, int(refImage),
                                           int(seed), LOSSES[loss], float(lossScale), int(maxIterations),
                                           int(maxLinearIterations), float(linearTol), _ptr(t), bufs[2].ptr,
                                           _ptr(cost), _ptr(trace) if len(trace) else None, _ptr(stats),
                                           ctypes.byref(ms)), "GlobalPositioning")
        if T:
            points = bufs[2].download(np.float64, 3 * T).reshape(T, 3)
    finally:
        for buf in bufs:
            buf.free()
    return t, points, (cost[0], cost[1]), trace[:int(stats[6])].copy(), stats, ms.value


class StereoImage(ctypes.Structure):
    """cs_image: a device float32 grayscale image, pitch in floats."""
    _fields_ = [("d_img", ctypes.c_void_p), ("width", ctypes.c_int), ("height", ctypes.c_int), ("pitch", ctypes.c_int)]


class StereoJob(ctypes.Structure):
    """cs_stereo_job: one depth map of image ref from its source images (a host array)."""
    _fields_ = [("ref", ctypes.c_int), ("sources", ctypes.c_void_p), ("numSources", ctypes.c_int),
                ("depthMin", ctypes.c_float), ("depthMax", ctypes.c_float), ("d_depth", ctypes.c_void_p),
                ("d_normal", ctypes.c_void_p), ("d_cost", ctypes.c_void_p)]


class DepthPrior(ctypes.Structure):
    """cs_depth_prior: an image's prior depth and normal maps (device floats), NULL for none."""
    _fields_ = [("d_depth", ctypes.c_void_p), ("d_normal", ctypes.c_void_p)]


def _upload_images(images):
    """Host float32 [H, W] images in dense device buffers, and their cs_image table."""
    arrs = [np.ascontiguousarray(im, np.float32) for im in images]
    for im in arrs:
        if im.ndim != 2:
            raise ValueError("images: 2-D float32 arrays, not shape %s" % (im.shape,))
    bufs = []
    try:
        for im in arrs:
            b = DeviceBuffer(max(im.nbytes, 4))
            bufs.append(b)
            b.upload(im)
    except BaseException:
        for b in bufs:
            b.free()
        raise
    table = (StereoImage * max(len(arrs), 1))(*[StereoImage(b.ptr, im.shape[1], im.shape[0], im.shape[1])
                                               for b, im in zip(bufs, arrs)])
    return arrs, bufs, table


def _stereo_jobs(jobs, shapes, maps):
    """jobs as (ref, sources, depthMin, depthMax) tuples and their cs_stereo_job table, each with its three maps:
    maps(shape) returns three device buffers (depth, normal, cost), or None to pass the jobs' existing maps."""
    parsed = []
    for ref, sources, dmin, dmax in jobs:
        src = np.ascontiguousarray(np.asarray(sources, np.int64).reshape(-1).astype(np.int32))
        parsed.append((int(ref), src, float(dmin), float(dmax)))
    table = (StereoJob * max(len(parsed), 1))()
    bufs = []
    for p, (ref, src, dmin, dmax) in enumerate(parsed):
        if not 0 <= ref < len(shapes):
            raise ValueError("jobs[%d]: ref %d is not an image" % (p, ref))
        m = maps(p, shapes[ref])
        bufs.append(m)
        table[p] = StereoJob(ref, src.ctypes.data if len(src) else None, len(src), dmin, dmax,
                             *[b.ptr for b in m])
    return parsed, table, bufs


def UndistortImages(images, Ks, dists):
    """Every image as the pinhole camera K would see it (cs_undistort_images): each output pixel sampled bilinearly
    from the input at its position under the radial model (k1, k2) of BundleAdjustIntrinsics, 0 outside the input.
    images are float32 [H, W] host arrays on any scale (the output keeps it; PatchMatchStereo expects grey levels
    0..255); Ks [3, 3] and dists [2] per image or one for every image.  Returns (undistorted float32 [H, W] list,
    outside counts int64 [S], ms)."""
    S = len(images)
    K, dist = _per_image(Ks, (3, 3), S, "Ks"), _per_image(dists, (2,), S, "dists")
    arrs, bufs, table = _upload_images(images)
    outs = []
    try:
        for im in arrs:
            outs.append(DeviceBuffer(max(im.nbytes, 4)))
        ptrs = (ctypes.c_void_p * max(S, 1))(*[o.ptr for o in outs])
        outside, ms = np.zeros(S, np.int64), ctypes.c_double(0.0)
        _check(lib().cs_undistort_images(table if S else None, S, _ptr(K) if S else None, _ptr(dist) if S else None,
                                         ptrs if S else None, _ptr(outside) if S else None, ctypes.byref(ms)),
               "UndistortImages")
        res = [o.download(np.float32, im.size).reshape(im.shape) for o, im in zip(outs, arrs)]
    finally:
        for b in bufs + outs:
            b.free()
    return res, outside, ms.value


def PatchMatchStereo(images, Ks, Rs, ts, jobs, windowRadius=5, windowStep=1, numIterations=5, topK=3, seed=0):
    """A depth, normal and cost map for every job in one call (cs_patch_match_stereo): PatchMatch stereo with red-black
    propagation, the cost the mean of the topK smallest 1 - NCC view costs.  images are float32 [H, W] host arrays
    of grey levels on a 0..255 scale (pinhole: UndistortImages first): a window whose variance is below 1 grey
    level^2 makes its view invalid, so images scaled to [0, 1] leave every cost at 2.  Ks, Rs, ts per image (X_c = R X + t), jobs (ref, sources, depthMin, depthMax)
    tuples as SelectStereoViews returns them.  Returns (depth [J] of float32 [H, W], normal [J] of float32 [H, W, 3]
    in the ref camera frame, cost [J] of float32 [H, W] (2: unsupported), stats int64 [J, 3] of {pixels, invalid view
    evaluations, pixels of cost 2}, ms)."""
    S = len(images)
    K, R, t = _per_image(Ks, (3, 3), S, "Ks"), _per_image(Rs, (3, 3), S, "Rs"), _per_image(ts, (3,), S, "ts")
    arrs, bufs, table = _upload_images(images)
    shapes = [im.shape for im in arrs]
    maps = []
    try:
        parsed, jt, maps = _stereo_jobs(jobs, shapes, lambda p, sh: [DeviceBuffer(4 * sh[0] * sh[1]),
                                                                     DeviceBuffer(12 * sh[0] * sh[1]),
                                                                     DeviceBuffer(4 * sh[0] * sh[1])])
        J = len(parsed)
        stats, ms = np.zeros((J, 3), np.int64), ctypes.c_double(0.0)
        _check(lib().cs_patch_match_stereo(table if S else None, S, _ptr(K), _ptr(R), _ptr(t), jt if J else None, J,
                                           int(windowRadius), int(windowStep), int(numIterations), int(topK),
                                           int(seed), _ptr(stats) if J else None, ctypes.byref(ms)),
               "PatchMatchStereo")
        depth, normal, cost = [], [], []
        for (ref, _, _, _), m in zip(parsed, maps):
            h, w = shapes[ref]
            depth.append(m[0].download(np.float32, h * w).reshape(h, w))
            normal.append(m[1].download(np.float32, 3 * h * w).reshape(h, w, 3))
            cost.append(m[2].download(np.float32, h * w).reshape(h, w))
    finally:
        for b in bufs + [b for m in maps for b in m]:
            b.free()
    return depth, normal, cost, stats, ms.value


def PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, depth, normal, windowRadius=5, windowStep=1, numIterations=5,
                              topK=3, geomWeight=0.3, geomMaxError=3.0, seed=0):
    """PatchMatch stereo with geometric consistency (cs_patch_match_stereo_geometric): every job's maps again, each
    view's cost joined by geomWeight times its forward-backward reprojection error (pixels, capped at geomMaxError)
    against that source's depth map.  depth and normal are PatchMatchStereo's maps for the same jobs, as FuseDepthMaps
    takes them: each job's ref gets its maps as its prior, and an image that is no job's ref has none.  Other arguments
    as for PatchMatchStereo; the defaults are COLMAP's.  Returns (depth [J], normal [J], cost [J], stats int64 [J, 5] of
    {pixels, invalid view evaluations, pixels of cost >= 2, valid view evaluations capped at geomMaxError, pixels started
    from a random hypothesis}, ms)."""
    S = len(images)
    K, R, t = _per_image(Ks, (3, 3), S, "Ks"), _per_image(Rs, (3, 3), S, "Rs"), _per_image(ts, (3,), S, "ts")
    if not (len(depth) == len(normal) == len(jobs)):
        raise ValueError("depth and normal: one map per job")
    arrs, bufs, table = _upload_images(images)
    shapes = [im.shape for im in arrs]
    maps = []
    try:
        parsed, jt, maps = _stereo_jobs(jobs, shapes, lambda p, sh: [DeviceBuffer(4 * sh[0] * sh[1]),
                                                                     DeviceBuffer(12 * sh[0] * sh[1]),
                                                                     DeviceBuffer(4 * sh[0] * sh[1])])
        J = len(parsed)
        priors = (DepthPrior * max(S, 1))()
        for p, (ref, _, _, _) in enumerate(parsed):
            h, w = shapes[ref]
            bufs.append(DeviceBuffer(4 * h * w))
            bufs.append(DeviceBuffer(12 * h * w))
            pd, pn = bufs[-2:]
            pd.upload(np.ascontiguousarray(np.asarray(depth[p], np.float32).reshape(h, w)))
            pn.upload(np.ascontiguousarray(np.asarray(normal[p], np.float32).reshape(h, w, 3)))
            priors[ref] = DepthPrior(pd.ptr, pn.ptr)
        stats, ms = np.zeros((J, 5), np.int64), ctypes.c_double(0.0)
        _check(lib().cs_patch_match_stereo_geometric(table if S else None, S, _ptr(K), _ptr(R), _ptr(t),
                                                     priors if S else None, jt if J else None, J, int(windowRadius),
                                                     int(windowStep), int(numIterations), int(topK),
                                                     float(geomWeight), float(geomMaxError), int(seed),
                                                     _ptr(stats) if J else None, ctypes.byref(ms)),
               "PatchMatchStereoGeometric")
        dep, nrm, cost = [], [], []
        for (ref, _, _, _), m in zip(parsed, maps):
            h, w = shapes[ref]
            dep.append(m[0].download(np.float32, h * w).reshape(h, w))
            nrm.append(m[1].download(np.float32, 3 * h * w).reshape(h, w, 3))
            cost.append(m[2].download(np.float32, h * w).reshape(h, w))
    finally:
        for b in bufs + [b for m in maps for b in m]:
            b.free()
    return dep, nrm, cost, stats, ms.value


def FuseDepthMaps(images, Ks, Rs, ts, jobs, depth, normal, cost, maxCost=0.5, minConsistent=2, maxReprojError=2.0,
                  maxDepthError=0.01, maxNormalErrorDeg=10.0, maxPoints=None):
    """One point cloud from the maps of PatchMatchStereo (cs_fuse_depth_maps): a pixel with cost <= maxCost emits a
    point when at least minConsistent of its sources that are themselves refs agree in depth (relative
    maxDepthError), normal (maxNormalErrorDeg degrees) and reprojection (maxReprojError px), and none of them has a
    lower image index.  Arguments as for PatchMatchStereo plus its maps; maxPoints None: room for every pixel.  Returns
    (xyz float32 [P, 3], normal float32 [P, 3], intensity float32 [P], source int32 [P, 2] of {image, y W + x} in
    ascending order, total (the full count, >= P), ms)."""
    S = len(images)
    K, R, t = _per_image(Ks, (3, 3), S, "Ks"), _per_image(Rs, (3, 3), S, "Rs"), _per_image(ts, (3,), S, "ts")
    if not (len(depth) == len(normal) == len(cost) == len(jobs)):
        raise ValueError("depth, normal and cost: one map per job")
    arrs, bufs, table = _upload_images(images)
    shapes = [im.shape for im in arrs]
    maps = []
    try:
        def upload(p, sh):
            m = [DeviceBuffer(4 * sh[0] * sh[1]), DeviceBuffer(12 * sh[0] * sh[1]), DeviceBuffer(4 * sh[0] * sh[1])]
            for b, a in zip(m, (depth[p], normal[p], cost[p])):
                b.upload(np.ascontiguousarray(a, np.float32))
            return m
        parsed, jt, maps = _stereo_jobs(jobs, shapes, upload)
        J = len(parsed)
        room = sum(shapes[ref][0] * shapes[ref][1] for ref, _, _, _ in parsed) if maxPoints is None else int(maxPoints)
        outs = [DeviceBuffer(max(12 * room, 4)), DeviceBuffer(max(12 * room, 4)), DeviceBuffer(max(4 * room, 4)),
                DeviceBuffer(max(8 * room, 8))]
        bufs += outs
        stats, ms = np.zeros(2, np.int64), ctypes.c_double(0.0)
        n = _check(lib().cs_fuse_depth_maps(table if S else None, S, _ptr(K), _ptr(R), _ptr(t), jt if J else None, J,
                                            float(maxCost), int(minConsistent), float(maxReprojError),
                                            float(maxDepthError), float(maxNormalErrorDeg),
                                            *[o.ptr if room else None for o in outs], room, _ptr(stats),
                                            ctypes.byref(ms)), "FuseDepthMaps")
        P = int(stats[1])
        xyz = outs[0].download(np.float32, 3 * P).reshape(P, 3)
        nrm = outs[1].download(np.float32, 3 * P).reshape(P, 3)
        inten = outs[2].download(np.float32, P)
        src = outs[3].download(np.int32, 2 * P).reshape(P, 2)
    finally:
        for b in bufs + [b for m in maps for b in m]:
            b.free()
    return xyz, nrm, inten, src, n, ms.value


def _poisson_call(call, name, nInfo, xyz, normal, intensity, depth, returnChi):
    """The host side of cs_poisson_mesh and cs_poisson_mesh_screened: upload, call(ins, outs, maxV, maxT, info, stats,
    ms) into output buffers of 12 N^2 vertices and 24 N^2 triangles, again into buffers of the full size while the mesh
    is larger, and download."""
    X = np.ascontiguousarray(np.asarray(xyz, np.float32).reshape(-1, 3))
    Nr = np.ascontiguousarray(np.asarray(normal, np.float32).reshape(-1, 3))
    if len(Nr) != len(X):
        raise ValueError("xyz and normal: one row per point")
    I = None if intensity is None else np.ascontiguousarray(np.asarray(intensity, np.float32).reshape(-1))
    if I is not None and len(I) != len(X):
        raise ValueError("intensity: one value per point")
    P, n = len(X), (1 << int(depth)) + 1 if 4 <= int(depth) <= 9 else 17
    maxV, maxT = 12 * (n - 1) ** 2, 24 * (n - 1) ** 2
    ins = [DeviceBuffer(max(X.nbytes, 4)), DeviceBuffer(max(Nr.nbytes, 4))] + ([DeviceBuffer(max(I.nbytes, 4))]
                                                                               if I is not None else [None])
    try:
        for b, a in zip(ins, (X, Nr, I)):
            if P and b is not None:
                b.upload(a)
        while True:
            outs = [DeviceBuffer(12 * maxV + 4), DeviceBuffer(12 * maxT + 4),
                    DeviceBuffer(4 * maxV + 4) if I is not None else None,
                    DeviceBuffer(4 * n ** 3) if returnChi else None]
            try:
                info, stats, ms = np.zeros(nInfo), np.zeros(10, np.int64), ctypes.c_double(0.0)
                T = _check(call(*[b.ptr if b is not None else None for b in ins + outs], P, maxV, maxT, _ptr(info),
                                _ptr(stats), ctypes.byref(ms)), name)
                V = int(stats[5])
                if V > maxV or T > maxT:
                    maxV, maxT = max(V, maxV), max(T, maxT)
                    continue
                verts = outs[0].download(np.float32, 3 * V).reshape(V, 3)
                tris = outs[1].download(np.int32, 3 * T).reshape(T, 3)
                vint = outs[2].download(np.float32, V) if outs[2] else None
                chi = outs[3].download(np.float32, n ** 3).reshape(n, n, n) if outs[3] else None
                return verts, tris, vint, info, stats, chi, ms.value
            finally:
                for b in outs:
                    if b is not None:
                        b.free()
    finally:
        for b in ins:
            if b is not None:
                b.free()


def PoissonMesh(xyz, normal, intensity=None, depth=8, scale=1.1, maxIterations=200, tol=1e-5, trim=0.0,
                returnChi=False):
    """A closed, oriented triangle mesh of an oriented point cloud (cs_poisson_mesh): Poisson reconstruction on a
    regular grid of 2^depth cells per axis, solved by multigrid-preconditioned CG to tol, the surface at the mean of
    chi over the points, extracted by marching tetrahedra; triangles with a vertex whose splatted density is below trim
    times the mean density are dropped.  xyz and normal are float32 [P, 3] host arrays (outward normals, any length),
    intensity [P] or None, as FuseDepthMaps returns them.  The output buffers first hold 12 N^2 vertices and 24 N^2
    triangles (N = 2^depth); a mesh with more is computed again into buffers of its full size, so nothing is
    truncated.  Returns (vertices float32 [V, 3], triangles int32 [T, 3], vertex intensity float32 [V] or None,
    info float64 [7] {o_x, o_y, o_z, h, tau, mean density, true relative residual}, stats int64 [10] (the header's),
    chi float32 [N + 1, N + 1, N + 1] indexed (z, y, x) or None, ms)."""
    def call(x, nr, inten, verts, tris, vint, chi, P, maxV, maxT, info, stats, ms):
        return lib().cs_poisson_mesh(x, nr, inten, P, int(depth), float(scale), int(maxIterations), float(tol),
                                     float(trim), verts, vint, maxV, tris, maxT, chi, info, stats, ms)
    return _poisson_call(call, "PoissonMesh", 7, xyz, normal, intensity, depth, returnChi)


def PoissonMeshScreened(xyz, normal, intensity=None, depth=8, scale=1.1, pointWeight=4.0, maxIterations=200, tol=1e-5,
                        trim=0.0, returnChi=False):
    """A triangle mesh of an oriented point cloud by screened Poisson reconstruction with a Neumann boundary
    (cs_poisson_mesh_screened): PoissonMesh's grid, splat, solver and extraction, with chi pulled towards 0 at the
    points by pointWeight (alpha; the effective weight is alpha over the mean density) and no boundary value, so open
    surfaces seen from one side get a mesh; untrimmed, such a mesh ends on the grid's faces, and trim cuts it back to
    where the points are.  Arguments and returns as PoissonMesh's, with info float64 [8]: PoissonMesh's 7 entries,
    then the effective weight omega."""
    def call(x, nr, inten, verts, tris, vint, chi, P, maxV, maxT, info, stats, ms):
        return lib().cs_poisson_mesh_screened(x, nr, inten, P, int(depth), float(scale), float(pointWeight),
                                              int(maxIterations), float(tol), float(trim), verts, vint, maxV, tris,
                                              maxT, chi, info, stats, ms)
    return _poisson_call(call, "PoissonMeshScreened", 8, xyz, normal, intensity, depth, returnChi)


def SimplifyMesh(vertices, triangles, intensity=None, targetTriangles=0, maxError=float("inf"), boundaryWeight=1.0):
    """Quadric-error edge collapse of a triangle mesh (cs_simplify_mesh) in parallel passes of independent collapses,
    until at most targetTriangles remain (the result ends at the target or one below) or no collapse has
    sqrt(cost / area) <= maxError.  vertices float32 [V, 3], triangles int32 [T, 3] and intensity [V] or None, as
    PoissonMesh returns them; boundaryWeight weighs the planes that hold boundary edges in place.  The outputs are
    never larger than the inputs, so buffers of the input's size hold them.  Returns (vertices float32 [V', 3],
    triangles int32 [T', 3], intensity float32 [V'] or None, info float64 [1] {largest applied sqrt(cost / area)},
    stats int64 [9] (the header's), ms)."""
    X = np.ascontiguousarray(np.asarray(vertices, np.float32).reshape(-1, 3))
    F = np.ascontiguousarray(np.asarray(triangles, np.int32).reshape(-1, 3))
    I = None if intensity is None else np.ascontiguousarray(np.asarray(intensity, np.float32).reshape(-1))
    if I is not None and len(I) != len(X):
        raise ValueError("intensity: one value per vertex")
    V, T = len(X), len(F)
    ins = [DeviceBuffer(max(X.nbytes, 4)), DeviceBuffer(max(F.nbytes, 4)),
           DeviceBuffer(max(I.nbytes, 4)) if I is not None else None]
    outs = [DeviceBuffer(12 * V + 4), DeviceBuffer(12 * T + 4), DeviceBuffer(4 * V + 4) if I is not None else None]
    try:
        for b, a in zip(ins, (X, F, I)):
            if b is not None and a.size:
                b.upload(a)
        ptr = lambda b: b.ptr if b is not None else None
        info, stats, ms = np.zeros(1), np.zeros(9, np.int64), ctypes.c_double(0.0)
        n = _check(lib().cs_simplify_mesh(ptr(ins[0]), ptr(ins[2]), V, ptr(ins[1]), T, int(targetTriangles),
                                          float(maxError), float(boundaryWeight), ptr(outs[0]), ptr(outs[2]), V,
                                          ptr(outs[1]), T, _ptr(info), _ptr(stats), ctypes.byref(ms)), "SimplifyMesh")
        nv = int(stats[4])
        verts = outs[0].download(np.float32, 3 * nv).reshape(nv, 3)
        tris = outs[1].download(np.int32, 3 * n).reshape(n, 3)
        vint = outs[2].download(np.float32, nv) if I is not None else None
        return verts, tris, vint, info, stats, ms.value
    finally:
        for b in ins + outs:
            if b is not None:
                b.free()


def CleanMesh(vertices, triangles, intensity=None, removeDegenerate=True, longEdgeFactor=20.0, removeNonManifold=True,
              minComponentFaces=50, minComponentFraction=0.0, maxHoleEdges=30, smoothIterations=0, smoothLambda=0.5,
              smoothMu=-0.53):
    """Mesh cleaning (cs_clean_mesh), in the header's order: degenerate and duplicate faces (removeDegenerate), faces
    with an edge longer than mean + longEdgeFactor * stddev of the edge lengths (0: off), faces past the first two on
    an edge held by three or more (removeNonManifold), components of fewer than minComponentFaces faces or
    minComponentFraction of the largest, then boundary loops of at most maxHoleEdges edges (0: off, at most 256) closed
    by ear cutting, and smoothIterations Taubin steps (smoothLambda, smoothMu).  vertices float32 [V, 3], triangles
    int32 [T, 3] and intensity [V] or None, as PoissonMesh returns them.  Returns (vertices float32 [V', 3], triangles
    int32 [T', 3], intensity float32 [V'] or None, info float64 [3] {edge length mean, stddev, threshold}, stats int64
    [19] (the header's), ms)."""
    X = np.ascontiguousarray(np.asarray(vertices, np.float32).reshape(-1, 3))
    F = np.ascontiguousarray(np.asarray(triangles, np.int32).reshape(-1, 3))
    I = None if intensity is None else np.ascontiguousarray(np.asarray(intensity, np.float32).reshape(-1))
    if I is not None and len(I) != len(X):
        raise ValueError("intensity: one value per vertex")
    V, T = len(X), len(F)
    ins = [DeviceBuffer(max(X.nbytes, 4)), DeviceBuffer(max(F.nbytes, 4)),
           DeviceBuffer(max(I.nbytes, 4)) if I is not None else None]
    maxT = T + T // 4 + 256 if maxHoleEdges else T
    try:
        for b, a in zip(ins, (X, F, I)):
            if b is not None and a.size:
                b.upload(a)
        ptr = lambda b: b.ptr if b is not None else None
        while True:
            outs = [DeviceBuffer(12 * V + 4), DeviceBuffer(12 * maxT + 4),
                    DeviceBuffer(4 * V + 4) if I is not None else None]
            try:
                info, stats, ms = np.zeros(3), np.zeros(19, np.int64), ctypes.c_double(0.0)
                n = _check(lib().cs_clean_mesh(ptr(ins[0]), ptr(ins[2]), V, ptr(ins[1]), T, int(bool(removeDegenerate)),
                                               float(longEdgeFactor), int(bool(removeNonManifold)),
                                               int(minComponentFaces), float(minComponentFraction), int(maxHoleEdges),
                                               int(smoothIterations), float(smoothLambda), float(smoothMu),
                                               ptr(outs[0]), ptr(outs[2]), V, ptr(outs[1]), maxT, _ptr(info),
                                               _ptr(stats), ctypes.byref(ms)), "CleanMesh")
                if n > maxT:
                    maxT = n
                    continue
                nv = int(stats[14])
                verts = outs[0].download(np.float32, 3 * nv).reshape(nv, 3)
                tris = outs[1].download(np.int32, 3 * n).reshape(n, 3)
                vint = outs[2].download(np.float32, nv) if I is not None else None
                return verts, tris, vint, info, stats, ms.value
            finally:
                for b in outs:
                    if b is not None:
                        b.free()
    finally:
        for b in ins:
            if b is not None:
                b.free()


def TextureMesh(images, Ks, Rs, ts, vertices, triangles, smoothness=0.5, maxViewAngle=75.0, depthTol=0.01, padding=2,
                atlasWidth=None, maxSweeps=100):
    """A texture atlas for a triangle mesh from the images that see it (cs_texture_mesh): every face takes the image
    that sees it largest, unoccluded (depth buffers, relative depthTol) and within maxViewAngle degrees of its normal,
    traded against smoothness (the labelling's lambda) per pair of adjacent faces with different images; adjacent faces
    with the same image form charts, whose image rectangles (padding pixels around) are copied into one atlas
    atlasWidth texels wide (None: the widest image, rounded up to a multiple of 256, at least 1024).  images, Ks, Rs, ts
    as for PatchMatchStereo (pinhole), vertices float32 [V, 3] and triangles int32 [T, 3] as SimplifyMesh or PoissonMesh
    return them.  The atlas is computed again into a buffer of its full height when the first guess is too small, so
    nothing is truncated.  Returns (atlas float32 [rows, atlasWidth], uv float32 [T, 3, 2] in atlas pixels (NaN for an
    unseen face), labels int32 [T] (the image, -1 unseen), charts int32 [C, 8] {image, x0, y0, width, height, ox, oy,
    faces}, info float64 [2] {energy before, after the sweeps}, stats int64 [11] (the header's), ms)."""
    return _texture_mesh("TextureMesh", lib().cs_texture_mesh, 11, images, Ks, Rs, ts, vertices,
                         triangles, smoothness, maxViewAngle, depthTol, padding, atlasWidth, maxSweeps)


def TextureMeshPhoto(images, Ks, Rs, ts, vertices, triangles, dataTerm="gmi", outlierK=3.0, outlierMinSigma=4.0,
                     smoothness=0.5, maxViewAngle=75.0, depthTol=0.01, padding=2, atlasWidth=None, maxSweeps=100):
    """TextureMesh with Waechter et al.'s view selection (cs_texture_mesh_photo): dataTerm "gmi" ranks a face's views
    by the projected area times (1 + the mean Sobel magnitude over its visible pixels, in grey levels per pixel), so a
    sharp view beats a blurred one of the same size ("area": TextureMesh's ranking); outlierK > 0 removes the views
    whose mean intensity over the face lies more than outlierK max(1.4826 MAD, outlierMinSigma) from the median of its
    views (MAD: the median absolute deviation), so an object seen in one view only (a passer-by) does not texture the
    face; 0 turns the test off.  Images on a 0..255 scale.  The other arguments and the returned tuple are TextureMesh's,
    with stats int64 [16]: TextureMesh's 11, then samples, centroid fallbacks, faces tested, candidates removed, faces
    whose best candidate was removed."""
    terms = {"area": 0, "gmi": 1}
    if dataTerm not in terms:
        raise ValueError("dataTerm: 'area' or 'gmi', not %r" % (dataTerm,))
    extra = (terms[dataTerm], float(outlierK), float(outlierMinSigma))
    return _texture_mesh("TextureMeshPhoto", lambda *a: lib().cs_texture_mesh_photo(*a[:9], *extra, *a[9:]), 16,
                         images, Ks, Rs, ts, vertices, triangles, smoothness, maxViewAngle, depthTol, padding,
                         atlasWidth, maxSweeps)


def TextureMeshBP(images, Ks, Rs, ts, vertices, triangles, dataTerm="gmi", outlierK=3.0, outlierMinSigma=4.0,
                  bpSweeps=32, smoothness=0.5, maxViewAngle=75.0, depthTol=0.01, padding=2, atlasWidth=None,
                  maxSweeps=100):
    """TextureMeshPhoto with its labelling solved by min-sum belief propagation before the ICM sweeps
    (cs_texture_mesh_bp): at most bpSweeps sweeps of messages in colour order, the labelling of lowest energy kept, then
    ICM from it.  BP removes islands of faces that ICM keeps (a run of faces that all prefer another view by a small
    margin), so the result has no more energy, and usually fewer seams and charts.  bpSweeps 0 gives TextureMeshPhoto's
    outputs.  The default, 32: on the texture bench's scene and sphere, 128 sweeps lower the final energy by under
    0.1 % more, at 2.4 to 3.2 times the call time (DESIGN.md section 8).  Returns TextureMeshPhoto's tuple with info float64 [3] {E at the start, E after the ICM sweeps, E of
    the labelling BP kept} and stats int64 [20]: TextureMeshPhoto's 16, then BP sweeps, the sweep kept (0: the start),
    messages changed in the last sweep (0: converged), faces whose label BP moved from their best view."""
    terms = {"area": 0, "gmi": 1}
    if dataTerm not in terms:
        raise ValueError("dataTerm: 'area' or 'gmi', not %r" % (dataTerm,))
    extra = (terms[dataTerm], float(outlierK), float(outlierMinSigma), int(bpSweeps))
    return _texture_mesh("TextureMeshBP", lambda *a: lib().cs_texture_mesh_bp(*a[:9], *extra, *a[9:]), 20,
                         images, Ks, Rs, ts, vertices, triangles, smoothness, maxViewAngle, depthTol, padding,
                         atlasWidth, maxSweeps, ninfo=3)


def RefineMesh(images, Ks, Rs, ts, vertices, triangles, pairs, windowRadius=4, smoothness=0.2, step=0.1,
               maxIterations=100, depthTol=0.01):
    """Photometric refinement of a triangle mesh (cs_mesh_refine, after Vu et al. and OpenMVS's RefineMesh): every
    free vertex moves by gradient descent on the windowed NCC (window 2 windowRadius + 1) between each ordered image
    pair, reprojected through the mesh, plus smoothness times a thin-plate term; each step moves a vertex by at most
    2 step mean edge lengths, and a halving line search accepts only steps that lower the energy, at most maxIterations
    of them.  Vertices on a boundary or non-manifold edge, and unused ones, stay put; the topology does not change.
    images, Ks, Rs, ts as for TextureMesh (pinhole, 0..255), vertices float32 [V, 3] and triangles int32 [T, 3];
    pairs an int [n, 2] array of (ref, src) or SelectStereoViews' jobs (each source of each job paired with its ref).
    Returns (vertices float32 [V, 3], info float64 [4] {E_photo, E_s at the start, at the end}, stats int64 [8]
    {pairs, free vertices, fixed vertices, P0, evaluations, accepted steps, halvings of the final step, status}, ms)."""
    if len(pairs) and not np.isscalar(pairs[0]) and len(pairs[0]) == 4:
        pairs = [(int(ref), int(s)) for ref, srcs, _, _ in pairs for s in np.asarray(srcs).reshape(-1)]
    P = np.ascontiguousarray(np.asarray(pairs, np.int64).reshape(-1, 2).astype(np.int32))
    S = len(images)
    K, R, t = _per_image(Ks, (3, 3), S, "Ks"), _per_image(Rs, (3, 3), S, "Rs"), _per_image(ts, (3,), S, "ts")
    X = np.ascontiguousarray(np.asarray(vertices, np.float32).reshape(-1, 3))
    F = np.ascontiguousarray(np.asarray(triangles, np.int32).reshape(-1, 3))
    V, T = len(X), len(F)
    arrs, bufs, table = _upload_images(images)
    try:
        ins = [DeviceBuffer(max(X.nbytes, 4)), DeviceBuffer(max(F.nbytes, 4)), DeviceBuffer(max(X.nbytes, 4))]
        bufs += ins
        for b, a in zip(ins, (X, F)):
            if a.size:
                b.upload(a)
        info, stats, ms = np.zeros(4), np.zeros(8, np.int64), ctypes.c_double(0.0)
        _check(lib().cs_mesh_refine(table if S else None, S, _ptr(K), _ptr(R), _ptr(t), ins[0].ptr, V, ins[1].ptr, T,
                                    _ptr(P) if len(P) else None, len(P), int(windowRadius), float(smoothness),
                                    float(step), int(maxIterations), float(depthTol), ins[2].ptr, _ptr(info),
                                    _ptr(stats), ctypes.byref(ms)), "RefineMesh")
        out = ins[2].download(np.float32, 3 * V).reshape(V, 3) if V and stats[7] != 2 else X.copy()
        return out, info, stats, ms.value
    finally:
        for b in bufs:
            b.free()


def _texture_mesh(name, call, nstats, images, Ks, Rs, ts, vertices, triangles, smoothness, maxViewAngle,
                  depthTol, padding, atlasWidth, maxSweeps, ninfo=2):
    """The body of TextureMesh, TextureMeshPhoto and TextureMeshBP: call takes cs_texture_mesh's arguments (the
    other calls' settings inserted by the caller), stats has nstats entries and info ninfo."""
    S = len(images)
    K, R, t = _per_image(Ks, (3, 3), S, "Ks"), _per_image(Rs, (3, 3), S, "Rs"), _per_image(ts, (3,), S, "ts")
    X = np.ascontiguousarray(np.asarray(vertices, np.float32).reshape(-1, 3))
    F = np.ascontiguousarray(np.asarray(triangles, np.int32).reshape(-1, 3))
    V, T = len(X), len(F)
    arrs, bufs, table = _upload_images(images)
    if atlasWidth is None:
        atlasWidth = max(1024, -(-max([im.shape[1] for im in arrs] + [1]) // 256) * 256)
    W = int(atlasWidth)
    rows, maxCharts = max(64, int(np.sqrt(max(sum(im.size for im in arrs), 1)))), max(T, 1)
    try:
        ins = [DeviceBuffer(max(X.nbytes, 4)), DeviceBuffer(max(F.nbytes, 4))]
        bufs += ins
        for b, a in zip(ins, (X, F)):
            if a.size:
                b.upload(a)
        outs = [DeviceBuffer(24 * T + 4), DeviceBuffer(4 * T + 4)]
        bufs += outs
        while True:
            atlas = DeviceBuffer(4 * rows * W + 4)
            try:
                charts = np.zeros((maxCharts, 8), np.int32)
                info, stats, ms = np.zeros(ninfo), np.zeros(nstats, np.int64), ctypes.c_double(0.0)
                C = _check(call(table if S else None, S, _ptr(K), _ptr(R), _ptr(t), ins[0].ptr, V, ins[1].ptr, T,
                                float(smoothness), float(maxViewAngle), float(depthTol), int(padding), W,
                                int(maxSweeps), atlas.ptr, rows, outs[0].ptr, outs[1].ptr, None, _ptr(charts),
                                maxCharts, _ptr(info), _ptr(stats), ctypes.byref(ms)), name)
                full = int(stats[8])
                if full > rows:
                    rows = full
                    continue
                img = atlas.download(np.float32, full * W).reshape(full, W)
                uv = outs[0].download(np.float32, 6 * T).reshape(T, 3, 2)
                labels = outs[1].download(np.int32, T)
                return img, uv, labels, charts[:C].copy(), info, stats, ms.value
            finally:
                atlas.free()
    finally:
        for b in bufs:
            b.free()


def _seams_inputs(bufs, vertices, triangles, atlas, uv, labels, charts):
    """The inputs of LevelTextureSeams and LevelTextureSeamsLocal as the C calls take them: the vertices, triangles,
    labels, uv and atlas in device buffers (appended to bufs, which the caller frees) and the chart table on the host.
    Returns (device buffers in that order, chart table, V, T, atlas rows, atlas width)."""
    X = np.ascontiguousarray(np.asarray(vertices, np.float32).reshape(-1, 3))
    F = np.ascontiguousarray(np.asarray(triangles, np.int32).reshape(-1, 3))
    A = np.ascontiguousarray(np.asarray(atlas, np.float32))
    U = np.ascontiguousarray(np.asarray(uv, np.float32).reshape(-1, 3, 2))
    Lb = np.ascontiguousarray(np.asarray(labels, np.int32).reshape(-1))
    Ct = np.ascontiguousarray(np.asarray(charts, np.int32).reshape(-1, 8))
    ins = [DeviceBuffer(max(a.nbytes, 4)) for a in (X, F, Lb, U, A)]
    bufs += ins
    for b, a in zip(ins, (X, F, Lb, U, A)):
        if a.size:
            b.upload(a)
    return ins, Ct, len(X), len(F), A.shape[0], A.shape[1]


def LevelTextureSeams(vertices, triangles, atlas, uv, labels, charts, padding=2, smoothness=0.1, regularization=1e-3,
                      maxIterations=1000, tol=1e-4):
    """Global seam levelling of a textured mesh (cs_level_texture_seams): one additive offset per (vertex, image) pair,
    solved so that the two sides of every seam agree while the offsets vary smoothly along each chart (smoothness, the
    weight of those rows; regularization, the pull of every offset towards 0), and added to the atlas texel by texel.
    The inputs are TextureMesh's outputs as it returns them (padding the value given to it); no image is needed.
    Returns (levelled atlas float32 [rows, width], corner offsets float32 [T, 3] (NaN for an unseen face), info
    float64 [3] {seam energy before, after, relative residual}, stats int64 [8] (the header's), ms)."""
    bufs = []
    try:
        ins, Ct, V, T, H, W = _seams_inputs(bufs, vertices, triangles, atlas, uv, labels, charts)
        outs = [DeviceBuffer(max(4 * H * W, 4)), DeviceBuffer(12 * T + 4)]
        bufs += outs
        info, stats, ms = np.zeros(3), np.zeros(8, np.int64), ctypes.c_double(0.0)
        _check(lib().cs_level_texture_seams(ins[0].ptr, V, ins[1].ptr, T, ins[2].ptr, ins[3].ptr, _ptr(Ct), len(Ct),
                                            ins[4].ptr, H, W, int(padding), float(smoothness), float(regularization),
                                            int(maxIterations), float(tol), outs[0].ptr, outs[1].ptr, _ptr(info),
                                            _ptr(stats), ctypes.byref(ms)), "LevelTextureSeams")
        out = outs[0].download(np.float32, H * W).reshape(H, W)
        off = outs[1].download(np.float32, 3 * T).reshape(T, 3)
        return out, off, info, stats, ms.value
    finally:
        for b in bufs:
            b.free()


def LevelTextureSeamsLocal(vertices, triangles, atlas, uv, labels, charts, padding=2, stripWidth=20, maxIterations=1000,
                           tol=1e-4):
    """Local seam levelling of a textured mesh (cs_level_texture_seams_local): Poisson editing of the texel strips
    along every seam.  Each seam texel takes the mean of the two sides' values sampled along the seam; the texels within
    stripWidth neighbour steps of a seam, in the same chart, get the smooth correction that keeps the atlas's own
    gradients and meets those values (a membrane solved by CG to tol).  Run it after LevelTextureSeams, on its output:
    the inputs are TextureMesh's (padding the value given to it) with the atlas replaced.  Returns (levelled atlas
    float32 [rows, width], info float64 [3] {sum (f* - g)^2 over seam texels, relative residual, max |delta|}, stats
    int64 [8] (the header's), ms)."""
    bufs = []
    try:
        ins, Ct, V, T, H, W = _seams_inputs(bufs, vertices, triangles, atlas, uv, labels, charts)
        out = DeviceBuffer(max(4 * H * W, 4))
        bufs.append(out)
        info, stats, ms = np.zeros(3), np.zeros(8, np.int64), ctypes.c_double(0.0)
        _check(lib().cs_level_texture_seams_local(ins[0].ptr, V, ins[1].ptr, T, ins[2].ptr, ins[3].ptr, _ptr(Ct),
                                                  len(Ct), ins[4].ptr, H, W, int(padding), int(stripWidth),
                                                  int(maxIterations), float(tol), out.ptr, _ptr(info), _ptr(stats),
                                                  ctypes.byref(ms)), "LevelTextureSeamsLocal")
        return out.download(np.float32, H * W).reshape(H, W), info, stats, ms.value
    finally:
        for b in bufs:
            b.free()


def _png_grey(path, img):
    """An 8-bit greyscale PNG of img (uint8 [H, W]) by zlib and struct alone."""
    import struct
    import zlib
    img = np.ascontiguousarray(img, np.uint8)
    H, W = img.shape

    def chunk(kind, data):
        body = kind + data
        return struct.pack(">I", len(data)) + body + struct.pack(">I", zlib.crc32(body) & 0xFFFFFFFF)

    raw = np.concatenate([np.zeros((H, 1), np.uint8), img], axis=1).tobytes()   # filter type 0 per row
    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n")
        f.write(chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 0, 0, 0, 0)))
        f.write(chunk(b"IDAT", zlib.compress(raw, 6)))
        f.write(chunk(b"IEND", b""))


def save_textured_obj(path, vertices, triangles, uv, atlas):
    """A textured mesh as OBJ + MTL + PNG: path.obj (or path as given when it ends in .obj), its .mtl and .png beside
    it.  uv are TextureMesh's atlas pixel coordinates (converted to OBJ's [0, 1] with v up); atlas the float atlas,
    written as 8-bit grey (rounded, clipped to 0..255).  Faces with NaN coordinates (unseen) are written without
    texture coordinates.  Returns the paths written (obj, mtl, png)."""
    import os as _os
    base = path[:-4] if path.endswith(".obj") else path
    name = _os.path.basename(base)
    objp, mtlp, pngp = base + ".obj", base + ".mtl", base + ".png"
    atlas = np.asarray(atlas, np.float32)
    H, W = atlas.shape
    _png_grey(pngp, np.clip(np.rint(atlas), 0, 255).astype(np.uint8))
    with open(mtlp, "w") as f:
        f.write("newmtl atlas\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nmap_Kd %s.png\n" % name)
    X = np.asarray(vertices, np.float32).reshape(-1, 3)
    F = np.asarray(triangles, np.int64).reshape(-1, 3)
    U = np.asarray(uv, np.float64).reshape(-1, 3, 2)
    seen = np.isfinite(U).all(axis=(1, 2))
    vt = np.stack([(U[..., 0] + 0.5) / W, 1.0 - (U[..., 1] + 0.5) / H], -1)   # texel (x, y) centred at x + 1/2, v up
    lines = ["mtllib %s.mtl" % name, "usemtl atlas"]
    lines += ["v %.9g %.9g %.9g" % tuple(p) for p in X]
    k = 0
    faces = []
    for f in range(len(F)):
        a, b, c = F[f] + 1
        if seen[f]:
            for j in range(3):
                lines.append("vt %.9g %.9g" % tuple(vt[f, j]))
            faces.append("f %d/%d %d/%d %d/%d" % (a, k + 1, b, k + 2, c, k + 3))
            k += 3
        else:
            faces.append("f %d %d %d" % (a, b, c))
    with open(objp, "w") as f:
        f.write("\n".join(lines + faces) + "\n")
    return objp, mtlp, pngp


def SelectStereoViews(Ks, Rs, ts, offsets, members, points, numSources=8, minTriAngle=1.0):
    """The stereo jobs of a sparse model (host, numpy): for every image a, the numSources images that share the most
    tracks with a finite point whose triangulation angle between the two images' rays is >= minTriAngle degrees (ties
    to the lower index, count > 0), and the depth range [0.75 p1, 1.25 p99] of the depths of a's observed points
    (COLMAP's rule).  offsets and members are BuildTracks' outputs, points TriangulateTracks'.  An image without such a
    point or without a source gets no job.  Returns a list of (ref, sources int32 array, depthMin, depthMax)."""
    S = len(np.asarray(Rs, np.float64).reshape(-1, 3, 3))
    K, R, t = _per_image(Ks, (3, 3), S, "Ks"), _per_image(Rs, (3, 3), S, "Rs"), _per_image(ts, (3,), S, "ts")
    off, mem, T, M = _tracks(offsets, members)
    X = np.asarray(points, np.float64).reshape(-1, 3)
    C = -np.einsum("aji,aj->ai", R, t)                      # camera centres
    shared = np.zeros((S, S), np.int64)
    depths = [[] for _ in range(S)]
    cosMin = np.cos(np.radians(float(minTriAngle)))
    for k in range(T):
        if not np.all(np.isfinite(X[k])):
            continue
        imgs = np.unique(mem[off[k]:off[k + 1], 0])
        imgs = imgs[(imgs >= 0) & (imgs < S)]
        for a in imgs:
            z = R[a, 2] @ X[k] + t[a, 2]
            if z > 0:
                depths[a].append(z)
        rays = X[k] - C[imgs]
        rays /= np.linalg.norm(rays, axis=1, keepdims=True)
        cos = np.clip(rays @ rays.T, -1.0, 1.0)
        ok = cos <= cosMin
        np.fill_diagonal(ok, False)
        shared[np.ix_(imgs, imgs)] += ok
    jobs = []
    for a in range(S):
        if not depths[a]:
            continue
        order = sorted((b for b in range(S) if b != a and shared[a, b] > 0), key=lambda b: (-shared[a, b], b))
        if not order:
            continue
        d = np.asarray(depths[a])
        jobs.append((a, np.array(order[:int(numSources)], np.int32), 0.75 * np.percentile(d, 1),
                     1.25 * np.percentile(d, 99)))
    return jobs


class PoseJob(ctypes.Structure):
    """cs_pose_job: one image to register, its point indices and its per-feature outputs (device pointers)."""
    _fields_ = [("pts", ctypes.c_void_p), ("n", ctypes.c_int), ("pointOf", ctypes.c_void_p),
                ("seed", ctypes.c_ulonglong), ("errors", ctypes.c_void_p), ("inlier", ctypes.c_void_p)]


def AbsolutePoseBatch(datas, pointOfs, points, Ks, numLoops=1024, maxError=4.0, seeds=None):
    """The pose of many images against known 3-D points, in one call (cs_absolute_pose_batch): RANSAC over P3P poses,
    inliers by reprojection error below maxError pixels, one Levenberg-Marquardt refinement.  datas[p] holds image p's
    records and pointOfs[p] (int, one per record) the point of each feature or < 0, for example
    trackOf[base_p : base_p + n_p] of BuildTracks; points [P, 3], for example TriangulateTracks' points; Ks [3, 3] per
    image or one for every image; seeds one per job (default 0, 1, ...).  The point indices and the points go up once
    each.  Returns (R float64 [J, 3, 3], t [J, 3] with X_c = R X + t (zero without a pose), counts int32 [J], errors: a
    list of float32 [n_p], inlier: a list of bool [n_p], stats int64 [J, 8] as the header describes them, ms)."""
    J = len(datas)
    if len(pointOfs) != J:
        raise ValueError("pointOfs: one per image, %d, not %d" % (J, len(pointOfs)))
    K = _per_image(Ks, (3, 3), J, "Ks")
    P = np.ascontiguousarray(np.asarray(points, np.float64).reshape(-1, 3))
    seeds = np.arange(J, dtype=np.uint64) if seeds is None else np.asarray(seeds, np.uint64).reshape(-1)
    if len(seeds) != J:
        raise ValueError("seeds: one per image, %d, not %d" % (J, len(seeds)))
    ns = [int(d.numPts) for d in datas]
    idx = [np.asarray(po, np.int64).reshape(-1) for po in pointOfs]
    for p in range(J):
        if len(idx[p]) != ns[p]:
            raise ValueError("pointOfs[%d]: %d entries for %d records" % (p, len(idx[p]), ns[p]))
    offs = np.concatenate([[0], np.cumsum(ns, dtype=np.int64)]).astype(np.int64)
    N = int(offs[-1])
    flat = np.ascontiguousarray(np.concatenate(idx).astype(np.int32)) if N else np.zeros(0, np.int32)
    R, t = np.zeros((J, 3, 3)), np.zeros((J, 3))
    counts, stats, ms = np.zeros(J, np.int32), np.zeros((J, 8), np.int64), ctypes.c_double(0.0)
    bufs = [DeviceBuffer(max(P.nbytes, 8)), DeviceBuffer(max(4 * N, 4)), DeviceBuffer(max(4 * N, 4)),
            DeviceBuffer(max(N, 1))]
    try:
        if len(P):
            bufs[0].upload(P)
        if N:
            bufs[1].upload(flat)
        table = (PoseJob * max(J, 1))()
        for p in range(J):
            o = int(offs[p])
            table[p] = PoseJob(datas[p].d_data if ns[p] else None, ns[p], bufs[1].ptr + 4 * o if ns[p] else None,
                               int(seeds[p]), bufs[2].ptr + 4 * o if ns[p] else None, bufs[3].ptr + o if ns[p] else None)
        _check(lib().cs_absolute_pose_batch(bufs[0].ptr if len(P) else None, len(P),
                                            ctypes.addressof(table) if J else None, J, _ptr(K), int(numLoops),
                                            float(maxError), _ptr(R), _ptr(t), _ptr(counts), _ptr(stats),
                                            ctypes.byref(ms)), "AbsolutePoseBatch")
        err = bufs[2].download(np.float32, N) if N else np.zeros(0, np.float32)
        inl = bufs[3].download(np.uint8, N).astype(bool) if N else np.zeros(0, bool)
    finally:
        for buf in bufs:
            buf.free()
    errors = [err[offs[p]:offs[p + 1]].copy() for p in range(J)]
    inlier = [inl[offs[p]:offs[p + 1]].copy() for p in range(J)]
    return R, t, counts, errors, inlier, stats, ms.value


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
