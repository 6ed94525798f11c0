"""ctypes binding of the CPU oracle (oracle/sift_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs, never by the cudasift_b200 package.
"""
import ctypes
import os
import subprocess

import numpy as np

_DIR = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_DIR, "liboracle.so")
_lib = None

SIFT_DTYPE = np.dtype([
    ("xpos", "<f4"), ("ypos", "<f4"), ("scale", "<f4"), ("sharpness", "<f4"), ("edgeness", "<f4"),
    ("orientation", "<f4"), ("score", "<f4"), ("ambiguity", "<f4"), ("match", "<i4"),
    ("match_xpos", "<f4"), ("match_ypos", "<f4"), ("match_error", "<f4"), ("subsampling", "<f4"),
    ("empty", "<f4", (3,)), ("data", "<f4", (128,))])


def build(force=False):
    src = os.path.join(_DIR, "sift_oracle.c")
    if (not force and os.path.exists(_LIB_PATH)
            and os.path.getmtime(_LIB_PATH) >= max(os.path.getmtime(src), os.path.getmtime(src[:-2] + ".h"))):
        return _LIB_PATH
    subprocess.check_call(["gcc", "-O2", "-mfma", "-ffp-contract=off", "-fPIC", "-shared", "-o", _LIB_PATH, src,
                           "-lm", "-lpthread"])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        try:
            build()
        except Exception:
            if not os.path.exists(_LIB_PATH):
                raise
        L = ctypes.CDLL(_LIB_PATH)
        c = ctypes
        vp, ip, fp = c.c_void_p, c.c_int, c.c_float
        L.oracle_scaledown_taps.argtypes = [fp, vp]
        L.oracle_lowpass_taps.argtypes = [fp, vp]
        L.oracle_laplace_taps.argtypes = [ip, fp, vp]
        L.oracle_lowpass.argtypes = [vp, vp, ip, ip, ip, fp]
        L.oracle_scaledown.argtypes = [vp, vp, ip, ip, ip, ip]
        L.oracle_scaleup.argtypes = [vp, vp, ip, ip, ip, ip]
        L.oracle_dog.argtypes = [vp, vp, ip, ip, ip, vp]
        L.oracle_find_points.argtypes = [vp, ip, ip, ip, fp, fp, fp, fp, fp, vp, vp, ip, ip]
        L.oracle_find_points.restype = ip
        L.oracle_tex2d.argtypes = [vp, ip, ip, ip, fp, fp]
        L.oracle_tex2d.restype = fp
        L.oracle_orientations.argtypes = [vp, ip, ip, ip, vp, ip, ip, vp, ip]
        L.oracle_descriptors.argtypes = [vp, ip, ip, ip, vp, ip, ip, fp]
        L.oracle_last_q22.restype = ip
        L.oracle_extract.argtypes = [vp, ip, ip, ip, ip, fp, fp, fp, ip, vp, ip, vp]
        L.oracle_extract.restype = ip
        L.oracle_match.argtypes = [vp, ip, vp, ip]
        L.oracle_match_mt.argtypes = [vp, ip, vp, ip, ip]
        L.oracle_find_homography.argtypes = [vp, ip, vp, vp, ip, fp, fp, fp]
        L.oracle_find_homography.restype = c.c_double
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def laplace_taps(numOctaves, initBlur=0.0):
    k = np.zeros(8 * 12 * 16, np.float32)
    lib().oracle_laplace_taps(numOctaves, initBlur, _p(k))
    return k


def lowpass(img, sigma):
    img = np.ascontiguousarray(img, np.float32)
    h, w = img.shape
    out = np.zeros_like(img)
    lib().oracle_lowpass(_p(img), _p(out), w, h, w, sigma)
    return out


def scaledown(img):
    img = np.ascontiguousarray(img, np.float32)
    h, w = img.shape
    out = np.zeros((h // 2, w // 2), np.float32)
    lib().oracle_scaledown(_p(img), _p(out), w, h, w, w // 2)
    return out


def scaleup(img):
    img = np.ascontiguousarray(img, np.float32)
    h, w = img.shape
    out = np.zeros((2 * h, 2 * w), np.float32)
    lib().oracle_scaleup(_p(img), _p(out), w, h, w, 2 * w)
    return out


def dog(base, numOctaves, octave):
    base = np.ascontiguousarray(base, np.float32)
    h, w = base.shape
    taps = laplace_taps(numOctaves)[octave * 192: octave * 192 + 128].copy()
    out = np.zeros((7, h, w), np.float32)
    lib().oracle_dog(_p(base), _p(out), w, h, w, _p(taps))
    return out


def tex2d(img, xs, ys):
    img = np.ascontiguousarray(img, np.float32)
    h, w = img.shape
    L = lib()
    return np.array([L.oracle_tex2d(_p(img), w, h, w, float(x), float(y)) for x, y in zip(xs, ys)], np.float32)


def orientations(level, pts):
    """oracle_orientations on one pyramid level: pts (records in level coordinates) with their orientations set and
    the secondaries appended, as the reference's ComputeOrientations leaves them."""
    level = np.ascontiguousarray(level, np.float32)
    h, w = level.shape
    out = np.zeros(2 * len(pts), SIFT_DTYPE)
    out[:len(pts)] = pts
    count = ctypes.c_int(len(pts))
    lib().oracle_orientations(_p(level), w, h, w, _p(out), 0, len(pts), ctypes.byref(count), len(out))
    return out[:count.value].copy()


def descriptors(level, pts, subsampling=1.0):
    """oracle_descriptors on one pyramid level: (records with descriptors, positions scaled by subsampling; the
    number of angi == 8 votes, quirk Q22)."""
    level = np.ascontiguousarray(level, np.float32)
    h, w = level.shape
    out = np.ascontiguousarray(pts, SIFT_DTYPE).copy()
    lib().oracle_descriptors(_p(level), w, h, w, _p(out), 0, len(out), subsampling)
    return out, int(lib().oracle_last_q22())


def set_cap32(on):
    """The reference's cap of 32 extrema per (30x8 block, scale), cudaSiftD.cu:1371: on by default."""
    lib().oracle_set_cap32(int(bool(on)))


def set_cap_limit(n):
    """Tests only: the cap's limit (32 in the reference); natural DoG planes never hold 33 extrema per block and scale."""
    lib().oracle_set_cap_limit(int(n))


def last_dropped():
    """Extrema the cap dropped during the last extract()."""
    return int(lib().oracle_last_dropped())


def extract(img, numOctaves=5, initBlur=1.0, thresh=3.0, lowestScale=0.0, scaleUp=False, maxPts=32768):
    """Returns (records[:numPts], total records written incl. the finest octave's secondaries)."""
    img = np.ascontiguousarray(img, np.float32)
    h, w = img.shape
    pts = np.zeros(maxPts, SIFT_DTYPE)
    total = ctypes.c_int(0)
    n = lib().oracle_extract(_p(img), w, h, w, numOctaves, initBlur, thresh, lowestScale, int(scaleUp), _p(pts),
                             maxPts, ctypes.byref(total))
    return pts[:n].copy(), total.value


def match(s1, s2, threads=1):
    s1 = np.ascontiguousarray(s1, SIFT_DTYPE).copy()
    s2 = np.ascontiguousarray(s2, SIFT_DTYPE)
    if threads > 1:
        lib().oracle_match_mt(_p(s1), len(s1), _p(s2), len(s2), threads)
    else:
        lib().oracle_match(_p(s1), len(s1), _p(s2), len(s2))
    return s1


def find_homography(pts, numLoops=1000, minScore=0.85, maxAmbiguity=0.95, thresh=5.0, seed=None):
    """Returns (3x3 homography, numMatches).  seed: srand() value set just before the call."""
    pts = np.ascontiguousarray(pts, SIFT_DTYPE)
    H = np.zeros(9, np.float32)
    n = ctypes.c_int(0)
    if seed is not None:
        ctypes.CDLL(None).srand(int(seed))
    lib().oracle_find_homography(_p(pts), len(pts), _p(H), ctypes.byref(n), numLoops, minScore, maxAmbiguity, thresh)
    return H.reshape(3, 3), n.value
