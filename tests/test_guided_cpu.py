"""CPU checks of guided matching (cs_match_knn2_guided, cs_match_guided, cs_match_guided_host): the entry points exist,
they reject bad arguments before any CUDA call, empty sets write nothing, the numpy float32 statement of the predicate
equals the C oracle's bit for bit and agrees with the float64 Sampson and transfer errors, and the strip bound the F
culling relies on holds in float64."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import guided_oracle as go
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("cs_match_knn2_guided", "cs_match_guided", "cs_match_guided_host")
CS_E_ARG = -2
REC = 576


def test_symbols_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for name in NEW + ("cs_match_guided_stats",):
        assert name in declared and name in exported, name
        assert hasattr(cs.lib(), name)
    for name in ("match_knn2_guided", "MatchSiftDataGuided", "match_guided_host", "guided_stats"):
        assert name in cs.__all__ and callable(getattr(cs, name)), name
    assert build.SOURCES.count("match_guided.cu") == 1


def _layout(base):
    """Two sets of 4 records, then 8-byte aligned room for idx, score and pairs."""
    s1, s2 = base, base + 4 * REC
    out = base + 8 * REC
    return s1, s2, out, out + 64, out + 128


def _models():
    good = np.eye(3).reshape(9)
    nan, inf = good.copy(), good.copy()
    nan[4], inf[8] = np.nan, np.inf
    return good, [("model nan", nan), ("model inf", inf), ("model zero", np.zeros(9)),
                  ("model norm overflows", np.full(9, 1e200))]


def _cases(entry, base):
    s1, s2, idx, sc, pairs = _layout(base)
    good, bad_models = _models()
    nan = float("nan")
    if entry == "cs_match_knn2_guided":
        def a(s1=s1, n1=4, s2=s2, n2=4, model=2, M=good, t=4.0, idx=idx, sc=sc):
            return (s1, n1, s2, n2, model, None if M is None else M.ctypes.data, t, idx, sc)
        cases = [("n1 < 0", a(n1=-1)), ("n2 < 0", a(n2=-3)), ("NULL set 1", a(s1=None)), ("NULL set 2", a(s2=None)),
                 ("NULL idx", a(idx=None)), ("NULL score", a(sc=None)), ("idx unaligned", a(idx=idx + 4)),
                 ("score inside set 2", a(sc=s2 + 3 * REC)), ("idx and score overlap", a(sc=idx + 16))]
    else:
        def a(s1=s1, n1=4, s2=s2, n2=4, model=2, M=good, t=4.0, r=0.8, d=0.7, cc=1, pairs=pairs, mp=4):
            return (s1, n1, s2, n2, model, None if M is None else M.ctypes.data, t, r, d, cc, pairs, mp)
        cases = [("n1 < 0", a(n1=-1)), ("n2 < 0", a(n2=-3)), ("NULL set 1", a(s1=None)), ("NULL set 2", a(s2=None)),
                 ("maxPairs < 0", a(mp=-1)), ("NULL pairs", a(pairs=None)), ("NaN maxRatio", a(r=nan)),
                 ("NaN maxDistance", a(d=nan)), ("pairs unaligned", a(pairs=pairs + 4)),
                 ("pairs inside set 1", a(pairs=s1 + 2 * REC))]
    cases += [("model 0", a(model=0)), ("model 3", a(model=3)), ("NULL model", a(M=None)),
              ("thresh 0", a(t=0.0)), ("thresh < 0", a(t=-1.0)), ("thresh nan", a(t=nan)),
              ("thresh inf", a(t=float("inf")))]
    cases += [(what, a(M=M)) for what, M in bad_models]
    return cases, good


@pytest.mark.parametrize("entry", NEW)
def test_invalid_arguments_return_cs_e_arg(entry):
    """Every invalid argument fails with CS_E_ARG, and *ms is reset, whether or not a device is present."""
    buf = np.zeros(8 * REC + 256 + 16, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    f = getattr(cs.lib(), entry)
    cases, _ = _cases(entry, base)
    for what, args in cases:
        ms = ctypes.c_double(-1.0)
        assert f(*args, ctypes.byref(ms)) == CS_E_ARG, (entry, what)
        msg = cs.lib().cs_last_error().decode()
        assert "invalid argument" in msg and "CS_E_ARG" in msg, (entry, what, msg)
        assert ms.value == 0.0, (entry, what)
    assert not buf.any()


@pytest.mark.parametrize("entry", NEW)
def test_empty_sets_write_nothing(entry):
    buf = np.zeros(8 * REC + 256 + 16, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    s1, s2, idx, sc, pairs = _layout(base)
    M = np.eye(3).reshape(9)
    f = getattr(cs.lib(), entry)
    ms = ctypes.c_double(-1.0)
    if entry == "cs_match_knn2_guided":
        assert f(s1, 0, s2, 4, 1, M.ctypes.data, 4.0, None, None, ctypes.byref(ms)) == 0 and ms.value == 0.0
        assert f(s1, 4, None, 0, 2, M.ctypes.data, 4.0, idx, sc, None) == 0
        assert f(None, 0, None, 0, 2, M.ctypes.data, 4.0, None, None, None) == 0
    else:
        assert f(s1, 0, s2, 4, 1, M.ctypes.data, 4.0, 0.8, 0.7, 1, None, 0, ctypes.byref(ms)) == 0 and ms.value == 0.0
        assert f(s1, 4, None, 0, 2, M.ctypes.data, 4.0, 0.8, 0.7, 0, pairs, 4, None) == 0
        assert f(s1, 0, s1, 4, 2, M.ctypes.data, 4.0, 0.8, 0.7, 1, pairs, 4, None) == 0
    assert not buf.any()


def test_python_wrappers_raise_on_rejection():
    z = np.zeros(3, cs.SIFT_DTYPE)
    with pytest.raises(cs.CudaSiftError, match="invalid argument"):
        cs.match_guided_host(z, z, "fundamental", np.zeros((3, 3)))
    with pytest.raises(cs.CudaSiftError, match="invalid argument"):
        cs.match_guided_host(z, z, "homography", np.eye(3), thresh=-1.0)
    with pytest.raises(cs.CudaSiftError, match="invalid argument"):
        cs.match_knn2_guided(z[:0], z, "homography", np.eye(3), thresh=float("nan"))
    with pytest.raises(ValueError):
        cs.match_guided_host(z, z, "affine", np.eye(3))


def _random_models(rng, k):
    """Fundamental matrices of random camera pairs (some with the epipole inside a 1920x1080 image) and homographies."""
    Fs, Hs = [], []
    K = np.array([[1400.0, 0, 960], [0, 1400.0, 540], [0, 0, 1]])
    for s in range(k):
        a = rng.normal(0, 0.1, 3)
        Ax = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        R = np.eye(3) + Ax + Ax @ Ax / 2
        t = rng.normal(0, 1, 3)
        if s % 3 == 0:
            t = np.array([rng.normal(0, 0.1), rng.normal(0, 0.1), 1.0])     # forward motion: epipole inside
        tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
        Fs.append(np.linalg.inv(K).T @ tx @ R @ np.linalg.inv(K) * 10 ** rng.uniform(-3, 3))
        Hs.append(K @ (R + np.outer(t, rng.normal(0, 0.1, 3))) @ np.linalg.inv(K) * 10 ** rng.uniform(-3, 3))
    return Fs, Hs


def _inputs(rng, n):
    x, y = rng.uniform(-50, 2000, n), rng.uniform(-50, 1130, n)
    u, v = rng.uniform(-50, 2000, n), rng.uniform(-50, 1130, n)
    return [a.astype(np.float32) for a in (x, y, u, v)]


def test_numpy_predicate_equals_c_bit_for_bit():
    rng = np.random.default_rng(3)
    Fs, Hs = _random_models(rng, 6)
    x, y, u, v = _inputs(rng, 200000)
    ext = np.array([0, -0.0, 1e7, -1e7, 3.4e38, -3.4e38, 1e-40, np.nan, np.inf, -np.inf, 960, 540], np.float32)
    g = np.array(np.meshgrid(ext, ext, ext, ext)).reshape(4, -1)
    for model, Ms in ((go.F, Fs), (go.H, Hs)):
        for M in Ms + [np.eye(3) * 1e-150, np.array([[0, 0, 0], [0, 0, 0], [0, 0, 1.0]])]:
            for t in (1.0, 4.0, 16.0, 1e5, 1e-20):
                want = go.admissible_c(model, M, t, x, y, u, v)
                assert np.array_equal(go.admissible_np(model, M, t, x, y, u, v), want), (model, t)
                assert np.array_equal(go.admissible_np(model, M, t, *g), go.admissible_c(model, M, t, *g)), (model, t)
            # near the threshold: set 2 points placed on the model's own boundary
            if model == go.H:
                p = np.column_stack([x, y, np.ones_like(x)]).astype(np.float64) @ M.T
                ang = rng.uniform(0, 2 * np.pi, len(x))
                for s in (1 - 1e-6, 1 + 1e-6):
                    uu = (p[:, 0] / p[:, 2] + 4.0 * s * np.cos(ang)).astype(np.float32)
                    vv = (p[:, 1] / p[:, 2] + 4.0 * s * np.sin(ang)).astype(np.float32)
                    assert np.array_equal(go.admissible_np(model, M, 4.0, x, y, uu, vv),
                                          go.admissible_c(model, M, 4.0, x, y, uu, vv))


def _sampson(F, x1, x2):
    l1 = x1 @ F.T
    l2 = x2 @ F
    num = (x2 * l1).sum(1)
    return np.sqrt(num ** 2 / (l1[:, 0] ** 2 + l1[:, 1] ** 2 + l2[:, 0] ** 2 + l2[:, 1] ** 2))


def _transfer(H, x1, x2):
    p = x1 @ H.T
    return np.hypot(x2[:, 0] - p[:, 0] / p[:, 2], x2[:, 1] - p[:, 1] / p[:, 2])


def test_predicate_agrees_with_float64_errors():
    """Away from a 1e-4 relative band around thresh, the FP32 predicate is the float64 error below thresh."""
    rng = np.random.default_rng(5)
    Fs, Hs = _random_models(rng, 6)
    n = 100000
    for model, Ms in ((go.F, Fs), (go.H, Hs)):
        for M in Ms:
            x, y = rng.uniform(0, 1920, n).astype(np.float32), rng.uniform(0, 1080, n).astype(np.float32)
            x1 = np.column_stack([x, y, np.ones(n)]).astype(np.float64)
            # set-2 points near the model: mostly within a few thresholds
            if model == go.H:
                p = x1 @ M.T
                c = p[:, :2] / p[:, 2:]
            else:
                l = x1 @ M.T
                foot = rng.uniform(0, 1920, n)
                c = np.column_stack([foot, -(l[:, 0] * foot + l[:, 2]) / l[:, 1]])
            x2 = np.column_stack([c + rng.normal(0, 6, (n, 2)), np.ones(n)]).astype(np.float32).astype(np.float64)
            # inside the second view: the FP32 band grows with the coordinates over thresh
            keep = np.isfinite(x2).all(1) & (x2[:, 0] >= 0) & (x2[:, 0] < 1920) & (x2[:, 1] >= 0) & (x2[:, 1] < 1080)
            x1, x2 = x1[keep], x2[keep]
            err = _sampson(M, x1, x2) if model == go.F else _transfer(M, x1, x2)
            for t in (1.0, 4.0, 16.0):
                got = go.admissible_np(model, M, t, x1[:, 0], x1[:, 1], x2[:, 0], x2[:, 1])
                clear = np.abs(err - t) > 1e-4 * t
                assert np.array_equal(got[clear], err[clear] < t), (model, t, int((got[clear] != (err[clear] < t)).sum()))
                assert got.sum() > 100


def test_fundamental_strip_bound():
    """Sampson error < t implies that x2 lies within t * sqrt(1 + B / a) of the epipolar line F x1 (a = |(F x1)_01|^2,
    B = max over set 2 of |(F^T x2)_01|^2), and x1 within t * sqrt(1 + A / b) of F^T x2: the half-widths of the strips
    the F culling enumerates (DESIGN.md section 4)."""
    rng = np.random.default_rng(7)
    Fs, _ = _random_models(rng, 12)
    n = 200000
    for F in Fs:
        F = F / np.linalg.norm(F)
        x1 = np.column_stack([rng.uniform(0, 1920, n), rng.uniform(0, 1080, n), np.ones(n)])
        x2 = np.column_stack([rng.uniform(0, 1920, n), rng.uniform(0, 1080, n), np.ones(n)])
        l1, l2 = x1 @ F.T, x2 @ F
        a, b = l1[:, 0] ** 2 + l1[:, 1] ** 2, l2[:, 0] ** 2 + l2[:, 1] ** 2
        A, B = a.max(), b.max()
        num = np.abs((x2 * l1).sum(1))
        for t in (1.0, 4.0, 16.0, 200.0):
            ok = num ** 2 < t * t * (a + b)
            assert ok.sum() > 0
            d2 = num / np.sqrt(a)                        # distance of x2 from the line F x1
            d1 = num / np.sqrt(b)                        # distance of x1 from the line F^T x2
            assert (d2[ok] < t * np.sqrt(1 + B / a[ok])).all()
            assert (d1[ok] < t * np.sqrt(1 + A / b[ok])).all()
            # and the bound is needed: Sampson < t does not imply a line distance < t
            if t == 200.0:
                assert (d2[ok] >= t).any() or (d1[ok] >= t).any()
