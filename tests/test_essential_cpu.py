"""CPU checks of calibrated verification (cs_verify_essential, _host, _stats, _models): the entry points exist, they
reject bad arguments before any CUDA call, the Python wrappers return the right shapes for empty inputs, and the
float64 restatement (tests/essential_oracle.py) is right on its own: the 5-point solver on exact calibrated samples,
the pose decomposition and the whole call on planted data."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import essential_oracle as eo
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("cs_verify_essential", "cs_verify_essential_host", "cs_verify_essential_stats", "cs_verify_essential_models")
CS_E_ARG = -2
REC = 576
W, H_ = 1920, 1080
K1 = np.array([[1500.0, 0.0, 960.0], [0.0, 1380.0, 540.0], [0.0, 0.0, 1.0]])
K2 = np.array([[1250.0, 2.0, 1000.0], [0.0, 1300.0, 520.0], [0.0, 0.0, 1.0]])       # fx != fy, a small skew


def _rotation(a):
    th = np.linalg.norm(a)
    Ax = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(th) / th * Ax + (1 - np.cos(th)) / th ** 2 * Ax @ Ax


def skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def calibrated_views(n, seed, motion="sideways", planar=False):
    """Exact correspondences of random 3-D points (or points on a plane) seen by two 1920x1080 cameras with the
    intrinsics K1, K2.  motion: "sideways" (t mostly along x), "forward" (t mostly along z: the epipole lies inside
    both images) or "rotation" (t = 0).  Only points inside both images are kept.  Returns (x1, x2 [n, 2], R, unit t,
    E = [t]x R), with X2 = R X1 + t."""
    rng = np.random.default_rng(seed)
    R = _rotation(rng.normal(0, 0.05, 3))
    t = {"sideways": np.array([1.0, 0.1, 0.05]), "forward": np.array([0.05, 0.02, 1.0]),
         "rotation": np.zeros(3)}[motion] + (rng.normal(0, 0.03, 3) if motion != "rotation" else 0.0)
    m = 20 * n
    if planar:
        nrm, d = np.array([0.1, -0.05, 1.0]), 8.0
        xy = rng.uniform([-5, -3], [5, 3], (m, 2))
        X = np.column_stack([xy, (d - nrm[0] * xy[:, 0] - nrm[1] * xy[:, 1]) / nrm[2]])
    else:
        X = np.column_stack([rng.uniform(-5, 5, m), rng.uniform(-3, 3, m), rng.uniform(6, 14, m)])
    p1, p2 = X @ K1.T, (X @ R.T + t) @ K2.T
    x1, x2 = p1[:, :2] / p1[:, 2:], p2[:, :2] / p2[:, 2:]
    inside = (x1 >= 0).all(1) & (x1 < [W, H_]).all(1) & (x2 >= 0).all(1) & (x2 < [W, H_]).all(1) & (p2[:, 2] > 0)
    x1, x2 = x1[inside][:n], x2[inside][:n]
    assert len(x1) == n
    tn = t / np.linalg.norm(t) if motion != "rotation" else t
    return x1, x2, R, tn, skew(tn) @ R


def test_symbols_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for name in NEW:
        assert name in declared and name in exported, name
        assert hasattr(cs.lib(), name)
    for name in ("VerifyEssential", "verify_essential_host", "essential_stats", "essential_to_fundamental"):
        assert name in cs.__all__ and callable(getattr(cs, name)), name


# ---- argument checks --------------------------------------------------------------------------------------------------
def _buffers():
    buf = np.zeros(8 * REC + 256 + 16, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    s1, s2 = base, base + 4 * REC
    pairs = base + 8 * REC
    return buf, s1, s2, pairs, pairs + 64


def _cases(s1, s2, pr, inl):
    nan, inf = float("nan"), float("inf")
    ok = dict(s1=s1, n1=4, s2=s2, n2=4, pairs=pr, np=4, K1="K1", K2="K2", loops=64, thresh=4.0, seed=0, E="E", R="R",
              t="t", inl=inl, mi=4)
    bad = []
    for name, K in (("K1", K1), ("K2", K2)):
        for what, k, v in (("K[3] != 0", 3, 0.5), ("K[6] != 0", 6, 1e-3), ("K[7] != 0", 7, -1.0), ("K[8] != 1", 8, 2.0),
                           ("fx = 0", 0, 0.0), ("fx < 0", 0, -100.0), ("fy = 0", 4, 0.0), ("fy < 0", 4, -5.0),
                           ("NaN entry", 2, nan), ("inf skew", 1, inf)):
            M = K.copy()
            M.reshape(-1)[k] = v
            bad.append(("%s %s" % (name, what), {name: M}))
        bad.append(("NULL " + name, {name: None}))
    cases = bad + [
        ("n1 < 0", dict(n1=-1)), ("n2 < 0", dict(n2=-2)), ("NULL set 1", dict(s1=None)), ("NULL set 2", dict(s2=None)),
        ("numPairs < 0", dict(np=-1)), ("NULL pairs", dict(pairs=None)),
        ("numLoops 0", dict(loops=0)), ("numLoops 65537", dict(loops=65537)),
        ("thresh 0", dict(thresh=0.0)), ("thresh < 0", dict(thresh=-1.0)), ("thresh NaN", dict(thresh=nan)),
        ("thresh inf", dict(thresh=inf)), ("NULL E_out", dict(E=None)), ("NULL R_out", dict(R=None)),
        ("NULL t_out", dict(t=None)), ("maxInliers < 0", dict(mi=-1)), ("NULL inliers", dict(inl=None)),
        ("pairs unaligned", dict(pairs=pr + 4)), ("inliers unaligned", dict(inl=inl + 4)),
        ("pairs inside set 1", dict(pairs=s1 + 8)), ("inliers inside set 2", dict(inl=s2 + 3 * REC)),
        ("pairs and inliers overlap", dict(inl=pr + 8)),
    ]
    return ok, cases


def _args(a, out):
    """The C arguments of case a: a string names an array of out, an array is passed as is (kept alive in out)."""
    def mat(v):
        if isinstance(v, str):
            return out[v].ctypes.data
        if v is None:
            return None
        out.setdefault("keep", []).append(np.ascontiguousarray(v, np.float64))
        return out["keep"][-1].ctypes.data
    return (a["s1"], a["n1"], a["s2"], a["n2"], a["pairs"], a["np"], mat(a["K1"]), mat(a["K2"]), a["loops"], a["thresh"],
            a["seed"], mat(a["E"]), mat(a["R"]), mat(a["t"]), a["inl"], a["mi"])


def _outputs():
    return {"K1": np.ascontiguousarray(K1), "K2": np.ascontiguousarray(K2), "E": np.full(9, 7.0), "R": np.full(9, 7.0),
            "t": np.full(3, 7.0)}


@pytest.mark.parametrize("entry", ("cs_verify_essential", "cs_verify_essential_host"))
def test_invalid_arguments_return_cs_e_arg(entry):
    """Every invalid argument fails with CS_E_ARG, and *ms is reset, whether or not a device is present."""
    buf, s1, s2, pr, inl = _buffers()
    f = getattr(cs.lib(), entry)
    ok, cases = _cases(s1, s2, pr, inl)
    out = _outputs()
    for what, change in cases:
        a = dict(ok, **change)
        ms = ctypes.c_double(-1.0)
        assert f(*_args(a, out), ctypes.byref(ms)) == CS_E_ARG, (entry, what)
        msg = cs.lib().cs_last_error().decode()
        assert "invalid argument" in msg and "CS_E_ARG" in msg, (entry, what, msg)
        assert ms.value == 0.0, (entry, what)
    assert not buf.any() and (out["E"] == 7.0).all() and (out["R"] == 7.0).all() and (out["t"] == 7.0).all()


def test_models_entry_rejects_the_same_arguments():
    _, s1, s2, pr, inl = _buffers()
    ok, cases = _cases(s1, s2, pr, inl)
    out = _outputs()
    res = np.zeros(9 * 10 * 64), np.zeros(10 * 64, np.int32), np.zeros(5)
    ptrs = [r.ctypes.data for r in res]
    for what, change in cases:
        if set(change) & {"E", "R", "t", "inl", "mi"}:
            continue                                  # the models hook has no E / R / t / inlier arguments
        a = dict(ok, **change)
        assert cs.lib().cs_verify_essential_models(*_args(a, out)[:11], *ptrs) == CS_E_ARG, what
    a = _args(ok, out)[:11]
    assert cs.lib().cs_verify_essential_models(*a, None, ptrs[1], ptrs[2]) == CS_E_ARG


@pytest.mark.parametrize("entry", ("cs_verify_essential", "cs_verify_essential_host"))
def test_no_pairs_returns_zero_before_any_cuda_call(entry):
    _, s1, s2, _, _ = _buffers()
    out = _outputs()
    ms = ctypes.c_double(-1.0)
    f = getattr(cs.lib(), entry)
    ptr = lambda k: out[k].ctypes.data                                  # noqa: E731
    assert f(s1, 4, s2, 4, None, 0, ptr("K1"), ptr("K2"), 16, 2.0, 5, ptr("E"), ptr("R"), ptr("t"), None, 0,
             ctypes.byref(ms)) == 0
    assert ms.value == 0.0 and not out["E"].any() and not out["R"].any() and not out["t"].any()
    assert f(None, 0, None, 0, None, 0, ptr("K1"), ptr("K2"), 1, 1.0, 0, ptr("E"), ptr("R"), ptr("t"), None, 0,
             None) == 0


class _FakeLib:
    """Records the calls the wrappers make instead of reaching the library."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            return 4096 + 1024 * len(self.calls) if name == "cs_device_alloc" else 0
        return f


def test_wrappers_on_empty_inputs(monkeypatch):
    """The host wrapper on no pairs reaches the library (no CUDA call is made); the device wrapper is checked through a
    stand-in library.  Both return float64 E, R (3x3), t (3) and int32 [0, 2] inliers."""
    E, R, t, inl, ms = cs.verify_essential_host(np.zeros(3, cs.SIFT_DTYPE), np.zeros(2, cs.SIFT_DTYPE),
                                                np.zeros((0, 2), np.int32), K1, K2)
    assert E.shape == (3, 3) and R.shape == (3, 3) and t.shape == (3,) and inl.shape == (0, 2)
    assert E.dtype == R.dtype == t.dtype == np.float64 and inl.dtype == np.int32 and ms == 0.0
    assert not E.any() and not R.any() and not t.any()
    with pytest.raises(cs.CudaSiftError, match="invalid argument"):
        cs.verify_essential_host(np.zeros(3, cs.SIFT_DTYPE), np.zeros(3, cs.SIFT_DTYPE), [[0, 0]], K1, np.eye(3) * 2)
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    d1, d2 = cs.SiftData(), cs.SiftData()
    d1._buf, d2._buf = cs.DeviceBuffer(64), cs.DeviceBuffer(64)
    d1.numPts, d2.numPts = 7, 5
    E, R, t, inl, ms = cs.VerifyEssential(d1, d2, np.zeros((0, 2)), K1, K2, numLoops=100, thresh=1.5, seed=9)
    (name, a), = [c for c in fake.calls if c[0] == "cs_verify_essential"]
    assert a[1] == 7 and a[3] == 5 and a[4] is None and a[5] == 0 and a[8] == 100 and a[9] == pytest.approx(1.5)
    assert a[10] == 9 and a[14] is None and a[15] == 0
    assert E.shape == (3, 3) and R.shape == (3, 3) and t.shape == (3,) and inl.shape == (0, 2) and inl.dtype == np.int32
    fake.calls.clear()
    cs.essential_stats()
    assert fake.calls[0][0] == "cs_verify_essential_stats"
    d1._buf = d2._buf = None


def test_essential_to_fundamental():
    x1, x2, R, t, E = calibrated_views(50, 3)
    F = cs.essential_to_fundamental(E, K1, K2)
    assert abs(np.linalg.norm(F) - 1) < 1e-12 and F.reshape(-1)[np.argmax(np.abs(F))] > 0
    h1, h2 = np.column_stack([x1, np.ones(50)]), np.column_stack([x2, np.ones(50)])
    assert np.abs(np.einsum("ij,jk,ik->i", h2, F, h1)).max() < 1e-9
    assert not cs.essential_to_fundamental(np.zeros((3, 3)), K1, K2).any()


# ---- the oracle on its own --------------------------------------------------------------------------------------------
def _solutions(x1, x2):
    q = eo.calibrated(np.column_stack([x1, x2]), K1, K2)
    return q, [eo.unit_sign(e) for e in eo.solve_e5(q)]


def _check_constraints(q, Es, tol):
    h1, h2 = np.column_stack([q[:, :2], np.ones(len(q))]), np.column_stack([q[:, 2:], np.ones(len(q))])
    for e in Es:
        assert np.abs(np.einsum("ij,jk,ik->i", h2, e, h1)).max() < 1e-9          # the five epipolar equations
        assert abs(np.linalg.det(e)) < tol
        assert np.abs(2 * e @ e.T @ e - np.trace(e @ e.T) * e).max() < tol


def test_five_point_recovers_planted_e_sideways():
    """Exact samples of sideways motion: one solution is the planted E to 1e-9 (after the output scaling) -- to 1e-6
    where the planted root is nearly double and the polynomial is flat there, as for the 7-point solver -- and every
    solution satisfies the epipolar equations to 1e-9, det E = 0 and the trace constraint to 1e-7 (the other roots of
    the degree-10 polynomial are less well conditioned than the planted one)."""
    errs = []
    for seed in range(40):
        x1, x2, _, _, E = calibrated_views(5, seed, "sideways")
        q, Es = _solutions(x1, x2)
        assert 1 <= len(Es) <= 10
        errs.append(min(eo.same_e(e, E) for e in Es))
        _check_constraints(q, Es, 1e-7)
    errs = np.array(errs)
    assert (errs < 1e-6).all() and (errs < 1e-9).mean() >= 0.9, errs


def _planted_root_gap(q, E):
    """The distance of the planted solution's z (in the solver's chart) to the nearest other root of the degree-10
    polynomial, complex roots included, relative to 1 + |z|."""
    import verify_oracle as vo
    N = eo.basis(vo.nullspace([vo.f_row(*r) for r in q]))
    c = np.linalg.lstsq(np.column_stack(list(N)), E.reshape(-1), rcond=None)[0]
    z = c[2] / c[3]
    d = eo.det_polynomial(eo.hidden_matrix(eo.gauss_jordan(eo.constraint_matrix(N))))
    return float(np.sort(np.abs(np.roots(d[::-1]) - z))[1] / (1 + abs(z)))


def test_five_point_recovers_planted_e_forward():
    """Exact samples of forward motion, the epipole inside both images.  Forward motion clusters the roots of the
    degree-10 polynomial around the planted one.  Where another root lies within 1e-2 (relative) of it, the root is
    nearly double: measured on these 40 seeds, the two samples whose planted E is missed (gaps 6e-4 and 3e-3, np.roots
    returns the planted root as a complex pair or merges it with its neighbour) are such cases.  Every sample with a
    separated planted root recovers it to 1e-6, most of them to 1e-9; the 1e-8 to 1e-6 errors of the rest are the
    conditioning of the hidden-variable back-substitution for forward motion (DESIGN.md section 4)."""
    errs, gaps = [], []
    for seed in range(40):
        x1, x2, _, _, E = calibrated_views(5, seed, "forward")
        e2 = K2 @ np.linalg.svd(E.T)[2][-1]                                 # the epipole in image 2: E^T e2 = 0
        assert 0 <= e2[0] / e2[2] < W and 0 <= e2[1] / e2[2] < H_
        q, Es = _solutions(x1, x2)
        assert len(Es) >= 1
        errs.append(min(eo.same_e(e, E) for e in Es))
        gaps.append(_planted_root_gap(q, E))
    errs, gaps = np.array(errs), np.array(gaps)
    separated = gaps > 1e-2
    assert separated.sum() >= 30 and (errs[separated] < 1e-6).all(), (errs, gaps)
    assert (errs[separated] < 1e-9).mean() >= 0.6, (errs, gaps)


def test_pose_decomposition_recovers_planted_pose():
    for motion in ("sideways", "forward"):
        for seed in range(5):
            x1, x2, R, t, E = calibrated_views(100, seed, motion)
            q = eo.calibrated(np.column_stack([x1, x2]), K1, K2)
            Rg, tg, front, runner = eo.choose_pose(eo.unit_sign(E), q)
            assert np.abs(Rg - R).max() < 1e-9 and np.abs(tg - t).max() < 1e-9, (motion, seed)
            assert abs(np.linalg.det(Rg) - 1) < 1e-12 and front == 100 and runner < 100
            Ex = skew(tg) @ Rg
            assert abs(abs(np.sum(Ex * eo.unit_sign(E))) / np.linalg.norm(Ex) - 1) < 1e-12


def test_oracle_verify_on_planted_data():
    """The whole restatement on exact data with outliers: the planted E, pose and inliers."""
    rng = np.random.default_rng(4)
    x1, x2, R, t, E = calibrated_views(200, 11)
    out = rng.random(200) < 0.3
    x2[out] = rng.uniform([0, 0], [W, H_], (out.sum(), 2))
    pairs = np.column_stack([np.arange(200), np.arange(200)])
    Eg, Rg, tg, inl, best, cnt = eo.verify(x1[:, 0], x1[:, 1], x2[:, 0], x2[:, 1], pairs, 200, 200, K1, K2, 64, 1.0, 3)
    assert eo.same_e(Eg, E) < 1e-6 and best >= 0 and cnt >= (~out).sum()
    assert np.abs(Rg - R).max() < 1e-6 and np.abs(tg - t).max() < 1e-6
    want = np.nonzero(eo.residuals(E, K1, K2, np.column_stack([x1, x2])) < 1.0)[0]
    assert np.array_equal(inl[:, 0], want)
