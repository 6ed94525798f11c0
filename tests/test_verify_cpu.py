"""CPU checks of geometric verification (cs_verify_pairs, cs_verify_pairs_host, cs_verify_stats, cs_verify_models): the
entry points exist, they reject bad arguments before any CUDA call, the Python wrappers pass their arguments through,
and the float64 restatement (tests/verify_oracle.py) is right on its own: the sampler, and both minimal solvers on
exact synthetic correspondences (and against OpenCV's 7-point solver when cv2 imports)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import verify_oracle as vo
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("cs_verify_pairs", "cs_verify_pairs_host", "cs_verify_stats", "cs_verify_models")
CS_E_ARG = -2
REC = 576


def test_symbols_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for name in NEW:
        assert name in declared and name in exported, name
        assert hasattr(cs.lib(), name)
    for name in ("VerifyPairs", "verify_pairs_host", "verify_stats"):
        assert name in cs.__all__ and callable(getattr(cs, name)), name
    assert "#define CS_GEOM_HOMOGRAPHY  1" in header and "#define CS_GEOM_FUNDAMENTAL 2" in header
    assert build.SOURCES.count("verify.cu") == 1


def _layout(base):
    """Two sets of 4 records, then 8-byte aligned room for 4 pairs and 4 inliers."""
    s1, s2 = base, base + 4 * REC
    pairs = base + 8 * REC
    return s1, s2, pairs, pairs + 64


def _bad(base):
    s1, s2, pr, inl = _layout(base)
    nan, inf = float("nan"), float("inf")
    M = "model_out"           # replaced by a real buffer in the test
    ok = dict(s1=s1, n1=4, s2=s2, n2=4, pairs=pr, np=4, model=2, loops=64, thresh=4.0, seed=0, out=M, inl=inl, mi=4)
    cases = [
        ("n1 < 0", dict(n1=-1)), ("n2 < 0", dict(n2=-2)), ("NULL set 1", dict(s1=None)), ("NULL set 2", dict(s2=None)),
        ("numPairs < 0", dict(np=-1)), ("NULL pairs", dict(pairs=None)),
        ("model 0", dict(model=0)), ("model 3", dict(model=3)),
        ("numLoops 0", dict(loops=0)), ("numLoops 65537", dict(loops=65537)),
        ("thresh 0", dict(thresh=0.0)), ("thresh < 0", dict(thresh=-1.0)), ("thresh NaN", dict(thresh=nan)),
        ("thresh inf", dict(thresh=inf)), ("NULL model_out", dict(out=None)),
        ("maxInliers < 0", dict(mi=-1)), ("NULL inliers", dict(inl=None)),
        ("pairs unaligned", dict(pairs=pr + 4)), ("inliers unaligned", dict(inl=inl + 4)),
        ("pairs inside set 1", dict(pairs=s1 + 8)), ("inliers inside set 2", dict(inl=s2 + 3 * REC)),
        ("pairs and inliers overlap", dict(inl=pr + 8)),
    ]
    return ok, cases


def _args(a, model_out):
    return (a["s1"], a["n1"], a["s2"], a["n2"], a["pairs"], a["np"], a["model"], a["loops"], a["thresh"], a["seed"],
            model_out if a["out"] == "model_out" else a["out"], a["inl"], a["mi"])


@pytest.mark.parametrize("entry", ("cs_verify_pairs", "cs_verify_pairs_host"))
def test_invalid_arguments_return_cs_e_arg(entry):
    """Every invalid argument fails with CS_E_ARG, and *ms is reset, whether or not a device is present."""
    buf = np.zeros(8 * REC + 256 + 16, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    f = getattr(cs.lib(), entry)
    ok, cases = _bad(base)
    model = np.full(9, 7.0)
    for what, change in cases:
        a = dict(ok, **change)
        ms = ctypes.c_double(-1.0)
        assert f(*_args(a, model.ctypes.data), ctypes.byref(ms)) == CS_E_ARG, (entry, what)
        msg = cs.lib().cs_last_error().decode()
        assert "invalid argument" in msg and "CS_E_ARG" in msg, (entry, what, msg)
        assert ms.value == 0.0, (entry, what)
    assert not buf.any() and (model == 7.0).all()


def test_models_entry_rejects_the_same_arguments():
    buf = np.zeros(8 * REC + 256 + 16, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    ok, cases = _bad(base)
    out = np.zeros(9 * 3 * 64), np.zeros(3 * 64, np.int32), np.zeros(5)
    ptrs = [a.ctypes.data for a in out]
    for what, change in cases:
        if set(change) & {"out", "inl", "mi"}:
            continue                                  # cs_verify_models has no model_out / inlier arguments
        a = dict(ok, **change)
        assert cs.lib().cs_verify_models(*_args(a, 0)[:10], *ptrs) == CS_E_ARG, what
    a = _args(ok, 0)[:10]
    assert cs.lib().cs_verify_models(*a, None, ptrs[1], ptrs[2]) == CS_E_ARG


@pytest.mark.parametrize("entry", ("cs_verify_pairs", "cs_verify_pairs_host"))
def test_no_pairs_returns_zero_before_any_cuda_call(entry):
    buf = np.zeros(8 * REC + 256 + 16, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    s1, s2, _, _ = _layout(base)
    model = np.full(9, 7.0)
    ms = ctypes.c_double(-1.0)
    f = getattr(cs.lib(), entry)
    assert f(s1, 4, s2, 4, None, 0, 1, 16, 2.0, 5, model.ctypes.data, None, 0, ctypes.byref(ms)) == 0
    assert ms.value == 0.0 and not model.any()
    assert f(None, 0, None, 0, None, 0, 2, 1, 1.0, 0, model.ctypes.data, None, 0, None) == 0
    # the records may overlap each other: they are only read
    assert f(s1, 4, s1 + REC, 3, None, 0, 2, 1, 1.0, 0, model.ctypes.data, None, 0, None) == 0


class _FakeLib:
    """Records the calls the wrappers make instead of reaching the library."""

    def __init__(self, count=3):
        self.calls = []
        self.count = count

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            if name == "cs_device_alloc":
                return 4096 + 1024 * len(self.calls)
            if name in ("cs_verify_pairs", "cs_verify_pairs_host"):
                return self.count
            return 0
        return f


def test_wrappers_map_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    d1, d2 = cs.SiftData(), cs.SiftData()
    d1._buf, d2._buf = cs.DeviceBuffer(64), cs.DeviceBuffer(64)
    d1.numPts, d2.numPts = 7, 5
    pairs = np.array([[0, 1], [2, 3], [4, 4], [6, 0]], np.int64)
    model, inl, ms = cs.VerifyPairs(d1, d2, pairs, model="homography", numLoops=100, thresh=1.5, seed=9)
    (name, a), = [c for c in fake.calls if c[0] == "cs_verify_pairs"]
    assert a[0] == d1.d_data and a[1] == 7 and a[2] == d2.d_data and a[3] == 5
    assert a[5] == 4 and a[6] == 1 and a[7] == 100 and a[8] == pytest.approx(1.5) and a[9] == 9 and a[12] == 4
    assert a[4] != a[11] and a[4] and a[11]
    uploads = [c for c in fake.calls if c[0] == "cs_memcpy_h2d"]
    assert len(uploads) == 1 and uploads[0][1][2] == 32                 # the pairs, as int32
    assert model.shape == (3, 3) and model.dtype == np.float64 and inl.shape == (3, 2) and inl.dtype == np.int32
    fake.calls.clear()
    cs.VerifyPairs(d1, d2, pairs)                                        # defaults: F, 4096 trials, 4 px, seed 0
    (name, a), = [c for c in fake.calls if c[0] == "cs_verify_pairs"]
    assert a[6] == 2 and a[7] == 4096 and a[8] == pytest.approx(4.0) and a[9] == 0
    d1._buf = d2._buf = None
    fake.calls.clear()
    fake.count = 2
    model, inl, ms = cs.verify_pairs_host(np.zeros(9, cs.SIFT_DTYPE), np.zeros(4, cs.SIFT_DTYPE), pairs, 2, 50, 3.0, 1)
    (name, a), = fake.calls
    assert name == "cs_verify_pairs_host" and a[1] == 9 and a[3] == 4 and a[5] == 4
    assert a[6] == 2 and a[7] == 50 and a[8] == pytest.approx(3.0) and a[9] == 1 and a[12] == 4
    assert inl.shape == (2, 2)
    fake.calls.clear()
    cs.verify_stats()
    assert fake.calls[0][0] == "cs_verify_stats"
    with pytest.raises(ValueError):
        cs.VerifyPairs(d1, d2, pairs, model="essential")


def test_python_wrapper_raises_on_rejection():
    with pytest.raises(cs.CudaSiftError, match="invalid argument"):
        cs.verify_pairs_host(np.zeros(3, cs.SIFT_DTYPE), np.zeros(3, cs.SIFT_DTYPE), [[0, 0]], thresh=-1.0)
    with pytest.raises(cs.CudaSiftError, match="invalid argument"):
        cs.verify_pairs_host(np.zeros(3, cs.SIFT_DTYPE), np.zeros(3, cs.SIFT_DTYPE), [[0, 0]], numLoops=0)


# ---- the oracle on its own --------------------------------------------------------------------------------------------
def test_sampler_is_splitmix64_and_draws_distinct_indices():
    assert int(vo.splitmix64(np.uint64(0))) == 0xE220A8397B1DCDAF        # splitmix64's first output from state 0
    for n, k in ((7, 7), (10, 7), (4, 4), (1000, 7), (2 ** 20, 4)):
        s = vo.samples(12345, 300, n, k)
        ok = s[:, 0] >= 0
        assert ok.mean() > 0.99
        assert ((s[ok] >= 0) & (s[ok] < n)).all()
        assert all(len(set(r)) == k for r in s[ok])
    assert (vo.samples(1, 10, 6, 7) == -1).all()                         # fewer valid pairs than the sample size
    a, b = vo.samples(1, 50, 500, 7), vo.samples(2, 50, 500, 7)
    assert not np.array_equal(a, b) and np.array_equal(a, vo.samples(1, 50, 500, 7))


def planted_views(n, seed, planar=False):
    """Exact correspondences of random 3-D points (or points on a plane) seen by two 1920x1080 cameras: (x1, x2 [n, 2],
    the planted F, the planted H when planar)."""
    rng = np.random.default_rng(seed)
    K = np.array([[1400.0, 0, 960], [0, 1400.0, 540], [0, 0, 1]])
    a = rng.normal(0, 0.08, 3)
    Ax = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    R = np.eye(3) + np.sin(np.linalg.norm(a)) / np.linalg.norm(a) * Ax + \
        (1 - np.cos(np.linalg.norm(a))) / np.linalg.norm(a) ** 2 * Ax @ Ax
    t = np.array([1.0, 0.2, 0.1]) + rng.normal(0, 0.05, 3)
    if planar:
        nrm, d = np.array([0.1, -0.05, 1.0]), 8.0
        xy = rng.uniform([-4, -2.5], [4, 2.5], (n, 2))
        X = np.column_stack([xy, (d - nrm[0] * xy[:, 0] - nrm[1] * xy[:, 1]) / nrm[2]])
        H = K @ (R + np.outer(t, nrm) / d) @ np.linalg.inv(K)
    else:
        X = np.column_stack([rng.uniform(-4, 4, n), rng.uniform(-2.5, 2.5, n), rng.uniform(6, 14, n)])
        H = None
    p1 = X @ K.T
    p2 = (X @ R.T + t) @ K.T
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    F = np.linalg.inv(K).T @ tx @ R @ np.linalg.inv(K)
    return p1[:, :2] / p1[:, 2:], p2[:, :2] / p2[:, 2:], F, (H / H[2, 2] if planar else None)


def _normalised(x1, x2):
    p = np.column_stack([x1, x2])
    c1, c2, s = vo.normalisation(p)
    return (p - np.concatenate([c1, c2])) * s, c1, c2, s


def test_seven_point_recovers_planted_f():
    """One root is the planted F to 1e-9 relative.  Where the planted root is nearly double, the determinant is flat
    there and the root is only good to about 1e-8: seed 19 (pencil roots 0.992618 and 0.992633) is such a case."""
    errs = []
    for seed in range(40):
        x1, x2, F, _ = planted_views(7, seed)
        u, c1, c2, s = _normalised(x1, x2)
        Fs = [vo.denormalise(m, vo.FUNDAMENTAL, c1, c2, s) for m in vo.solve_f7(u)]
        assert 1 <= len(Fs) <= 3
        errs.append(min(vo.same_model(f, F, vo.FUNDAMENTAL) for f in Fs))
        for f in Fs:                                                       # every root fits the seven points
            assert vo.residuals(f, vo.FUNDAMENTAL, np.column_stack([x1, x2])).max() < 1e-6
            assert abs(np.linalg.det(f)) < 1e-9
    errs = np.array(errs)
    assert (errs < 1e-7).all() and (errs >= 1e-9).sum() <= 1, errs


def test_four_point_recovers_planted_h():
    for seed in range(5):
        x1, x2, _, H = planted_views(4, seed, planar=True)
        u, c1, c2, s = _normalised(x1, x2)
        h = vo.solve_h4(u)
        assert h is not None
        assert vo.same_model(vo.denormalise(h, vo.HOMOGRAPHY, c1, c2, s), H, vo.HOMOGRAPHY) < 1e-9, seed


def test_degenerate_minimal_samples():
    x1, x2, _, _ = planted_views(4, 3, planar=True)
    x1[2] = 0.5 * (x1[0] + x1[1])                                          # three collinear points in image 1
    u, _, _, _ = _normalised(x1, x2)
    assert vo.solve_h4(u) is None
    x1, x2, _, _ = planted_views(7, 3)
    u, _, _, _ = _normalised(np.repeat(x1[:1], 7, 0), x2)                  # image 1: one point seven times
    assert vo.solve_f7(u) == []


def test_cubic_roots_cover_the_cases():
    assert sorted(vo.cubic_roots([-6.0, 11.0, -6.0, 1.0])) == pytest.approx([1.0, 2.0, 3.0])
    assert vo.cubic_roots([1.0, 0.0, 0.0, 1.0]) == pytest.approx([-1.0])
    assert sorted(vo.cubic_roots([2.0, -3.0, 1.0, 1e-14])) == pytest.approx([1.0, 2.0])   # vanishing leading coefficient
    assert vo.cubic_roots([3.0, -1.5, 0.0, 0.0]) == pytest.approx([2.0])
    assert vo.cubic_roots([0.0, 0.0, 0.0, 0.0]) == []


def test_seven_point_matches_opencv():
    cv2 = pytest.importorskip("cv2")
    for seed in range(5):
        x1, x2, _, _ = planted_views(7, 100 + seed)
        x2 = x2 + np.random.default_rng(seed).normal(0, 0.3, x2.shape)     # not an exact F: three roots are common
        u, c1, c2, s = _normalised(x1, x2)
        ours = [vo.denormalise(m, vo.FUNDAMENTAL, c1, c2, s) for m in vo.solve_f7(u)]
        theirs, _ = cv2.findFundamentalMat(x1.astype(np.float64), x2.astype(np.float64), cv2.FM_7POINT)
        theirs = [] if theirs is None else [theirs[3 * k:3 * k + 3] for k in range(len(theirs) // 3)]
        assert len(ours) == len(theirs), seed
        for f in theirs:
            assert min(vo.same_model(o, f, vo.FUNDAMENTAL) for o in ours) < 1e-5, seed


def test_oracle_verify_on_planted_data():
    """The whole restatement on exact data with outliers: the planted model and exactly the planted inliers."""
    rng = np.random.default_rng(4)
    for planar, model in ((False, vo.FUNDAMENTAL), (True, vo.HOMOGRAPHY)):
        x1, x2, F, H = planted_views(200, 11, planar)
        out = rng.random(200) < 0.3
        x2[out] = rng.uniform([0, 0], [1920, 1080], (out.sum(), 2))
        pairs = np.column_stack([np.arange(200), np.arange(200)])
        M, inl, best, cnt = vo.verify(x1[:, 0], x1[:, 1], x2[:, 0], x2[:, 1], pairs, 200, 200, model, 256, 1.0, 3)
        want = F if model == vo.FUNDAMENTAL else H
        assert vo.same_model(M, want, model) < 1e-6
        assert best >= 0 and cnt >= (~out).sum()
        assert np.array_equal(inl[:, 0], np.nonzero(vo.residuals(want, model, np.column_stack([x1, x2])) < 1.0)[0])
