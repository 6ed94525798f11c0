"""CPU checks of camera registration (cs_absolute_pose_batch): the entry points are declared, exported and typed, every
invalid argument is rejected with the offending job named before any CUDA call, numJobs == 0 returns 0 without a
device, the numpy statement's P3P (pose_oracle) recovers the true pose of noise-free samples among its solutions and
agrees with OpenCV's solveP3P where it is installed, its refinement converges to the truth from a perturbed start, and
the Python wrapper builds its tables."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import pose_cases as pc
import pose_oracle as po
import triangulate_cases as tc
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_E_ARG = -2
RECORD = 576


def test_symbols_declared_exported_and_typed():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for name in ("cs_absolute_pose_batch", "cs_absolute_pose_models"):
        assert name in declared and name in exported, name
    f = cs.lib().cs_absolute_pose_batch
    assert f.restype is ctypes.c_int and len(f.argtypes) == 12 and f.argtypes[6] is ctypes.c_double
    g = cs.lib().cs_absolute_pose_models
    assert g.restype is ctypes.c_int and len(g.argtypes) == 9 and g.argtypes[5] is ctypes.c_double
    assert ctypes.sizeof(cs.PoseJob) == 48 and cs.PoseJob.seed.offset == 24
    for name in ("PoseJob", "AbsolutePoseBatch"):
        assert name in cs.__all__ and hasattr(cs, name)


class Arena:
    """Host memory laid out as on the device: two jobs of 4 records, their pointOf, errors and inlier buffers and 4
    points.  Nothing is dereferenced: every case fails its checks."""

    def __init__(self):
        self.buf = np.zeros(2 * 4 * RECORD + 4096, np.uint8)
        base = self.buf.ctypes.data + (-self.buf.ctypes.data) % 64
        self.pts = [base, base + 4 * RECORD]
        o = base + 8 * RECORD
        self.pointOf = [o, o + 16]
        self.errors = [o + 32, o + 48]
        self.inlier = [o + 64, o + 72]
        self.points = o + 128

    def common(self):
        K = np.array([[800.0, 1.0, 640], [0, 790, 480], [0, 0, 1]])
        jobs = [dict(pts=self.pts[p], n=4, pointOf=self.pointOf[p], seed=p, errors=self.errors[p],
                     inlier=self.inlier[p]) for p in range(2)]
        return dict(points=self.points, numPoints=4, jobs=jobs, Ks=np.stack([K, K]), numLoops=64, maxError=4.0,
                    out=True)


def _call(c):
    J = c.get("numJobs", len(c["jobs"]))
    table = (cs.PoseJob * max(len(c["jobs"]), 1))(*[cs.PoseJob(j["pts"], j["n"], j["pointOf"], j["seed"], j["errors"],
                                                                j["inlier"]) for j in c["jobs"]])
    K = np.ascontiguousarray(c["Ks"], np.float64)
    R, t = np.full((2, 9), 5.0), np.full((2, 3), 5.0)
    counts, stats = np.full(2, 7, np.int32), np.full((2, 8), 7, np.int64)
    ms = ctypes.c_double(-1.0)
    o = c["out"]
    r = cs.lib().cs_absolute_pose_batch(c["points"], c["numPoints"], table if c.get("jobsPtr", 1) else None, J,
                                        K.ctypes.data if c.get("KPtr", 1) else None, c["numLoops"], c["maxError"],
                                        R.ctypes.data if o else None, t.ctypes.data, counts.ctypes.data,
                                        stats.ctypes.data, ctypes.byref(ms))
    return r, ms.value, (R, t, counts, stats)


def _expect(r, ms, outs, what, name):
    assert r == CS_E_ARG, (what, r)
    msg = cs.lib().cs_last_error().decode()
    assert "invalid argument" in msg and "CS_E_ARG" in msg, (what, msg)
    assert name in msg, (what, name, msg)
    assert ms == 0.0, what
    R, t, counts, stats = outs
    assert (R == 5).all() and (t == 5).all() and (counts == 7).all() and (stats == 7).all(), what


def test_rejects_every_invalid_argument():
    a = Arena()
    nan, inf = float("nan"), float("inf")

    def job(p, **kw):
        c = a.common()
        c["jobs"][p].update(kw)
        return dict(jobs=c["jobs"])

    def K(**kw):
        k = a.common()["Ks"].copy()
        for key, v in kw.items():
            k[1][int(key[1]) // 3, int(key[1]) % 3] = v
        return k

    cases = [
        ("numJobs < 0", dict(numJobs=-1), "numJobs"),
        ("numJobs 65537", dict(numJobs=65537), "numJobs"),
        ("NULL jobs", dict(jobsPtr=0), "jobs"),
        ("NULL Ks", dict(KPtr=0), "Ks"),
        ("numPoints < 0", dict(numPoints=-1), "numPoints"),
        ("NULL points", dict(points=None), "d_points"),
        ("points unaligned", dict(points=a.points + 4), "d_points"),
        ("n < 0", job(1, n=-1), "jobs[1]"),
        ("NULL pts", job(1, pts=None), "jobs[1]"),
        ("NULL pointOf", job(0, pointOf=None), "jobs[0]"),
        ("pointOf unaligned", job(1, pointOf=a.pointOf[1] + 2), "jobs[1]"),
        ("errors unaligned", job(1, errors=a.errors[1] + 1), "jobs[1]"),
        ("K[8] != 1", dict(Ks=K(k8=2.0)), "jobs[1]"),
        ("K[3] != 0", dict(Ks=K(k3=0.5)), "jobs[1]"),
        ("K[4] <= 0", dict(Ks=K(k4=0.0)), "jobs[1]"),
        ("K not finite", dict(Ks=K(k2=nan)), "jobs[1]"),
        ("numLoops 0", dict(numLoops=0), "numLoops"),
        ("numLoops 65537", dict(numLoops=65537), "numLoops"),
        ("maxError 0", dict(maxError=0.0), "maxError"),
        ("maxError inf", dict(maxError=inf), "maxError"),
        ("maxError NaN", dict(maxError=nan), "maxError"),
        ("NULL R_out", dict(out=False), "R_out"),
        ("errors over the other job's errors", job(1, errors=a.errors[0] + 8), "jobs[0].errors and jobs[1].errors"),
        ("inlier over own errors", job(1, inlier=a.errors[1] + 12), "jobs[1].errors and jobs[1].inlier"),
        ("errors over a record range", job(0, errors=a.pts[1] + 4 * RECORD - 8), "jobs[0].errors and jobs[1].pts"),
        ("inlier over pointOf", job(1, inlier=a.pointOf[0] + 8), "jobs[1].inlier and jobs[0].pointOf"),
        ("errors over the points", job(0, errors=a.points + 80), "jobs[0].errors and d_points"),
    ]
    for what, ch, name in cases:
        c = a.common()
        c.update(ch)
        _expect(*_call(c), what, name)
    assert not a.buf.any()
    # inputs may overlap each other (they are only read), touching ranges pass, and an invalid K of an empty job is
    # still an error
    c = a.common()
    c["jobs"][1].update(pointOf=a.pointOf[0], pts=a.pts[0])
    c.update(numJobs=0)
    r, ms, outs = _call(c)
    assert r == 0 and ms == 0.0 and (outs[2] == 7).all()
    c = a.common()
    c["jobs"][1].update(n=0)
    c.update(Ks=K(k0=-1.0))
    _expect(*_call(c), "invalid K of an empty job", "jobs[1]")


def test_no_jobs_and_empty_jobs_return_zero_before_any_cuda_call():
    ms = ctypes.c_double(-1.0)
    L = cs.lib()
    assert L.cs_absolute_pose_batch(None, 0, None, 0, None, 1024, 4.0, None, None, None, None, ctypes.byref(ms)) == 0
    assert ms.value == 0.0
    # only empty jobs: zero outputs and statistics, no CUDA call (this holds without a device)
    K = np.stack([np.array([[800.0, 0, 640], [0, 800, 480], [0, 0, 1]])] * 2)
    table = (cs.PoseJob * 2)(cs.PoseJob(None, 0, None, 1, None, None), cs.PoseJob(None, 0, None, 2, None, None))
    R, t = np.full((2, 9), 5.0), np.full((2, 3), 5.0)
    counts, stats = np.full(2, 7, np.int32), np.full((2, 8), 7, np.int64)
    assert L.cs_absolute_pose_batch(None, 0, table, 2, K.ctypes.data, 16, 2.0, R.ctypes.data, t.ctypes.data,
                                    counts.ctypes.data, stats.ctypes.data, None) == 0
    assert not R.any() and not t.any() and not counts.any() and not stats.any()
    h = np.zeros(64)
    assert L.cs_absolute_pose_models(None, 0, table, K.ctypes.data, 16, 2.0, h.ctypes.data, h.ctypes.data,
                                     h.ctypes.data) == 0


def _sample(rng, noise_free=True):
    K = tc.intrinsics(rng)
    Ks, Rs, ts = tc.cameras(rng, 1)
    R, t = Rs[0], ts[0]
    while True:
        X = rng.uniform(-3, 3, (3, 3))
        if ((X @ R.T + t)[:, 2] > 1).all():
            break
    u = (X @ R.T + t) @ K.T
    return K, R, t, X, u[:, :2] / u[:, 2:]


def test_oracle_p3p_recovers_the_true_pose():
    """From exact (float64) pixels the true pose is among the <= 4 solutions to 1e-8: the solver's FP64 rounding,
    amplified by the conditioning of the sample, stays far below it for these well-spread samples."""
    rng = np.random.default_rng(5)
    found = 0
    for _ in range(200):
        K, R, t, X, px = _sample(rng)
        deg, poses = po.p3p(po.bearings(K, px), X)
        assert not deg and 1 <= len(poses) <= 4
        err = min(np.abs(Rr - R).max() + np.abs(tr - t).max() / np.abs(t).max() for Rr, tr in poses)
        found += err < 1e-8
        for Rr, tr in poses:                       # every solution is a rotation that sees the three points
            assert np.allclose(Rr @ Rr.T, np.eye(3), atol=1e-6) and np.linalg.det(Rr) > 0
            assert ((X @ Rr.T + tr)[:, 2] > 0).all()
    assert found == 200


def test_oracle_p3p_degenerate_samples():
    rng = np.random.default_rng(6)
    K, R, t, X, px = _sample(rng)
    Xc = X.copy()
    Xc[2] = 0.5 * (Xc[0] + Xc[1])                  # collinear world points
    assert po.p3p(po.bearings(K, px), Xc) == (True, [])
    b = po.bearings(K, px)
    b[2] = b[1]                                    # parallel bearings
    assert po.p3p(b, X) == (True, [])


def test_oracle_p3p_agrees_with_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    for _ in range(50):
        K, R, t, X, px = _sample(rng)
        K[0, 1] = 0.0                              # OpenCV's P3P reads fx, fy, cx, cy only: no skew
        u = (X @ R.T + t) @ K.T
        px = u[:, :2] / u[:, 2:]
        _, poses = po.p3p(po.bearings(K, px), X)
        n, rv, tv = cv2.solveP3P(X.reshape(3, 1, 3), px.reshape(3, 1, 2), K, None, flags=cv2.SOLVEPNP_P3P)
        theirs = [(cv2.Rodrigues(r)[0], np.asarray(tt).reshape(3)) for r, tt in zip(rv, tv)]
        # every solution of OpenCV that sees the points is one of ours, and ours hold the truth
        for Rc, tcv in theirs:
            if ((X @ Rc.T + tcv)[:, 2] > 0).all():
                assert min(np.abs(Rr - Rc).max() + np.abs(tr - tcv).max() / np.abs(t).max() for Rr, tr in poses) < 1e-5
        assert min(np.abs(Rr - R).max() for Rr, _ in poses) < 1e-8


def test_oracle_refinement_converges_from_a_perturbed_start():
    rng = np.random.default_rng(8)
    for _ in range(10):
        xy, po_, X, K, R, t = pc.job(rng, 200, noise=0.0, outlier=0.0)
        Xw, px = X[po_], xy.astype(np.float64)
        w = rng.normal(0, 0.02, 3)
        R0, t0 = po._rodrigues(w) @ R, t + rng.normal(0, 0.05, 3)
        R1, t1, acc = po.refine(K, R0, t0, Xw, px)
        assert acc >= 1
        # the records hold float32 positions: about 6e-5 px of rounding, far below 1e-6 of the pose
        assert np.abs(R1 - R).max() < 1e-6 and np.abs(t1 - t).max() < 1e-6 * (1 + np.abs(t).max())


def test_oracle_whole_job_on_a_clean_scene():
    rng = np.random.default_rng(9)
    xy, pointOf, X, K, R, t = pc.job(rng, 300, noise=0.3, outlier=0.3, extra=5)
    o = po.pose_job(xy, pointOf, X, K, numLoops=64, maxError=2.0, seed=3)
    assert o["stats"][0] == 300 and o["stats"][1] == 0 and o["count"] >= 150
    assert np.abs(o["R"] - R).max() < 1e-3 and np.abs(o["t"] - t).max() < 1e-2
    assert np.isnan(o["errors"][pointOf < 0]).all() and not o["inlier"][pointOf < 0].any()
    assert o["inlier"].sum() == o["count"] == o["stats"][7]


class _FakeLib:
    def __init__(self, found=2):
        self.calls, self.found, self.uploads = [], found, {}

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            if name == "cs_absolute_pose_batch":
                J = args[3]
                self.jobs = [cs.PoseJob.from_address(args[2] + k * ctypes.sizeof(cs.PoseJob)) for k in range(J)]
                self.jobs = [(j.pts, j.n, j.pointOf, j.seed, j.errors, j.inlier) for j in self.jobs]
                self.K = np.ctypeslib.as_array((ctypes.c_double * (9 * J)).from_address(args[4].value)).copy()
                return self.found
            if name == "cs_device_alloc":
                return 4096 * (1 + len(self.calls))
            if name == "cs_memcpy_h2d":
                self.uploads[args[0]] = ctypes.string_at(args[1].value, args[2])
            return 0
        return f


class _Data:
    def __init__(self, ptr, n):
        self.d_data, self.numPts = ptr, n


def test_wrapper_builds_its_tables(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    K = np.array([[800.0, 0, 640], [0, 800, 480], [0, 0, 1]])
    pts = np.arange(12, dtype=np.float64).reshape(4, 3)
    pointOfs = [np.array([0, -1, 3]), np.zeros(0, np.int64), np.array([2, 2])]
    R, t, counts, errors, inlier, stats, ms = cs.AbsolutePoseBatch(
        [_Data(4096, 3), _Data(0, 0), _Data(8192, 2)], pointOfs, pts, K, numLoops=32, maxError=2.5, seeds=[7, 8, 9])
    (name, a), = [c for c in fake.calls if c[0] == "cs_absolute_pose_batch"]
    assert a[1] == 4 and a[3] == 3 and a[5:7] == (32, 2.5)
    assert fake.uploads[a[0]] == pts.tobytes()
    j = fake.jobs
    assert [x[1] for x in j] == [3, 0, 2] and [x[3] for x in j] == [7, 8, 9]
    assert j[0][0] == 4096 and j[2][0] == 8192 and j[1][0] is None and j[1][2] is None
    flat = fake.uploads[j[0][2]]
    assert flat == np.array([0, -1, 3, 2, 2], np.int32).tobytes() and j[2][2] == j[0][2] + 12
    assert j[2][4] == j[0][4] + 12 and j[2][5] == j[0][5] + 3
    assert np.array_equal(fake.K, np.concatenate([K.ravel()] * 3))
    assert R.shape == (3, 3, 3) and t.shape == (3, 3) and counts.shape == (3,) and stats.shape == (3, 8)
    assert [e.shape for e in errors] == [(3,), (0,), (2,)] and [i.dtype for i in inlier] == [bool] * 3
    with pytest.raises(ValueError):
        cs.AbsolutePoseBatch([_Data(4096, 3)], [np.zeros(2)], pts, K)
