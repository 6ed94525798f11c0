"""cs_bundle_adjust without a device: the symbol, every argument check, the calls that make no CUDA call, the wrapper
through a fake library, and the float64 statement itself (Jacobians, the Schur + CG step, the LM optimum)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import bundle_cases as bc
import bundle_oracle as bo
import cudasift_b200 as cs
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_E_ARG = -2
RECORD = 576


def test_symbols_declared_exported_and_typed():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE,
                         text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert "cs_bundle_adjust" in declared and "cs_bundle_adjust" in exported
    f = cs.lib().cs_bundle_adjust
    assert f.restype is ctypes.c_int and len(f.argtypes) == 24
    assert f.argtypes[14] is ctypes.c_double and f.argtypes[15] is ctypes.c_double
    assert "BundleAdjust" in cs.__all__ and hasattr(cs, "BundleAdjust")


class Arena:
    """Host memory laid out as on the device: two sets of 4 records, 2 tracks of 2 members, their points, errors,
    inlier and use bytes.  Nothing is dereferenced: every case fails its checks."""

    def __init__(self):
        self.buf = np.zeros(2 * 4 * RECORD + 4096, np.uint8)
        base = self.buf.ctypes.data + (-self.buf.ctypes.data) % 64
        self.pts = [base, base + 4 * RECORD]
        o = base + 8 * RECORD
        self.offsets, self.members, self.points = o, o + 64, o + 128
        self.errors, self.inlier, self.use = o + 192, o + 224, o + 256

    def common(self):
        K = np.array([[800.0, 1.0, 640], [0, 790, 480], [0, 0, 1]])
        return dict(sets=[(self.pts[0], 4), (self.pts[1], 4)], S=2, Ks=np.stack([K, K]),
                    Rs=np.stack([np.eye(3)] * 2), ts=np.zeros((2, 3)), fixed=np.zeros(2, np.uint8),
                    offsets=self.offsets, T=2, members=self.members, M=4, use=self.use, points=self.points,
                    maxIterations=10, maxLinear=50, tol=1e-6, maxError=4.0, errors=self.errors, inlier=self.inlier,
                    out=True, cost=True)


def _call(c):
    sets = (cs.MatchSet * 2)(*[cs.MatchSet(p, n) for p, n in c["sets"]])
    K, R, t = (np.ascontiguousarray(c[k], np.float64) for k in ("Ks", "Rs", "ts"))
    fix = None if c["fixed"] is None else np.ascontiguousarray(c["fixed"], np.uint8)
    R_out, t_out = np.full((2, 9), 5.0), np.full((2, 3), 5.0)
    cost, trace, stats = np.full(2, 5.0), np.full(4 * max(c["maxIterations"], 1), 5.0), np.full(8, 7, np.int64)
    ms = ctypes.c_double(-1.0)
    r = cs.lib().cs_bundle_adjust(sets if c.get("setsPtr", 1) else None, c["S"], K.ctypes.data, R.ctypes.data,
                                  t.ctypes.data, fix.ctypes.data if fix is not None else None, c["offsets"], c["T"],
                                  c["members"], c["M"], c["use"], c["points"], c["maxIterations"], c["maxLinear"],
                                  c["tol"], c["maxError"], R_out.ctypes.data if c["out"] else None, t_out.ctypes.data,
                                  c["errors"], c["inlier"], cost.ctypes.data if c["cost"] else None, trace.ctypes.data,
                                  stats.ctypes.data, ctypes.byref(ms))
    return r, ms.value, (R_out, t_out, cost, stats)


def test_rejects_every_invalid_argument():
    a = Arena()
    nan = float("nan")

    def Rbad():
        R = np.stack([np.eye(3)] * 2)
        R[1, 0, 0] = 1.1
        return R

    cases = [
        ("numImages < 0", dict(S=-1), "numImages"),
        ("numTracks < 0", dict(T=-1), "numTracks"),
        ("numMembers < 0", dict(M=-1), "numMembers"),
        ("NULL sets", dict(setsPtr=0), "sets"),
        ("a set without records", dict(sets=[(a.pts[0], 4), (None, 4)]), "sets[1]"),
        ("K not finite", dict(Ks=np.stack([np.eye(3), np.full((3, 3), nan)])), "Ks[1]"),
        ("R not a rotation", dict(Rs=Rbad()), "Rs[1]"),
        ("t not finite", dict(ts=np.array([[0, 0, 0], [0, nan, 0]])), "ts[1]"),
        ("fixed 5", dict(fixed=np.array([0, 5], np.uint8)), "fixed[1]"),
        ("maxIterations -1", dict(maxIterations=-1), "maxIterations"),
        ("maxIterations 1001", dict(maxIterations=1001), "maxIterations"),
        ("maxLinearIterations 0", dict(maxLinear=0), "maxLinearIterations"),
        ("maxLinearIterations 10001", dict(maxLinear=10001), "maxLinearIterations"),
        ("linearTol 0", dict(tol=0.0), "linearTol"),
        ("linearTol 1", dict(tol=1.0), "linearTol"),
        ("linearTol NaN", dict(tol=nan), "linearTol"),
        ("maxError 0", dict(maxError=0.0), "maxError"),
        ("NULL R_out", dict(out=False), "R_out"),
        ("NULL cost_out", dict(cost=False), "cost_out"),
        ("NULL offsets", dict(offsets=None), "d_offsets"),
        ("NULL points", dict(points=None), "d_points"),
        ("NULL members", dict(members=None), "d_members"),
        ("offsets unaligned", dict(offsets=a.offsets + 2), "d_offsets"),
        ("members unaligned", dict(members=a.members + 4), "d_members"),
        ("points unaligned", dict(points=a.points + 4), "d_points"),
        ("errors unaligned", dict(errors=a.errors + 1), "d_errors"),
        ("errors over the points", dict(errors=a.points + 40), "d_points and d_errors"),
        ("inlier over the errors", dict(inlier=a.errors + 8), "d_errors and d_inlier"),
        ("points over the members", dict(points=a.members + 8), "d_points and d_members"),
        ("inlier over d_use", dict(inlier=a.use + 2), "d_inlier and d_use"),
        ("errors over a record range", dict(errors=a.pts[1] + 8), "d_errors and sets[1].pts"),
    ]
    for what, ch, name in cases:
        c = a.common()
        c.update(ch)
        r, ms, (R, t, cost, stats) = _call(c)
        assert r == CS_E_ARG, (what, r)
        msg = cs.lib().cs_last_error().decode()
        assert "invalid argument" in msg and name in msg, (what, name, msg)
        assert ms == 0.0 and (R == 5).all() and (t == 5).all() and (cost == 5).all() and (stats == 7).all(), what
    assert not a.buf.any()


def test_no_tracks_and_no_images_make_no_cuda_call():
    """numTracks == 0 returns 0 with the input poses, zero costs, trace and statistics (this holds without a device)."""
    a = Arena()
    c = a.common()
    c.update(T=0, M=0, Rs=np.stack([np.eye(3), np.eye(3)[[1, 2, 0]]]), ts=np.arange(6.0).reshape(2, 3))
    r, ms, (R, t, cost, stats) = _call(c)
    assert r == 0 and ms == 0.0
    assert R.reshape(2, 3, 3).tolist() == c["Rs"].tolist() and t.tolist() == c["ts"].tolist()
    assert not cost.any() and not stats.any()
    c.update(S=0, sets=[(None, 0), (None, 0)])
    r, ms, (R, t, cost, stats) = _call(c)
    assert r == 0 and not cost.any() and (R == 5).all()
    assert not a.buf.any()


class _FakeLib:
    def __init__(self):
        self.calls = []

    def cs_device_alloc(self, n):
        return 4096 * (len(self.calls) + 1)

    def cs_device_free(self, p):
        return 0

    def cs_memcpy_h2d(self, dst, src, n):
        return 0

    def cs_memcpy_d2h(self, dst, src, n):
        return 0

    def cs_bundle_adjust(self, *args):
        self.calls.append(args)
        return 0


class _Data:
    def __init__(self, n):
        self.d_data, self.numPts = 1 << 20, n


def test_wrapper_builds_its_arguments_and_the_default_gauge(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    ts = np.array([[0.0, 0, 0], [0.1, -2.0, 0.5], [1.0, 0, 0]])
    offsets, members = np.array([0, 2, 4]), np.array([[0, 0], [1, 0], [1, 1], [2, 0]])
    pts = np.zeros((2, 3))
    cs.BundleAdjust([_Data(1), _Data(2), _Data(1)], np.eye(3), np.eye(3), ts, offsets, members, pts)
    args = fake.calls[-1]
    assert args[1] == 3 and args[7] == 2 and args[9] == 4 and args[10] is None
    fixed = np.ctypeslib.as_array(ctypes.cast(args[5], ctypes.POINTER(ctypes.c_uint8)), (3,))
    assert fixed.tolist() == [1, 3, 0]                         # image 0 held, image 1 holds t[1] (|-2| largest)
    assert args[12] == 50 and args[13] == 100 and args[14] == 1e-6 and args[15] == 4.0
    cs.BundleAdjust([_Data(1), _Data(2), _Data(1)], np.eye(3), np.eye(3), ts, offsets, members, pts,
                    use=[1, 0, 1, 1], fixed=[0, 0, 4], maxIterations=0)
    args = fake.calls[-1]
    fixed = np.ctypeslib.as_array(ctypes.cast(args[5], ctypes.POINTER(ctypes.c_uint8)), (3,))
    assert fixed.tolist() == [0, 0, 4] and args[10] is not None and args[12] == 0 and args[21] is None
    with pytest.raises(ValueError):
        cs.BundleAdjust([_Data(1)] * 3, np.eye(3), np.eye(3), ts, offsets, members, pts, use=[1, 1])
    with pytest.raises(ValueError):
        cs.BundleAdjust([_Data(1)] * 3, np.eye(3), np.eye(3), ts, offsets, members, np.zeros((3, 3)))


def _problem(seed=1, **kw):
    s = bc.scene(seed, **kw)
    return s, bo.Problem(s["xy"], s["K"], s["R0"], s["t0"], s["offsets"], s["members"], s["X0"], use=s["use"],
                         fixed=bc.gauge(s["t0"]))


def test_oracle_jacobians_against_central_differences():
    s, P = _problem(2, numPoints=40)
    R, t, X = P.R0, P.t0, P.X0
    Jc, Jp, r = P.jacobians(R, t, X)
    h = 1e-6
    for o in range(0, P.N, 7):
        a, k = int(P.a[o]), int(P.k[o])
        for i in range(6):
            d = np.zeros((P.S, 6))
            d[a, i] = h
            Rp, tp = P.apply(R, t, np.ones((P.S, 6), bool), d)
            Rm, tm = P.apply(R, t, np.ones((P.S, 6), bool), -d)
            num = (P.residuals(Rp, tp, X)[0][o] - P.residuals(Rm, tm, X)[0][o]) / (2 * h)
            np.testing.assert_allclose(num, Jc[o, :, i], rtol=1e-5, atol=1e-6 * np.abs(Jc[o]).max())
        for j in range(3):
            Xp, Xm = X.copy(), X.copy()
            Xp[k, j] += h
            Xm[k, j] -= h
            num = (P.residuals(R, t, Xp)[0][o] - P.residuals(R, t, Xm)[0][o]) / (2 * h)
            np.testing.assert_allclose(num, Jp[o, :, j], rtol=1e-5, atol=1e-6 * np.abs(Jp[o]).max())


@pytest.mark.parametrize("lam", [1e-3, 1.0])
def test_oracle_schur_cg_step_against_the_dense_system(lam):
    s, P = _problem(4)
    Jc, Jp, r = P.jacobians(P.R0, P.t0, P.X0)
    ok, dc, dp, it = P.solve(Jc, Jp, r, lam, 1000, 1e-14)
    dc2, dp2 = P.dense_step(Jc, Jp, r, lam)
    assert ok and it > 0
    assert np.abs(dc - dc2).max() <= 1e-10 * np.abs(dc2).max()
    assert np.abs(dp - dp2).max() <= 1e-10 * np.abs(dp2).max()
    assert not dc[0].any() and dc[1, 3 + int(np.argmax(np.abs(P.t0[1])))] == 0.0


def test_oracle_converges_to_scipys_optimum():
    from scipy.optimize import least_squares
    s, P = _problem(6, numImages=5, numPoints=50)
    R, t, X, cost, trace, acc = P.run(100, 200, 1e-10)
    free = P.mask

    def fun(v):
        dc = np.zeros((P.S, 6))
        dc[free] = v[:free.sum()]
        Rr, tt = P.apply(P.R0, P.t0, free, dc)
        XX = P.X0.copy()
        XX[P.parts] = P.X0[P.parts] + v[free.sum():].reshape(-1, 3)
        return P.residuals(Rr, tt, XX)[0].reshape(-1)
    sol = least_squares(fun, np.zeros(free.sum() + 3 * len(P.parts)), method="lm", xtol=1e-15, ftol=1e-15,
                        gtol=1e-15)
    best = float(sol.fun @ sol.fun)
    assert acc > 0 and abs(cost[1] - best) <= 1e-8 * best, (cost, best)
