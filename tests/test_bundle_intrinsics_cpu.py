"""cs_bundle_adjust_intrinsics and cs_undistort_records without a device: the symbols, the new argument checks, the
overlap sweep, the calls that make no CUDA call, the wrappers through a fake library, the float64 statement (the NC = 9
Jacobians and robust scaling, the LM optimum), the undistortion rule, and the NC = 6 trivial-loss kernels' SASS."""
import ctypes
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

import bundle_intrinsics_cases as bic
import bundle_intrinsics_oracle as bio
import bundle_cases as bc
import cudasift_b200 as cs
import test_arg_ranges_cpu as ar
from cudasift_b200 import build
from test_bundle_cpu import Arena

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_E_ARG = -2


def test_symbols_declared_exported_and_typed():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE,
                         text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for fn, n in (("cs_bundle_adjust_intrinsics", 30), ("cs_undistort_records", 6)):
        assert fn in declared and fn in exported
        f = getattr(cs.lib(), fn)
        assert f.restype is ctypes.c_int and len(f.argtypes) == n
    f = cs.lib().cs_bundle_adjust_intrinsics
    assert [f.argtypes[i] for i in (5, 6, 18, 19)] == [ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_double]
    for name in ("BundleAdjustIntrinsics", "UndistortRecords"):
        assert name in cs.__all__ and hasattr(cs, name)


def _call(a, c, **ch):
    """cs_bundle_adjust_intrinsics on the Arena of test_bundle_cpu with its common arguments, changed by ch."""
    c = dict(c, dists=np.zeros((2, 2)), refine=np.array([1, 3], np.uint8), loss=2, scale=1.0, K_out=None,
             dist_out=None)
    c.update(ch)
    sets = (cs.MatchSet * 2)(*[cs.MatchSet(p, n) for p, n in c["sets"]])
    K, R, t = (np.ascontiguousarray(c[k], np.float64) for k in ("Ks", "Rs", "ts"))
    dist = None if c["dists"] is None else np.ascontiguousarray(c["dists"], np.float64)
    ref = None if c["refine"] is None else np.ascontiguousarray(c["refine"], np.uint8)
    out = dict(R=np.full((2, 9), 5.0), t=np.full((2, 3), 5.0), K=np.full((2, 9), 5.0), d=np.full((2, 2), 5.0))
    K_out = out["K"].ctypes.data if c["K_out"] is None else c["K_out"](K, dist, R, t)
    d_out = out["d"].ctypes.data if c["dist_out"] is None else c["dist_out"](K, dist, R, t)
    R_out = c["R_out"](K, dist, R, t) if "R_out" in c else out["R"].ctypes.data
    cost, stats, ms = np.full(2, 5.0), np.full(8, 7, np.int64), ctypes.c_double(-1.0)
    r = cs.lib().cs_bundle_adjust_intrinsics(
        sets, c["S"], K.ctypes.data, dist.ctypes.data if dist is not None else None,
        ref.ctypes.data if ref is not None else None, c["loss"], c["scale"], R.ctypes.data, t.ctypes.data,
        np.ascontiguousarray(c["fixed"], np.uint8).ctypes.data, c["offsets"], c["T"], c["members"], c["M"], c["use"],
        c["points"], c["maxIterations"], c["maxLinear"], c["tol"], c["maxError"], K_out, d_out, R_out,
        out["t"].ctypes.data, c["errors"], c["inlier"], cost.ctypes.data, None, stats.ctypes.data, ctypes.byref(ms))
    return r, ms.value, out, cost, stats, (K, dist, R, t)


def test_rejects_every_invalid_argument():
    a = Arena()
    nan, inf = float("nan"), float("inf")
    cases = [
        ("refine 8", dict(refine=np.array([0, 8], np.uint8)), "refine[1]"),
        ("loss -1", dict(loss=-1), "loss"),
        ("loss 3", dict(loss=3), "loss"),
        ("lossScale 0", dict(scale=0.0), "lossScale"),
        ("lossScale NaN", dict(scale=nan), "lossScale"),
        ("lossScale inf", dict(scale=inf), "lossScale"),
        ("dists NaN", dict(dists=np.array([[0, 0], [0, nan]])), "dists[1]"),
        ("dists inf", dict(dists=np.array([[inf, 0], [0, 0]])), "dists[0]"),
        ("K_out over Rs", dict(K_out=lambda K, d, R, t: R.ctypes.data), "K_out and Rs"),
        ("K_out inside Ks", dict(K_out=lambda K, d, R, t: K.ctypes.data + 8), "K_out and Ks"),
        ("dist_out over ts", dict(dist_out=lambda K, d, R, t: t.ctypes.data + 8), "dist_out and ts"),
        ("R_out over dists", dict(R_out=lambda K, d, R, t: d.ctypes.data), "R_out and dists"),
        # a bundle_args check names the new call
        ("maxError 0", dict(maxError=0.0), "maxError"),
    ]
    for what, ch, name in cases:
        c = a.common()
        r, ms, out, cost, stats, _ = _call(a, c, **ch)
        assert r == CS_E_ARG, (what, r)
        msg = cs.lib().cs_last_error().decode()
        assert msg.startswith("cs_bundle_adjust_intrinsics:") and "invalid argument" in msg and name in msg, (what, msg)
        assert ms == 0.0 and all((v == 5).all() for v in out.values()) and (cost == 5).all() and (stats == 7).all()
    assert not a.buf.any()


def test_no_tracks_makes_no_cuda_call_and_outputs_may_alias_inputs():
    a = Arena()
    c = a.common()
    c.update(T=0, M=0, Rs=np.stack([np.eye(3), np.eye(3)[[1, 2, 0]]]), ts=np.arange(6.0).reshape(2, 3))
    dist = np.array([[0.1, -0.2], [0.0, 0.3]])
    r, ms, out, cost, stats, (K, d, R, t) = _call(a, c, dists=dist)
    assert r == 0 and ms == 0.0 and not cost.any() and not stats.any()
    assert out["K"].reshape(2, 3, 3).tolist() == c["Ks"].tolist() and out["d"].tolist() == dist.tolist()
    assert out["R"].reshape(2, 3, 3).tolist() == c["Rs"].tolist() and out["t"].tolist() == c["ts"].tolist()
    # exact aliases are allowed, and NULL dists come out as zeros
    r, *_ , (K, d, R, t) = _call(a, c, dists=dist, K_out=lambda K, d, R, t: K.ctypes.data,
                                 dist_out=lambda K, d, R, t: d.ctypes.data, R_out=lambda K, d, R, t: R.ctypes.data)
    assert r == 0 and d.tolist() == dist.tolist() and K.tolist() == c["Ks"].tolist()
    r, ms, out, *_ = _call(a, c, dists=None)
    assert r == 0 and not out["d"].any()
    assert not a.buf.any()


def test_undistort_rejects_every_invalid_argument():
    a = Arena()
    K = np.stack([np.array([[800.0, 1.0, 640], [0, 790, 480], [0, 0, 1]])] * 2)
    nan = float("nan")

    def call(sets=None, S=2, Ks=K, dists=np.zeros((2, 2)), outs=None, setsPtr=True):
        sets = sets or [(a.pts[0], 4), (a.pts[1], 4)]
        st = (cs.MatchSet * 2)(*[cs.MatchSet(p, n) for p, n in sets])
        o = (ctypes.c_void_p * 2)(*(outs if outs is not None else [a.pts[0], a.pts[1]]))
        Kc = np.ascontiguousarray(Ks)
        dc = None if dists is None else np.ascontiguousarray(dists, np.float64)
        ms = ctypes.c_double(-1.0)
        r = cs.lib().cs_undistort_records(st if setsPtr else None, S, Kc.ctypes.data,
                                          dc.ctypes.data if dc is not None else None, o, ctypes.byref(ms))
        return r, ms.value

    Kbad = K.copy()
    Kbad[1, 2, 2] = 2.0
    cases = [
        ("numImages < 0", dict(S=-1), "numImages"),
        ("NULL sets", dict(setsPtr=False), "sets"),
        ("a set without records", dict(sets=[(a.pts[0], 4), (None, 4)]), "sets[1]"),
        ("K not pinhole", dict(Ks=Kbad), "Ks[1]"),
        ("dists NaN", dict(dists=np.array([[0, nan], [0, 0]])), "dists[0]"),
        ("NULL output", dict(outs=[a.pts[0], None]), "d_out[1]"),
        ("output unaligned", dict(outs=[a.pts[0] + 2, a.pts[1]]), "d_out[0]"),
        ("output over its records", dict(outs=[a.pts[0] + 8, a.pts[1]]), "d_out[0] and sets[0].pts"),
        ("two in-place sets overlapping", dict(sets=[(a.pts[0], 4), (a.pts[0] + 576, 4)],
                                               outs=[a.pts[0], a.pts[0] + 576]), "d_out[0] and d_out[1]"),
    ]
    for what, ch, name in cases:
        r, ms = call(**ch)
        assert r == CS_E_ARG, (what, r)
        msg = cs.lib().cs_last_error().decode()
        assert msg.startswith("cs_undistort_records:") and name in msg, (what, msg)
        assert ms == 0.0
    # no records: nothing to do, no CUDA call
    assert call(sets=[(None, 0), (None, 0)], outs=[None, None]) == (0, 0.0)
    assert call(S=0) == (0, 0.0)
    assert not a.buf.any()


# ---- the overlap sweep (the rule of test_arg_ranges_cpu.py) ----

def _bundle_intrinsics(rng):
    sizes, forbidden, _ = ar.bundle(rng)
    I = sum(1 for x in sizes if x.startswith("sets["))
    n = [sizes["sets[%d].pts" % a] // ar.REC for a in range(I)]
    T, M = sizes["d_points"] // 24, sizes["d_members"] // 8
    Ks, Rs, ts = np.stack([ar.K] * I), np.stack([np.eye(3)] * I), np.zeros((I, 3))
    dist, ref = np.zeros((I, 2)), np.full(I, 3, np.uint8)
    out = np.zeros((4, I, 9))
    cost = np.zeros(2)

    def call(at):
        st = (cs.MatchSet * I)(*[cs.MatchSet(at["sets[%d].pts" % a], n[a]) for a in range(I)])
        return cs.lib().cs_bundle_adjust_intrinsics(
            st, I, Ks.ctypes.data, dist.ctypes.data, ref.ctypes.data, 2, 1.0, Rs.ctypes.data, ts.ctypes.data, None,
            at["d_offsets"], T, at["d_members"], M, at["d_use"], at["d_points"], 10, 50, 0.1, 4.0, out[0].ctypes.data,
            out[1].ctypes.data, out[2].ctypes.data, out[3].ctypes.data, at["d_errors"], at["d_inlier"],
            cost.ctypes.data, None, None, None)

    return sizes, forbidden, call


def _undistort(rng):
    I = int(rng.integers(1, 5))
    n = ar._counts(rng, I)
    inplace = rng.random(I) < 0.3
    sizes = {}
    for a in range(I):
        sizes["d_out[%d]" % a] = n[a] * ar.REC
        if not inplace[a]:
            sizes["sets[%d].pts" % a] = n[a] * ar.REC
    if len(sizes) < 2:                                          # one in-place image: nothing can conflict
        return _undistort(rng)
    Ks, dist = np.stack([ar.K] * I), np.zeros((I, 2))

    def call(at):
        src = [at["d_out[%d]" % a] if inplace[a] else at["sets[%d].pts" % a] for a in range(I)]
        st = (cs.MatchSet * I)(*[cs.MatchSet(src[a], n[a]) for a in range(I)])
        o = (ctypes.c_void_p * I)(*[at["d_out[%d]" % a] for a in range(I)])
        return cs.lib().cs_undistort_records(st, I, Ks.ctypes.data, dist.ctypes.data, o, None)

    return sizes, lambda a, b: a.startswith("d_out") or b.startswith("d_out"), call


@pytest.mark.parametrize("fn", ["cs_bundle_adjust_intrinsics", "cs_undistort_records"])
def test_every_overlap_is_rejected_and_named(fn):
    make = dict(cs_bundle_adjust_intrinsics=_bundle_intrinsics, cs_undistort_records=_undistort)[fn]
    rng = np.random.default_rng(sum(map(ord, fn)))
    for _ in range(ar.LAYOUTS):
        sizes, forbidden, call = make(rng)
        while True:
            at = ar._layout(rng, sizes, forbidden)
            # an output exactly on its own set's records is the in-place case, which is allowed: draw again
            if not any(x.startswith("d_out[") and at[x] == at.get("sets[%s].pts" % x[6:-1]) for x in at):
                break
        r = call({x: ar.BASE + v for x, v in at.items()})
        msg = cs.lib().cs_last_error().decode()
        assert r == CS_E_ARG, (fn, r, msg, at, sizes)
        m = ar.MSG.match(msg)
        assert m, (fn, msg)
        _, a, b = m.groups()
        assert a in sizes and b in sizes, (fn, msg, sorted(sizes))
        assert forbidden(a, b) and ar._share((at[a], sizes[a]), (at[b], sizes[b])), (fn, msg, at, sizes)
    assert not ar._buf.any(), fn


# ---- the wrappers ----

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

    def cs_bundle_adjust_intrinsics(self, *args):
        self.calls.append(args)
        return 0

    def cs_undistort_records(self, *args):
        self.calls.append(args)
        return 0


class _Buf:
    ptr = 1 << 21

    def free(self):
        return 0


class _Data:
    def __init__(self, n):
        self.d_data, self.numPts = 1 << 20, n


def _bytes(p, n, ctype):
    return np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctype)), (n,))


def test_wrappers_build_their_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    ts = np.array([[0.0, 0, 0], [0.1, -2.0, 0.5], [1.0, 0, 0]])
    offsets, members = np.array([0, 2, 4]), np.array([[0, 0], [1, 0], [1, 1], [2, 0]])
    pts = np.zeros((2, 3))
    datas = [_Data(1), _Data(2), _Data(1)]
    out = cs.BundleAdjustIntrinsics(datas, np.eye(3), np.eye(3), ts, offsets, members, pts)
    args = fake.calls[-1]
    assert len(args) == 30 and len(out) == 11
    assert args[1] == 3 and _bytes(args[3], 6, ctypes.c_double).tolist() == [0.0] * 6
    assert _bytes(args[4], 3, ctypes.c_uint8).tolist() == [3, 3, 3] and args[5] == 0 and args[6] == 1.0
    assert _bytes(args[9], 3, ctypes.c_uint8).tolist() == [1, 3, 0]          # BundleAdjust's default gauge
    assert args[11] == 2 and args[13] == 4 and args[14] is None
    assert args[16] == 50 and args[17] == 100 and args[18] == 1e-6 and args[19] == 4.0
    assert args[20] is not None and args[21] is not None and args[27] is not None
    cs.BundleAdjustIntrinsics(datas, np.eye(3), np.eye(3), ts, offsets, members, pts, dists=[[0.1, 0.2]] * 3,
                              refine=[1, 0, 7], loss="cauchy", lossScale=2.5, use=[1, 0, 1, 1], fixed=[0, 0, 4],
                              maxIterations=3)
    args = fake.calls[-1]
    assert _bytes(args[3], 6, ctypes.c_double).tolist() == [0.1, 0.2] * 3
    assert _bytes(args[4], 3, ctypes.c_uint8).tolist() == [1, 0, 7] and args[5] == 2 and args[6] == 2.5
    assert _bytes(args[9], 3, ctypes.c_uint8).tolist() == [0, 0, 4] and args[14] is not None and args[16] == 3
    for bad in (dict(refine=[1, 2]), dict(refine=8), dict(loss="huber"), dict(dists=[[0.0, 0.0]] * 2)):
        with pytest.raises(ValueError):
            cs.BundleAdjustIntrinsics(datas, np.eye(3), np.eye(3), ts, offsets, members, pts, **bad)
    monkeypatch.setattr(cs, "InitSiftData", lambda d, n: setattr(d, "_buf", _Buf()) or d)
    outs = cs.UndistortRecords(datas, np.eye(3), [0.1, 0.0])
    args = fake.calls[-1]
    assert len(outs) == 3 and [o.numPts for o in outs] == [1, 2, 1] and args[1] == 3
    assert _bytes(args[3], 6, ctypes.c_double).tolist() == [0.1, 0.0] * 3


# ---- the float64 statement ----

def _problem(seed=2, loss=0, refine=7, **kw):
    s = bic.scene(seed, noise=0.5, **kw)
    P = bio.Intrinsics(s["xy"], s["K0"], s["R0"], s["t0"], s["offsets"], s["members"], s["X0"],
                       dists=np.tile([0.02, -0.01], (len(s["K"]), 1)), refine=refine, loss=loss, lossScale=2.0,
                       use=s["use"], fixed=bc.gauge(s["t0"]))
    return s, P


@pytest.mark.parametrize("loss", [0, 1, 2])
def test_oracle_jacobians_and_robust_scaling_against_central_differences(loss):
    s, P = _problem(2, loss=loss, numPoints=40, outlier=0.1)
    R, t, X, K, k = P.R0, P.t0, P.X0, P.K, P.k0
    Jc, Jp, r = P.jacobians(R, t, X, K, k, robust=False)
    full = np.ones((P.S, 9), bool)
    h = 1e-6
    for o in range(0, P.N, 7):
        a, kk = int(P.a[o]), int(P.k[o])
        for i in range(9):
            d = np.zeros((P.S, 9))
            d[a, i] = h * (K[a, 0, 0] if i == 6 else 1.0)
            rp = P.residuals(*_take(P.apply9(R, t, K, k, full, d), X))[0][o]
            rm = P.residuals(*_take(P.apply9(R, t, K, k, full, -d), X))[0][o]
            num = (rp - rm) / (2 * d[a, i])
            np.testing.assert_allclose(num, Jc[o, :, i], rtol=1e-5, atol=1e-6 * np.abs(Jc[o]).max())
        for j in range(3):
            Xp, Xm = X.copy(), X.copy()
            Xp[kk, j] += h
            Xm[kk, j] -= h
            num = (P.residuals(R, t, Xp, K, k)[0][o] - P.residuals(R, t, Xm, K, k)[0][o]) / (2 * h)
            np.testing.assert_allclose(num, Jp[o, :, j], rtol=1e-5, atol=1e-6 * np.abs(Jp[o]).max())
    # the corrector: sqrt(rho') scales r and both blocks, so (J w)^T (r w) is the gradient of the robust cost / 2
    Jcw, Jpw, rw = P.jacobians(R, t, X, K, k)
    s2 = (r * r).sum(1)
    rho, w = bio.loss_rho(P.loss, P.c2, s2)
    np.testing.assert_allclose(rw, r * w[:, None], rtol=1e-15)
    np.testing.assert_allclose(Jcw, Jc * w[:, None, None], rtol=1e-15)
    hs = 1e-4 * s2
    num = (bio.loss_rho(P.loss, P.c2, s2 + hs)[0] - bio.loss_rho(P.loss, P.c2, s2 - hs)[0]) / (2 * hs)
    np.testing.assert_allclose(num, w * w, rtol=1e-6)
    np.testing.assert_allclose(rho.sum(), P.cost(R, t, X, K, k)[0], rtol=1e-15)


def _take(cam, X):
    R1, t1, K1, k1 = cam
    return R1, t1, X, K1, k1


@pytest.mark.parametrize("loss", [0, 2])
def test_oracle_converges_to_scipys_optimum(loss):
    """scipy's least_squares over the same parameters (the pose update of the oracle from the start, f with the K
    ratios held, k1, k2, the points) and gauge, started at the oracle's result, finds nothing lower."""
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    s, P = _problem(6, loss=loss, refine=[3, 7, 1, 3, 5], numImages=5, numPoints=50, outlier=0.1 if loss else 0.0)
    K, k, R, t, X, cost, trace, acc = P.run(100, 200, 1e-10)
    free = P.mask

    def fun(v):
        dc = np.zeros((P.S, 9))
        dc[free] = v[:free.sum()]
        Rr, tt, KK, kk = P.apply9(P.R0, P.t0, P.K, P.k0, free, dc)
        XX = P.X0.copy()
        XX[P.parts] = P.X0[P.parts] + v[free.sum():].reshape(-1, 3)
        r = P.residuals(Rr, tt, XX, KK, kk)[0]
        if loss == 0:
            return r.reshape(-1)
        return np.sqrt(bio.loss_rho(loss, P.c2, (r * r).sum(1))[0])
    dc = np.zeros((P.S, 9))
    dc[:, :3] = Rotation.from_matrix(np.einsum("aij,akj->aik", R, P.R0)).as_rotvec()
    dc[:, 3:6], dc[:, 6] = t - P.t0, K[:, 0, 0] - P.K[:, 0, 0]
    dc[:, 7:] = k - P.k0
    v0 = np.concatenate([dc[free], (X - P.X0)[P.parts].reshape(-1)])
    assert abs(float(fun(v0) @ fun(v0)) - cost[1]) <= 1e-9 * cost[1]
    sol = least_squares(fun, v0, method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    best = float(sol.fun @ sol.fun)
    assert acc > 0 and cost[1] < 0.1 * cost[0] and best >= cost[1] * (1 - 1e-8), (cost, best)
    assert P.stats[5] == free.sum() and free[:, 6:].sum() > 0


@pytest.mark.parametrize("k", [(-0.2, 0.05), (0.1, -0.02), (-0.35, 0.0), (0.0, 0.0)])
def test_undistortion_round_trips_through_the_distortion(k):
    rng = np.random.default_rng(3)
    K = np.array([[900.0, 2.0, 640], [0, 880, 480], [0, 0, 1]])
    Xc = np.concatenate([rng.uniform(-0.6, 0.6, (200, 2)), np.ones((200, 1))], 1)
    px = bio.distort(K, k, Xc)
    und = bio.undistort(K, k, px.astype(np.float32))
    want = (K @ Xc.T).T[:, :2]
    # the float32 input position is the only rounding: its error, through the inverse's slope, bounds the result's
    assert np.isfinite(und).all()
    np.testing.assert_allclose(und, want, rtol=0, atol=2e-4)
    # the rule itself in float64: r_u (1 + k1 r_u^2 + k2 r_u^4) = r_d to 1e-12 relative
    for r in np.linspace(0.0, 0.85, 41):                     # the radii of the points above
        rd = r * (1 + k[0] * r * r + k[1] * r ** 4)
        ru, ok = bio.solve_ru(rd, k)
        assert ok and abs(ru * (1 + k[0] * ru * ru + k[1] * ru ** 4) - rd) <= 1e-12 * rd, (rd, ru)
        assert abs(ru - r) <= 1e-12, (r, ru)


def test_undistortion_nan_where_the_inverse_does_not_exist():
    K = np.array([[500.0, 0, 320], [0, 500, 240], [0, 0, 1]])
    k = (-0.5, 0.0)                      # r (1 - 0.5 r^2) peaks at r = sqrt(2/3), r_d = 0.544
    xy = np.array([[320 + 500 * 0.3, 240], [320 + 500 * 0.6, 240], [np.nan, 240], [320, 240]], np.float32)
    und = bio.undistort(K, k, xy)
    assert np.isfinite(und[0]).all() and np.isnan(und[1]).all() and np.isnan(und[2]).all()
    assert und[3].tolist() == [320.0, 240.0]


# ---- the NC = 6 trivial-loss kernels are the parent's, instruction for instruction ----

# sha256 of the normalised `cuobjdump -sass` (addresses dropped) of cs_bundle_adjust's three kernels before the camera
# block became a template parameter, from nvcc 12.9 (V12.9.86) with the library's flags.
SASS = {"bundle_kernel": "01fe401d8a9c051219f48391f7f841eccdf7b9684a82bc246467d1db1881ab00",
        "bundle_fill_kernel": "a177aecb1e71fbb91031abbf03b6e81d4eb15d6a278c972df30b5708dc744e9a",
        "bundle_count_kernel": "3ea644fadbbd17f2bfef94add88fa39bf27509ab23aeca05563d2badc33c9b8b"}
INSTANTIATION = {"bundle_kernel": "ILi6ELb0E", "bundle_fill_kernel": "ILi6E", "bundle_count_kernel": "ILi6E"}


def _sass(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], stdout=subprocess.PIPE, text=True).stdout
    fs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            fs[cur] = []
        elif cur and re.match(r"\s*/\*[0-9a-f]{4,6}\*/", line):
            fs[cur].append(re.sub(r"/\*[0-9a-f]{4,6}\*/", "", line.split(";")[0]).strip())
    return fs


def test_nc6_trivial_kernels_are_unchanged():
    nvcc = build.nvcc_path()
    if nvcc is None or "V12.9.86" not in subprocess.run([nvcc, "--version"], stdout=subprocess.PIPE,
                                                        text=True).stdout:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    build.build_library()
    fs = _sass(os.path.join(build.OBJDIR, "bundle.o"))
    for name, digest in SASS.items():
        key = [f for f in fs if re.search(r"\d+%s%s" % (name, INSTANTIATION[name]), f)]
        assert len(key) == 1, (name, sorted(fs))
        assert hashlib.sha256("\n".join(fs[key[0]]).encode()).hexdigest() == digest, name
