"""cs_bundle_adjust on the device against the float64 statement in bundle_oracle.py and the dense normal equations."""
import ctypes

import numpy as np
import pytest

import bundle_cases as bc
import bundle_oracle as bo
from test_triangulate_gpu import Scene

pytestmark = pytest.mark.gpu
LAUNCHES = 3
SENTINEL_F = np.float32(-12345.0)


class Bundle(Scene):
    """A scene of bundle_cases in device memory; run() makes one call with a sentinel past every member output."""

    def __init__(self, cs, s):
        super().__init__(cs, s["xy"], s["K"], s["R0"], s["t0"], s["offsets"], s["members"])
        self.s = s
        self.d_use = cs.DeviceBuffer(max(self.M, 1))
        self.d_use.upload(np.asarray(s["use"], np.uint8))
        self.bufs.append(self.d_use)

    def run(self, points=None, fixed=None, use=True, maxIterations=30, maxLinear=100, tol=1e-6, maxError=4.0,
            memberOutputs=True, Rs=None, ts=None):
        cs, T, M, S = self.cs, self.T, self.M, self.S
        X = np.ascontiguousarray(self.s["X0"] if points is None else points, np.float64)
        Rs = np.ascontiguousarray(self.Rs if Rs is None else Rs)
        ts = np.ascontiguousarray(self.ts if ts is None else ts)
        fix = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
        outs = [cs.DeviceBuffer(8 * 3 * T), cs.DeviceBuffer(4 * (M + 1)), cs.DeviceBuffer(M + 8)]
        R_out, t_out = np.zeros((S, 3, 3)), np.zeros((S, 3))
        cost, trace = np.zeros(2), np.full((maxIterations + 1, 4), -7.0)
        stats, ms = np.full(8, 7, np.int64), ctypes.c_double(0.0)
        try:
            outs[0].upload(X)
            outs[1].upload(np.full(M + 1, SENTINEL_F, np.float32))
            outs[2].upload(np.full(M + 8, 0xAB, np.uint8))
            before = cs.lib().cs_launch_count()
            r = cs.lib().cs_bundle_adjust(self.sets, S, self.Ks.ctypes.data, Rs.ctypes.data, ts.ctypes.data,
                                          fix.ctypes.data if fix is not None else None, self.d_off.ptr, T,
                                          self.d_mem.ptr, M, self.d_use.ptr if use else None, outs[0].ptr,
                                          maxIterations, maxLinear, tol, maxError, R_out.ctypes.data,
                                          t_out.ctypes.data, outs[1].ptr if memberOutputs else None,
                                          outs[2].ptr if memberOutputs else None, cost.ctypes.data,
                                          trace.ctypes.data, stats.ctypes.data, ctypes.byref(ms))
            launches = cs.lib().cs_launch_count() - before
            assert r >= 0, cs.lib().cs_last_error().decode()
            pts = outs[0].download(np.float64, 3 * T).reshape(T, 3)
            err = outs[1].download(np.float32, M + 1)
            inl = outs[2].download(np.uint8, M + 8)
        finally:
            for b in outs:
                b.free()
        assert (trace[maxIterations] == -7.0).all()
        assert err[M] == SENTINEL_F and (inl[M:] == 0xAB).all()
        if not memberOutputs:
            assert (err == SENTINEL_F).all() and (inl == 0xAB).all()
        return dict(r=r, R=R_out, t=t_out, X=pts, err=err[:M], inl=inl[:M], cost=cost, trace=trace[:maxIterations],
                    stats=stats, ms=ms.value, launches=launches)

    def oracle(self, points=None, fixed=None, use=True, Rs=None, ts=None):
        return bo.Problem(self.xy, self.Ks, self.Rs if Rs is None else Rs, self.ts if ts is None else ts,
                          self.offsets, self.members, self.s["X0"] if points is None else points,
                          use=self.s["use"] if use else None, fixed=fixed)


def rot_log(R):
    c = np.clip((np.trace(R) - 1) / 2, -1, 1)
    th = np.arccos(c)
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return v * (0.5 if th < 1e-12 else th / (2 * np.sin(th)))


def clear_iterations(P):
    """The leading iterations of the oracle's run none of whose CG or LM decisions lies within 1e-6 relative of its
    threshold.  Near the optimum the cost decreases by less than that, so the comparison stops before."""
    for i, h in enumerate(P.history):
        ok = True
        if np.isfinite(h["cand"]):
            ok = abs(h["cand"] - h["cost"]) > 1e-6 * h["cost"]
            ok = ok and abs(h["cost"] - h["cand"] - 1e-10 * h["cost"]) > 1e-6 * h["cost"]
        ok = ok and all(abs(rr - thr) > 1e-6 * thr for rr, thr, _ in h["cg"])
        if not ok:
            return i
    return len(P.history)


def test_first_step_against_the_dense_system(cs):
    s = bc.scene(3)
    b = Bundle(cs, s)
    try:
        fixed = bc.gauge(s["t0"])
        got = b.run(fixed=fixed, maxIterations=1, maxLinear=1000, tol=1e-14)
        P = b.oracle(fixed=fixed)
        Jc, Jp, r = P.jacobians(P.R0, P.t0, P.X0)
        dc, dp = P.dense_step(Jc, Jp, r, 1e-3)
        assert got["trace"][0, 3] == 1.0 and got["r"] == 1
        for a in range(b.S):
            w = rot_log(got["R"][a] @ P.R0[a].T)
            np.testing.assert_allclose(w, dc[a, :3], rtol=0, atol=1e-9 * np.abs(dc[:, :3]).max())
            np.testing.assert_allclose(got["t"][a] - P.t0[a], dc[a, 3:], rtol=0, atol=1e-9 * np.abs(dc[:, 3:]).max())
        d = got["X"][P.parts] - P.X0[P.parts]
        np.testing.assert_allclose(d, dp[P.parts], rtol=0, atol=1e-9 * np.abs(dp).max())
    finally:
        b.free()


@pytest.mark.parametrize("seed", [1, 2, 5])
def test_trace_against_the_oracle(cs, seed):
    s = bc.scene(seed)
    b = Bundle(cs, s)
    try:
        fixed = bc.gauge(s["t0"])
        P = b.oracle(fixed=fixed)
        P.run(20, 100, 1e-6)
        n = clear_iterations(P)
        assert n >= 3
        P = b.oracle(fixed=fixed)
        R, t, X, cost, trace, acc = P.run(n, 100, 1e-6)
        got = b.run(fixed=fixed, maxIterations=n, tol=1e-6)
        n = len(trace)
        assert got["r"] == acc and got["stats"][6] == n
        np.testing.assert_array_equal(got["trace"][:n, 3], trace[:, 3])
        np.testing.assert_array_equal(got["trace"][:n, 2], trace[:, 2])
        np.testing.assert_allclose(got["trace"][:n, 0], trace[:, 0], rtol=1e-9)
        assert (got["trace"][n:] == 0).all()
        np.testing.assert_allclose(got["cost"], cost, rtol=1e-9)
        np.testing.assert_allclose(got["R"], R, rtol=0, atol=1e-6)
        np.testing.assert_allclose(got["t"], t, rtol=0, atol=1e-6)
        np.testing.assert_allclose(got["X"], X, rtol=0, atol=1e-6)
        np.testing.assert_array_equal(got["stats"][:6], P.stats[:6])
        assert got["stats"][7] == trace[:, 2].sum()
        err, inl, written = P.outputs(R, t, X, 4.0)
        np.testing.assert_array_equal(got["inl"][written], inl[written].astype(np.uint8))
        np.testing.assert_allclose(got["err"][written], err[written], rtol=1e-5)
    finally:
        b.free()


def test_convergence_to_the_truth(cs):
    s = bc.scene(7, noise=0.0, outlier=0.0, rot=0.005, trans=0.05, point=0.03)
    b = Bundle(cs, s)
    try:
        got = b.run(fixed=bc.gauge(s["t"]), maxIterations=50, tol=1e-10)
        # the record positions are float32: about 3e-5 px of rounding per coordinate is all that is left
        assert got["cost"][1] < 1e-6 and got["cost"][0] > 1e4
        np.testing.assert_allclose(got["R"], s["R"], atol=1e-6)
        np.testing.assert_allclose(got["t"], s["t"], atol=1e-5)
        np.testing.assert_allclose(got["X"], s["X"], atol=1e-5)
    finally:
        b.free()


def test_held_values_stay_bit_identical(cs):
    s = bc.scene(11, numImages=7)
    s["xy"] = s["xy"] + [np.zeros((0, 2), np.float32)]          # image 7: no observation
    s["K"] = np.concatenate([s["K"], s["K"][:1]])
    s["R0"] = np.concatenate([s["R0"], s["R0"][:1]])
    s["t0"] = np.concatenate([s["t0"], s["t0"][:1] + 1.0])
    X0 = s["X0"].copy()
    X0[3] = np.nan
    b = Bundle(cs, s)
    try:
        use = np.asarray(s["use"], np.uint8).copy()
        lo, hi = int(s["offsets"][5]), int(s["offsets"][6])
        use[lo + 1:hi] = 0                                      # track 5: one used observation
        b.d_use.upload(use)
        fixed = np.array([1, 3, 0, 4, 0, 1, 0, 0], np.uint8)
        got = b.run(points=X0, fixed=fixed, maxIterations=10)
        assert got["r"] > 0
        for a in (0, 5, 7):
            assert got["R"][a].tobytes() == s["R0"][a].tobytes() and got["t"][a].tobytes() == s["t0"][a].tobytes()
        assert got["t"][1][1].tobytes() == s["t0"][1][1].tobytes()
        assert got["t"][3][2].tobytes() == s["t0"][3][2].tobytes()
        assert got["X"][3].tobytes() == X0[3].tobytes() and got["X"][5].tobytes() == X0[5].tobytes()
    finally:
        b.free()


def test_edge_cases(cs):
    s = bc.scene(13)
    s["offsets"] = np.concatenate([s["offsets"], [int(s["offsets"][-1]) + 5]]).astype(np.int32)   # malformed
    s["X0"] = np.concatenate([s["X0"], np.zeros((1, 3))])
    s["members"] = s["members"].copy()
    s["members"][0] = (99, 0)                                   # invalid member
    s["members"][4, 1] = 10 ** 6                                # invalid member
    b = Bundle(cs, s)
    try:
        fixed = bc.gauge(s["t0"])
        ones = b.run(fixed=fixed, use=False, maxIterations=5)
        b.d_use.upload(np.ones(b.M, np.uint8))
        alls = b.run(fixed=fixed, maxIterations=5)
        for key in ("R", "t", "X", "err", "inl", "cost", "trace", "stats"):
            assert ones[key].tobytes() == alls[key].tobytes(), key
        assert ones["stats"][1] == 1 and ones["stats"][2] == 2
        assert ones["launches"] == LAUNCHES
        # maxIterations = 0: evaluation only
        b.d_use.upload(np.asarray(s["use"], np.uint8))
        ev = b.run(fixed=fixed, maxIterations=0)
        P = b.oracle(fixed=fixed)
        assert ev["r"] == 0 and ev["stats"][6] == 0
        assert ev["R"].tobytes() == b.Rs.tobytes() and ev["t"].tobytes() == b.ts.tobytes()
        assert ev["X"].tobytes() == np.ascontiguousarray(s["X0"]).tobytes()
        c0, _ = P.cost(P.R0, P.t0, P.X0)
        np.testing.assert_allclose(ev["cost"], [c0, c0], rtol=1e-12)
        err, inl, written = P.outputs(P.R0, P.t0, P.X0, 4.0)
        np.testing.assert_array_equal(ev["inl"][written], inl[written].astype(np.uint8))
        np.testing.assert_allclose(ev["err"][written], err[written], rtol=1e-6)
        assert (ev["err"][~written] == SENTINEL_F).all() and (ev["inl"][~written] == 0xAB).all()
        # every camera held: structure only, no CG iteration
        st = b.run(fixed=np.ones(b.S, np.uint8), maxIterations=5, memberOutputs=False)
        assert st["stats"][5] == 0 and st["stats"][7] == 0 and st["r"] > 0
        assert st["R"].tobytes() == b.Rs.tobytes() and st["t"].tobytes() == b.ts.tobytes()
        Ps = b.oracle(fixed=np.ones(b.S, np.uint8))
        R, t, X, cost, trace, acc = Ps.run(5, 100, 1e-6)
        np.testing.assert_allclose(st["X"], X, atol=1e-6)
        # an observation behind its camera is not used
        X0 = s["X0"].copy()
        k = 2
        a = int(s["members"][int(s["offsets"][k]), 0])
        C = -s["R0"][a].T @ s["t0"][a]
        X0[k] = C - 3.0 * s["R0"][a][2]                        # behind camera a
        bh = b.run(points=X0, fixed=fixed, maxIterations=0)
        Pb = b.oracle(points=X0, fixed=fixed)
        np.testing.assert_array_equal(bh["stats"][:6], Pb.stats[:6])
        assert bh["stats"][3] < ev["stats"][3]
    finally:
        b.free()


def test_determinism_and_launches(cs):
    s = bc.scene(17)
    b = Bundle(cs, s)
    try:
        x = b.run(fixed=bc.gauge(s["t0"]))
        y = b.run(fixed=bc.gauge(s["t0"]))
        for key in ("R", "t", "X", "err", "inl", "cost", "trace", "stats"):
            assert x[key].tobytes() == y[key].tobytes(), key
        assert x["launches"] == LAUNCHES and x["ms"] > 0
    finally:
        b.free()
    # 500 images: 16 tiles of 32 cameras, so the camera phases and their partials span several CTAs
    L = bc.large(0, 500, 250000, perPoint=4)
    b = Bundle(cs, L)
    try:
        x = b.run(fixed=bc.gauge(L["t0"]), maxIterations=3)
        y = b.run(fixed=bc.gauge(L["t0"]), maxIterations=3)
        for key in ("R", "t", "X", "err", "inl", "cost", "trace", "stats"):
            assert x[key].tobytes() == y[key].tobytes(), key
        assert x["stats"][3] == 10 ** 6 and x["launches"] == LAUNCHES
        assert x["cost"][1] < x["cost"][0] and x["stats"][7] > 3
    finally:
        b.free()


def test_many_cameras_against_the_oracle(cs):
    """300 images (10 tiles of 32 cameras over two CTAs) against the float64 statement.  The circle's long chain of
    cameras is ill-conditioned, so CG runs tens of iterations, and the comparison is to 1e-6 rather than 1e-9."""
    s = bc.large(3, 300, 4000, perPoint=10)
    b = Bundle(cs, s)
    try:
        fixed = bc.gauge(s["t0"])
        P = b.oracle(fixed=fixed)
        R, t, X, cost, trace, acc = P.run(2, 100, 1e-4)
        assert clear_iterations(P) == 2 and (trace[:, 3] == 1).all()
        got = b.run(fixed=fixed, maxIterations=2, maxLinear=100, tol=1e-4)
        assert got["r"] == acc == 2
        np.testing.assert_array_equal(got["trace"][:, 2], trace[:, 2])
        np.testing.assert_allclose(got["trace"][:, 0], trace[:, 0], rtol=1e-6)
        np.testing.assert_allclose(got["cost"], cost, rtol=1e-6)
        np.testing.assert_allclose(got["R"], R, rtol=0, atol=1e-6)
        np.testing.assert_allclose(got["t"], t, rtol=0, atol=1e-5)
        np.testing.assert_allclose(got["X"], X, rtol=0, atol=1e-5)
    finally:
        b.free()


def test_no_images_with_tracks(cs):
    """numImages == 0 with tracks runs on the device: every member is invalid, the well-formed tracks' member outputs
    are NaN and 0, the points do not move, and the statistics count the tracks and members."""
    s = bc.scene(21, numPoints=20)
    s["offsets"] = np.concatenate([s["offsets"], [int(s["offsets"][-1]) + 3]]).astype(np.int32)   # malformed
    s["X0"] = np.concatenate([s["X0"], np.zeros((1, 3))])
    M = len(s["members"])
    b = Scene(cs, [], np.zeros((0, 3, 3)), np.zeros((0, 3, 3)), np.zeros((0, 3)), s["offsets"], s["members"])
    T = b.T
    pts, err, inl = cs.DeviceBuffer(8 * 3 * T), cs.DeviceBuffer(4 * M), cs.DeviceBuffer(M)
    try:
        pts.upload(s["X0"])
        err.upload(np.zeros(M, np.float32))
        inl.upload(np.full(M, 7, np.uint8))
        cost, stats = np.full(2, 5.0), np.full(8, 7, np.int64)
        r = cs.lib().cs_bundle_adjust(None, 0, None, None, None, None, b.d_off.ptr, T, b.d_mem.ptr, M, None, pts.ptr,
                                      10, 50, 1e-6, 4.0, None, None, err.ptr, inl.ptr, cost.ctypes.data, None,
                                      stats.ctypes.data, None)
        assert r == 0, cs.lib().cs_last_error().decode()
        assert stats.tolist() == [T - 1, 1, M, 0, 0, 0, 0, 0] and not cost.any()
        assert np.isnan(err.download(np.float32, M)).all() and not inl.download(np.uint8, M).any()
        assert pts.download(np.float64, 3 * T).tobytes() == np.ascontiguousarray(s["X0"]).tobytes()
    finally:
        for buf in (pts, err, inl):
            buf.free()
        b.free()


def test_wrapper_default_gauge_and_scipy_optimum(cs):
    from scipy.optimize import least_squares
    s = bc.scene(19, numImages=5, numPoints=60)
    datas = []
    try:
        for p in s["xy"]:
            d = cs.SiftData()
            cs.InitSiftData(d, max(len(p), 1))
            rec = np.zeros(len(p), cs.SIFT_DTYPE)
            rec["xpos"], rec["ypos"] = p[:, 0], p[:, 1]
            d._buf.upload(rec)
            d.numPts = len(p)
            datas.append(d)
        R, t, X, err, inl, cost, trace, stats, ms = cs.BundleAdjust(
            datas, s["K"], s["R0"], s["t0"], s["offsets"], s["members"], s["X0"], use=s["use"], maxIterations=100,
            linearTol=1e-10)
        P = bo.Problem(s["xy"], s["K"], s["R0"], s["t0"], s["offsets"], s["members"], s["X0"], use=s["use"],
                       fixed=bc.gauge(s["t0"]))
        assert R[0].tobytes() == np.ascontiguousarray(s["R0"][0]).tobytes()
        assert len(trace) == stats[6] and cost[1] < cost[0]
        # scipy's optimum over the same parameters and gauge
        free = P.mask

        def unpack(v):
            dc = np.zeros((P.S, 6))
            dc[free] = v[:free.sum()]
            Rr, tt = P.apply(P.R0, P.t0, free, dc)
            XX = P.X0.copy()
            XX[P.parts] = P.X0[P.parts] + v[free.sum():].reshape(-1, 3)
            return Rr, tt, XX

        def fun(v):
            return P.residuals(*unpack(v))[0].reshape(-1)
        v0 = np.zeros(free.sum() + 3 * len(P.parts))
        sol = least_squares(fun, v0, method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
        best = float(sol.fun @ sol.fun)
        assert abs(cost[1] - best) <= 1e-6 * best, (cost, best)
    finally:
        for d in datas:
            cs.FreeSiftData(d)


def test_chain_on_extracted_views(cs):
    """The six shifted views of the incremental chain test (a plane Z = Z0 = 10 seen by cameras R = I, f = 200,
    translated by the shifts): extraction, the ratio, verify and guided batches, BuildTracks, then TriangulateTracks
    with views 2 to 5 given about two pixels of pose error, then BundleAdjust with the default gauge (view 0 held, view
    1's x held, both true).  The reprojection RMS falls, every pose ends within the pose test's one-pixel bounds
    (|R - I| <= 1 / f, |t_xy - t_xy true| <= Z0 / f, |t_z| <= Z0 / (w / 2)), and triangulating again loses no track.
    The second triangulation drops the angle test: at these baselines (0.3 to 0.8 units at depth 10) a two-view
    track's angle can fall below 0.5 degrees when its poses are corrected (one track of about 1 100 here), which says
    nothing about the adjustment."""
    c = bc.chain(cs)
    datas, offsets, members, K, ts, Rs, ts0 = (c[k] for k in ("datas", "offsets", "members", "K", "ts", "Rs", "ts0"))
    f, Z0, w = c["f"], c["Z0"], c["w"]
    try:
        pts, cnt, err0, inl0, stats, _ = cs.TriangulateTracks(datas, K, Rs, ts0, offsets, members, numTrials=64,
                                                              maxError=4.0, minTriAngle=0.5, seed=1)
        assert stats[5] > 100
        R, t, X, err, inl1, cost, trace, st, ms = cs.BundleAdjust(datas, K, Rs, ts0, offsets, members, pts, use=inl0,
                                                                  maxError=4.0)
        assert ms > 0 and cost[1] < cost[0] and st[4] > 100
        rms0 = np.sqrt(np.mean(err0[inl0].astype(np.float64) ** 2))
        rms1 = np.sqrt(np.mean(err[inl0].astype(np.float64) ** 2))
        assert rms1 < rms0, (rms0, rms1)
        assert R[0].tobytes() == np.eye(3).tobytes() and t[0].tobytes() == ts[0].tobytes() and t[1][0] == ts[1][0]
        for a in range(6):
            assert np.abs(R[a] - np.eye(3)).max() <= 1 / f, (a, R[a])
            assert np.abs(t[a][:2] - ts[a][:2]).max() <= Z0 / f and abs(t[a][2]) <= Z0 / (w / 2), (a, t[a])
        pts2, cnt2, _, _, _, _ = cs.TriangulateTracks(datas, K, R, t, offsets, members, numTrials=64, maxError=4.0,
                                                      minTriAngle=0.0, seed=1)
        assert (cnt2[cnt > 0] > 0).all()
    finally:
        for d in datas:
            cs.FreeSiftData(d)
