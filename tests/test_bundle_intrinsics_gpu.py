"""cs_bundle_adjust_intrinsics and cs_undistort_records on the device against the float64 statement in
bundle_intrinsics_oracle.py, the truth of distorted scenes, cs_bundle_adjust and the pinhole stages downstream."""
import ctypes

import numpy as np
import pytest

import bundle_cases as bc
import bundle_intrinsics_cases as bic
import bundle_intrinsics_oracle as bio
from test_bundle_gpu import Bundle, clear_iterations

pytestmark = pytest.mark.gpu
LAUNCHES = 3
FOCAL, K1, K2 = 1, 2, 4


class Calib(Bundle):
    """A bundle_intrinsics_cases scene in device memory, started from its guessed K0."""

    def __init__(self, cs, s):
        s = dict(s, K=s["K0"], Ktrue=s["K"])
        super().__init__(cs, s)

    def run_i(self, refine=FOCAL | K1, loss=0, lossScale=1.0, dists=None, fixed=None, use=True, maxIterations=30,
              maxLinear=100, tol=1e-6, maxError=4.0, points=None):
        cs, T, M, S = self.cs, self.T, self.M, self.S
        X = np.ascontiguousarray(self.s["X0"] if points is None else points, np.float64)
        fix = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
        ref = None if refine is None else np.ascontiguousarray(np.broadcast_to(refine, (S,)), np.uint8)
        dist = None if dists is None else np.ascontiguousarray(dists, np.float64)
        outs = [cs.DeviceBuffer(8 * 3 * T), cs.DeviceBuffer(4 * M), cs.DeviceBuffer(M)]
        K_out, d_out = np.zeros((S, 3, 3)), np.zeros((S, 2))
        R_out, t_out = np.zeros((S, 3, 3)), np.zeros((S, 3))
        cost, trace = np.zeros(2), np.zeros((maxIterations, 4))
        stats, ms = np.zeros(8, np.int64), ctypes.c_double(0.0)
        try:
            outs[0].upload(X)
            before = cs.lib().cs_launch_count()
            r = cs.lib().cs_bundle_adjust_intrinsics(
                self.sets, S, self.Ks.ctypes.data, dist.ctypes.data if dist is not None else None,
                ref.ctypes.data if ref is not None else None, loss, lossScale, self.Rs.ctypes.data,
                self.ts.ctypes.data, fix.ctypes.data if fix is not None else None, self.d_off.ptr, T, self.d_mem.ptr,
                M, self.d_use.ptr if use else None, outs[0].ptr, maxIterations, maxLinear, tol, maxError,
                K_out.ctypes.data, d_out.ctypes.data, R_out.ctypes.data, t_out.ctypes.data, outs[1].ptr, outs[2].ptr,
                cost.ctypes.data, trace.ctypes.data if maxIterations else None, stats.ctypes.data, ctypes.byref(ms))
            launches = cs.lib().cs_launch_count() - before
            assert r >= 0, cs.lib().cs_last_error().decode()
            pts = outs[0].download(np.float64, 3 * T).reshape(T, 3)
            err, inl = outs[1].download(np.float32, M), outs[2].download(np.uint8, M)
        finally:
            for b in outs:
                b.free()
        return dict(r=r, K=K_out, k=d_out, R=R_out, t=t_out, X=pts, err=err, inl=inl, cost=cost, trace=trace,
                    stats=stats, ms=ms.value, launches=launches)

    def oracle_i(self, refine=FOCAL | K1, loss=0, lossScale=1.0, dists=None, fixed=None, use=True):
        return bio.Intrinsics(self.xy, self.Ks, self.Rs, self.ts, self.offsets, self.members, self.s["X0"],
                              dists=dists, refine=refine, loss=loss, lossScale=lossScale,
                              use=self.s["use"] if use else None, fixed=fixed)


@pytest.mark.parametrize("loss", [0, 2])
@pytest.mark.parametrize("refine", [FOCAL, FOCAL | K1, FOCAL | K1 | K2])
def test_trace_against_the_oracle(cs, refine, loss):
    s = bic.scene(5, noise=0.5, outlier=0.1)
    b = Calib(cs, s)
    try:
        fixed = bc.gauge(s["t0"])
        kw = dict(refine=refine, loss=loss, lossScale=2.0, fixed=fixed)
        P = b.oracle_i(**kw)
        P.run(20, 100, 1e-6)
        n = clear_iterations(P)
        assert n >= 3
        P = b.oracle_i(**kw)
        K, k, R, t, X, cost, trace, acc = P.run(n, 100, 1e-6)
        got = b.run_i(maxIterations=n, **kw)
        n = len(trace)
        assert got["r"] == acc and got["stats"][6] == n and got["launches"] == LAUNCHES
        np.testing.assert_array_equal(got["trace"][:n, 3], trace[:, 3])
        np.testing.assert_array_equal(got["trace"][:n, 2], trace[:, 2])
        np.testing.assert_allclose(got["trace"][:n, 0], trace[:, 0], rtol=1e-9)
        np.testing.assert_allclose(got["cost"], cost, rtol=1e-9)
        np.testing.assert_allclose(got["K"], K, rtol=1e-9)
        np.testing.assert_allclose(got["k"], k, rtol=0, atol=1e-9)
        np.testing.assert_allclose(got["R"], R, rtol=0, atol=1e-6)
        np.testing.assert_allclose(got["X"], X, rtol=0, atol=1e-6)
        np.testing.assert_array_equal(got["stats"][:6], P.stats[:6])
        err, inl, written = P.outputs9(K, k, R, t, X, 4.0)
        np.testing.assert_array_equal(got["inl"][written], inl[written].astype(np.uint8))
        np.testing.assert_allclose(got["err"][written], err[written], rtol=1e-5)
    finally:
        b.free()


def test_focal_and_distortion_recovered_from_a_guess(cs):
    s = bic.scene(7, k=(-0.1, 0.0), focal=1.08, noise=0.0, numPoints=200)
    b = Calib(cs, s)
    try:
        got = b.run_i(refine=FOCAL | K1, fixed=bc.gauge(s["t"]), maxIterations=100, tol=1e-10)
        # noise-free but for the float32 rounding of the record positions (about 3e-5 px per coordinate at 1 000 px):
        # the optimum's cost is of that order squared per observation, and the parameters move by about that rounding
        # over the focal length (3e-8 relative) times the conditioning of the block
        assert got["cost"][1] < 1e-6 and got["cost"][0] > 1e4
        np.testing.assert_allclose(got["K"], s["K"], rtol=1e-6)
        np.testing.assert_allclose(got["k"], s["k"], rtol=0, atol=1e-6)
        np.testing.assert_allclose(got["R"], s["R"], atol=1e-6)
        np.testing.assert_allclose(got["t"], s["t"], atol=1e-5)
    finally:
        b.free()


def test_held_values_determinism_and_the_plain_call(cs):
    s = bic.scene(11, noise=0.5)
    b = Calib(cs, s)
    try:
        fixed = np.array([1, 3, 0, 1, 0, 0], np.uint8)
        refine = np.array([7, 1, 0, 3, 6, 0], np.uint8)
        dists = np.tile([0.01, -0.002], (6, 1))
        x = b.run_i(refine=refine, dists=dists, fixed=fixed, loss=2, lossScale=2.0, maxIterations=8)
        y = b.run_i(refine=refine, dists=dists, fixed=fixed, loss=2, lossScale=2.0, maxIterations=8)
        assert x["r"] > 0 and x["launches"] == LAUNCHES
        for key in ("K", "k", "R", "t", "X", "err", "inl", "cost", "trace", "stats"):
            assert x[key].tobytes() == y[key].tobytes(), key
        K0 = b.Ks
        for a in (0, 3):
            assert x["R"][a].tobytes() == b.Rs[a].tobytes() and x["t"][a].tobytes() == b.ts[a].tobytes()
        for a in (2, 5):
            assert x["K"][a].tobytes() == K0[a].tobytes() and x["k"][a].tobytes() == dists[a].tobytes()
        assert x["k"][1].tobytes() == dists[1].tobytes() and x["K"][4].tobytes() == K0[4].tobytes()
        assert x["k"][3][1].tobytes() == dists[3][1].tobytes() and x["k"][4][0] != dists[4][0]
        assert x["t"][1][1].tobytes() == b.ts[1][1].tobytes()
        assert x["K"][1][0, 0] != K0[1][0, 0] and x["k"][0][1] != dists[0][1]
        # no refinement, zero k, trivial loss: cs_bundle_adjust's bytes
        fixed = bc.gauge(s["t0"])
        p = b.run_i(refine=None, fixed=fixed, maxIterations=10)
        q = b.run(fixed=fixed, maxIterations=10)
        for key in ("R", "t", "X", "err", "inl", "cost", "trace", "stats"):
            assert p[key].tobytes() == q[key].tobytes(), key
        assert p["K"].tobytes() == b.Ks.tobytes() and not p["k"].any()
    finally:
        b.free()


def test_cauchy_beats_the_squared_loss_under_gross_outliers(cs):
    s = bic.scene(13, noise=0.5, outlier=0.2)
    b = Calib(cs, s)
    try:
        fixed = bc.gauge(s["t"])
        errs = {}
        for loss in (0, 2):
            got = b.run_i(refine=FOCAL | K1, loss=loss, lossScale=2.0, fixed=fixed, use=False, maxIterations=100)
            rot = max(np.abs(got["R"][a] - s["R"][a]).max() for a in range(b.S))
            foc = np.abs(got["K"][:, 0, 0] / s["K"][:, 0, 0] - 1).max()
            errs[loss] = (rot, foc)
        assert errs[2][0] < errs[0][0] and errs[2][1] < errs[0][1], errs
    finally:
        b.free()


def _records(cs, xy, extra=None):
    datas = []
    for p in xy:
        d = cs.SiftData()
        cs.InitSiftData(d, max(len(p), 1))
        rec = np.zeros(len(p), cs.SIFT_DTYPE)
        rec["xpos"], rec["ypos"] = p[:, 0], p[:, 1]
        if extra is not None:
            extra(rec)
        d._buf.upload(rec)
        d.numPts = len(p)
        datas.append(d)
    return datas


def test_undistort_records_against_the_rule(cs):
    rng = np.random.default_rng(4)
    K = np.array([[[900.0, 2.0, 640], [0, 880, 480], [0, 0, 1]], [[500.0, 0, 320], [0, 500, 240], [0, 0, 1]]])
    k = np.array([[-0.2, 0.05], [-0.5, 0.0]])
    xy = [rng.uniform([0, 0], [1280, 960], (3000, 2)).astype(np.float32),
          np.concatenate([rng.uniform([0, 0], [640, 480], (500, 2)), [[np.nan, 1.0], [320, 240]]]).astype(np.float32)]

    def extra(rec):
        rec["scale"] = rng.uniform(1, 5, len(rec))
        rec["orientation"] = rng.uniform(0, 360, len(rec))
        rec["data"] = rng.uniform(0, 1, rec["data"].shape)

    datas = _records(cs, xy, extra)
    outs = []
    try:
        before = cs.lib().cs_launch_count()
        outs = cs.UndistortRecords(datas, K, k)
        assert cs.lib().cs_launch_count() - before == 1
        for a in range(2):
            src = datas[a]._buf.download(cs.SIFT_DTYPE, datas[a].numPts)
            got = outs[a]._buf.download(cs.SIFT_DTYPE, outs[a].numPts)
            want = bio.undistort(K[a], k[a], xy[a])
            pos = np.stack([got["xpos"], got["ypos"]], 1)
            assert (np.isnan(pos) == np.isnan(want)).all()
            np.testing.assert_allclose(pos[np.isfinite(want)], want[np.isfinite(want)], rtol=1e-6, atol=0)
            g, w = got.copy(), src.copy()
            g["xpos"] = g["ypos"] = w["xpos"] = w["ypos"] = 0
            assert g.tobytes() == w.tobytes()
        assert np.isnan(want).any() and np.isfinite(want).sum() > 200
        # in place: the same bytes
        ptrs = (ctypes.c_void_p * 2)(*[d.d_data for d in datas])
        r = cs.lib().cs_undistort_records(cs._set_table(datas), 2, np.ascontiguousarray(K).ctypes.data,
                                          np.ascontiguousarray(k).ctypes.data, ptrs, None)
        assert r == 0
        for a in range(2):
            assert (datas[a]._buf.download(cs.SIFT_DTYPE, datas[a].numPts).tobytes() ==
                    outs[a]._buf.download(cs.SIFT_DTYPE, outs[a].numPts).tobytes())
    finally:
        for d in datas + outs:
            cs.FreeSiftData(d)


def test_calibrated_loop_end_to_end(cs):
    """Adjust a distorted scene from a guessed K, undistort with the refined model, then triangulate and register with
    the refined K; the same with the true K and k.  Triangulated inlier counts and registered inlier counts agree
    within 2 %, rotations within 2e-3.  Translations agree within 0.25 (2.5 % of the 10-unit camera distance): with
    0.3 px of noise the refined focal length is off by a fraction of a percent, and each run's points and poses move
    together with it, so the registered positions differ by that fraction of the distance."""
    s = bic.scene(17, k=(-0.1, 0.0), focal=1.06, noise=0.3, numPoints=300)
    datas = _records(cs, s["xy"])
    und = []
    try:
        K, k, R, t, X, err, inl, cost, trace, st, ms = cs.BundleAdjustIntrinsics(
            datas, s["K0"], s["R0"], s["t0"], s["offsets"], s["members"], s["X0"], refine=FOCAL | K1,
            maxIterations=100, linearTol=1e-10)
        assert cost[1] < cost[0] and ms > 0
        runs = {}
        for name, KK, kk, RR, tt in (("refined", K, k, R, t), ("truth", s["K"], s["k"], s["R"], s["t"])):
            u = cs.UndistortRecords(datas, KK, kk)
            und += u
            pts, cnt, _, tin, _, _ = cs.TriangulateTracks(u, KK, RR, tt, s["offsets"], s["members"],
                                                          numTrials=64, maxError=2.0, minTriAngle=0.5, seed=1)
            trackOf = [np.full(d.numPts, -1, np.int64) for d in u]
            for kk_ in range(len(s["offsets"]) - 1):
                for m in range(int(s["offsets"][kk_]), int(s["offsets"][kk_ + 1])):
                    a, f = s["members"][m]
                    trackOf[a][f] = kk_
            Rp, tp, counts, _, _, _, _ = cs.AbsolutePoseBatch(u, trackOf, pts, KK, numLoops=256, maxError=2.0)
            runs[name] = (int(tin.sum()), Rp, tp, counts)
        (n1, R1, t1, c1), (n2, R2, t2, c2) = runs["refined"], runs["truth"]
        assert abs(n1 - n2) <= 0.02 * n2, (n1, n2)
        assert (np.abs(c1 - c2) <= 0.02 * c2 + 1).all(), (c1, c2)
        np.testing.assert_allclose(R1, R2, atol=2e-3)
        np.testing.assert_allclose(t1, t2, atol=0.25)
    finally:
        for d in datas + und:
            cs.FreeSiftData(d)
