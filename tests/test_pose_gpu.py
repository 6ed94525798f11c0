"""GPU checks of camera registration (cs_absolute_pose_batch, cs_absolute_pose_models) against the float64 statement
(tests/pose_oracle.py): every slot's pose and count; counts, inlier bytes and statistics exactly, poses to a stated
tolerance and errors to float rounding, with every inlier decision kept out of its boundary band; the pose against the
ground truth; bit-identical jobs alone, in a batch, permuted, repeated and over several waves; edge cases; sentinels
and NULL per-feature outputs; and the incremental chain on the six shifted views of the triangulation chain test."""
import ctypes
import itertools

import numpy as np
import pytest

import pose_cases as pc
import pose_oracle as po
from cudasift_b200.synth import synth_image

pytestmark = pytest.mark.gpu
LAUNCHES = 5
BAND = 1e-6
SENTINEL_F = np.float32(-12345.0)
SENTINEL_B = 0xA5


class Batch:
    """Record sets, pointOf tables and points in device memory, and one call of cs_absolute_pose_batch with a sentinel
    past every per-feature output."""

    def __init__(self, cs, xys, pointOfs, points):
        self.cs, self.bufs = cs, []
        self.xys, self.pointOfs, self.points = xys, [np.asarray(p, np.int32) for p in pointOfs], np.asarray(points)
        self.rec, self.pof = [], []
        for xy, pof in zip(xys, self.pointOfs):
            r = self._buf(pc.records(xy))
            p = self._buf(pof)
            self.rec.append(r)
            self.pof.append(p)
        self.d_points = self._buf(np.ascontiguousarray(self.points, np.float64).reshape(-1, 3))

    def _buf(self, a):
        b = self.cs.DeviceBuffer(max(a.nbytes, 8))
        if a.nbytes:
            b.upload(a)
        self.bufs.append(b)
        return b

    def run(self, Ks, numLoops, maxError, seeds, order=None, outputs=True):
        """Jobs in the given order.  Returns (r, R [J, 3, 3], t, counts, errors list, inlier list, stats, ms) in that
        order; errors and inlier None without per-feature outputs."""
        cs = self.cs
        order = list(range(len(self.xys))) if order is None else list(order)
        J = len(order)
        outs = []
        table = (cs.PoseJob * max(J, 1))()
        for q, p in enumerate(order):
            n = len(self.xys[p])
            e = cs.DeviceBuffer(4 * (n + 1))
            i = cs.DeviceBuffer(n + 1)
            e.upload(np.full(n + 1, SENTINEL_F, np.float32))
            i.upload(np.full(n + 1, SENTINEL_B, np.uint8))
            outs.append((e, i))
            table[q] = cs.PoseJob(self.rec[p].ptr if n else None, n, self.pof[p].ptr if n else None, int(seeds[p]),
                                  e.ptr if outputs else None, i.ptr if outputs else None)
        K = np.ascontiguousarray(np.asarray(Ks, np.float64).reshape(-1, 3, 3)[order])
        R, t = np.full((J, 3, 3), 7.0), np.full((J, 3), 7.0)
        counts, stats, ms = np.full(J, -9, np.int32), np.full((J, 8), -9, np.int64), ctypes.c_double(0.0)
        try:
            r = cs.lib().cs_absolute_pose_batch(self.d_points.ptr, len(self.points), table, J, K.ctypes.data, numLoops,
                                                float(maxError), R.ctypes.data, t.ctypes.data, counts.ctypes.data,
                                                stats.ctypes.data, ctypes.byref(ms))
            errors, inlier = [], []
            for q, p in enumerate(order):
                n = len(self.xys[p])
                e = outs[q][0].download(np.float32, n + 1)
                i = outs[q][1].download(np.uint8, n + 1)
                assert e[n] == SENTINEL_F and i[n] == SENTINEL_B
                if outputs:
                    assert set(np.unique(i[:n])) <= {0, 1}
                    errors.append(e[:n])
                    inlier.append(i[:n].astype(bool))
                else:
                    assert (e == SENTINEL_F).all() and (i == SENTINEL_B).all()
        finally:
            for e, i in outs:
                e.free()
                i.free()
        return r, R, t, counts, errors if outputs else None, inlier if outputs else None, stats, ms.value

    def models(self, p, K, numLoops, maxError, seed):
        cs = self.cs
        n = len(self.xys[p])
        job = cs.PoseJob(self.rec[p].ptr, n, self.pof[p].ptr, int(seed), None, None)
        S = 4 * numLoops
        R, t, c = np.zeros((S, 3, 3)), np.zeros((S, 3)), np.zeros(S, np.int32)
        V = cs.lib().cs_absolute_pose_models(self.d_points.ptr, len(self.points), ctypes.byref(job),
                                             np.ascontiguousarray(K, np.float64).ctypes.data, numLoops,
                                             float(maxError), R.ctypes.data, t.ctypes.data, c.ctypes.data)
        return V, R, t, c

    def free(self):
        for b in self.bufs:
            b.free()


def oracle(b, Ks, numLoops, maxError, seeds):
    band = po.Band()
    return [po.pose_job(b.xys[p], b.pointOfs[p], b.points, Ks[p], numLoops, maxError, seeds[p], band)
            for p in range(len(b.xys))], band


def compare(got, want, band, rtol_pose=1e-6):
    """Counts, inlier bytes and statistics exactly (every decision at least BAND from its boundary), R and t to
    rtol_pose: the refinement sums per warp lane on the device and in rank order here, and it stops on a step of 1e-12
    or a relative decrease of 1e-12, so the two minima agree far below 1e-6.  Errors to float rounding."""
    r, R, t, counts, errors, inlier, stats, ms = got
    assert band.e2 > BAND, band.e2
    assert r == sum(w["count"] > 0 for w in want)
    for p, w in enumerate(want):
        n = len(w["errors"])
        st = stats[p].tolist()
        if n == 0:
            assert counts[p] == 0 and st == [0] * 8 and not R[p].any() and not t[p].any()
            continue
        assert counts[p] == w["count"] and st == w["stats"].tolist(), (p, st, w["stats"].tolist())
        scale = 1.0 + np.abs(w["t"]).max()
        assert np.abs(R[p] - w["R"]).max() <= rtol_pose and np.abs(t[p] - w["t"]).max() <= rtol_pose * scale, p
        if errors is not None:
            assert np.array_equal(inlier[p], w["inlier"]), p
            e, f = errors[p], w["errors"]
            assert np.array_equal(np.isnan(e), np.isnan(f)) and np.array_equal(np.isinf(e), np.isinf(f)), p
            fin = np.isfinite(f)
            assert np.allclose(e[fin], f[fin], rtol=1e-5, atol=1e-4), p


SIZES = [3, 4, 7, 30, 200, 1000, 5000, 0, 2]


def test_slots_match_the_oracle(cs):
    """Every slot of cs_absolute_pose_models: the same empty slots, R and t to 1e-9 (t relative to its scale), counts
    exactly.  Both run the same FP64 formulas; only contraction into fused multiply-adds differs."""
    xys, pofs, pts, Ks, Rs, ts = pc.batch(11, [40, 600, 2000], outliers=(0.2, 0.5))
    b = Batch(cs, xys, pofs, pts)
    try:
        for p, L in ((0, 64), (1, 128), (2, 96)):
            V, R, t, c = b.models(p, Ks[p], L, 4.0, 100 + p)
            ok, pos, Xw, px, _ = po.correspondences(xys[p], pofs[p], pts)
            assert V == len(pos)
            wR, wt, _ = po.slot_models(Ks[p], Xw, po.bearings(Ks[p], px), L, 100 + p)
            live = ~np.isnan(wR[:, 0, 0])
            assert np.array_equal(~np.isnan(R[:, 0, 0]), live) and live.sum() > L
            assert np.isnan(R[~live]).all() and np.isnan(t[~live]).all() and not c[~live].any()
            dR = np.abs(R[live] - wR[live]).max(axis=(1, 2))
            dt = np.abs(t[live] - wt[live]).max(axis=1) / (1 + np.abs(wt[live]).max(axis=1))
            assert dR.max() <= 1e-9 and dt.max() <= 1e-9, (dR.max(), dt.max())
            band = po.Band()
            inl, d, e = po.inliers(po.camera(Ks[p], wR[live], wt[live]), Xw, px, 16.0)
            band.add(d, e, 16.0)
            assert band.e2 > BAND
            assert np.array_equal(c[live], inl.sum(1))
    finally:
        b.free()


@pytest.mark.parametrize("seed", [21, 22])
def test_batch_matches_the_oracle_and_the_truth(cs, seed):
    """Skewed, unequal K per job, 0.5 px noise, 10-50 % outliers, V from 0 to 5 000.  Against the ground truth: with n
    inliers of 0.5 px noise at focal length f, the pose's angular error is of order 0.5 / (f sqrt(n)) times a geometry
    factor (points within 3 units at distances 5 to 18) below 20, so a job with at least 50 inliers is within
    |R - R_true| <= 10 / (f sqrt(n)) and |t - t_true| <= 18 * 10 / (f sqrt(n))."""
    xys, pofs, pts, Ks, Rs, ts = pc.batch(seed, SIZES)
    b = Batch(cs, xys, pofs, pts)
    seeds = np.arange(len(SIZES)) * 7 + seed
    try:
        got = b.run(Ks, 256, 4.0, seeds)
        want, band = oracle(b, Ks, 256, 4.0, seeds)
        compare(got, want, band)
        r, R, t, counts = got[:4]
        assert got[-1] > 0
        for p in range(len(SIZES)):
            if counts[p] >= 50:
                bound = 10.0 / (Ks[p][0, 0] * np.sqrt(counts[p]))
                assert np.abs(R[p] - Rs[p]).max() <= bound and np.abs(t[p] - ts[p]).max() <= 18 * bound, p
        # each job alone, the jobs reversed and a repeated call: the same bytes
        for p in range(len(SIZES)):
            one = b.run(Ks, 256, 4.0, seeds, order=[p])
            for a, c in zip(one[1:4], got[1:4]):
                assert np.array_equal(a[0], c[p])
            assert np.array_equal(one[6][0], got[6][p])
            assert one[4][0].tobytes() == got[4][p].tobytes() and np.array_equal(one[5][0], got[5][p])
        rev = list(reversed(range(len(SIZES))))
        back = b.run(Ks, 256, 4.0, seeds, order=rev)
        for k in (1, 2, 3, 6):
            assert np.array_equal(back[k], got[k][rev])
        again = b.run(Ks, 256, 4.0, seeds)
        for k in (1, 2, 3, 6):
            assert got[k].tobytes() == again[k].tobytes()
        assert all(x.tobytes() == y.tobytes() for x, y in zip(got[4], again[4]))
        # NULL per-feature outputs change nothing else
        bare = b.run(Ks, 256, 4.0, seeds, outputs=False)
        for k in (1, 2, 3, 6):
            assert np.array_equal(bare[k], got[k])
    finally:
        b.free()


def test_multi_wave_batch(cs):
    """numLoops 65536: a wave holds floor(256 MiB / (4 x 65536 x 100 B)) = 10 jobs, so 23 jobs take 3 waves and 15
    launches; every job equals its single-job call bit for bit."""
    sizes = [12 + 3 * k for k in range(23)]
    xys, pofs, pts, Ks, Rs, ts = pc.batch(31, sizes, outliers=(0.0, 0.3))
    b = Batch(cs, xys, pofs, pts)
    seeds = np.arange(23) + 5
    try:
        L0 = cs.lib().cs_launch_count()
        got = b.run(Ks, 65536, 3.0, seeds)
        assert cs.lib().cs_launch_count() - L0 == LAUNCHES * 3
        assert got[0] == (got[3] > 0).sum() and got[0] >= 20
        for p in (0, 9, 10, 22):
            L0 = cs.lib().cs_launch_count()
            one = b.run(Ks, 65536, 3.0, seeds, order=[p])
            assert cs.lib().cs_launch_count() - L0 == LAUNCHES
            for k in (1, 2, 3, 6):
                assert np.array_equal(one[k][0], got[k][p])
            assert one[4][0].tobytes() == got[4][p].tobytes()
    finally:
        b.free()


def test_edge_cases(cs):
    rng = np.random.default_rng(41)
    xy, pof, X, K, R, t = pc.job(rng, 60, noise=0.3, outlier=0.0)
    P = len(X)
    pts = np.concatenate([X, [[np.nan, 0.0, 0.0]]])
    cases = []
    cases.append((xy[:2], pof[:2]))                                     # V = 2 < 3
    cases.append((xy[:10], np.full(10, -1, np.int32)))                  # no point at all
    bad = pof[:20].copy()
    bad[:5] = 10 ** 6                                                   # out of range
    bad[5:8] = P                                                        # the NaN point
    xyb = xy[:20].copy()
    xyb[8:10, 0] = np.nan                                               # NaN positions
    cases.append((xyb, bad))
    shared = np.concatenate([pof[:30], pof[:30]])                       # every point named twice
    cases.append((np.concatenate([xy[:30], xy[:30]]), shared))
    # collinear world points: every sample is degenerate
    line = np.outer(np.linspace(-1, 1, 40), [0.3, 0.2, 0.1]) + [0, 0, 0]
    u = (line @ R.T + t) @ K.T
    cases.append(((u[:, :2] / u[:, 2:]).astype(np.float32), np.arange(40, dtype=np.int32) + P + 1))
    # every point behind the camera: the pose that sees them does not exist among in-front solutions of the truth
    behind = 2 * (-R.T @ t) - X[:40]
    ub = (behind @ R.T + t) @ K.T
    cases.append(((ub[:, :2] / ub[:, 2:]).astype(np.float32), np.arange(40, dtype=np.int32) + P + 41))
    pts = np.concatenate([pts, line, behind])
    xys = [c[0] for c in cases]
    pofs = [c[1] for c in cases]
    Ks = np.stack([K] * len(cases))
    b = Batch(cs, xys, pofs, pts)
    seeds = np.arange(len(cases))
    try:
        got = b.run(Ks, 128, 2.0, seeds)
        want, band = oracle(b, Ks, 128, 2.0, seeds)
        compare(got, want, band)
        st = got[6]
        assert got[3][0] == 0 and st[0].tolist() == [2, 0, 0, 0, -1, 0, 0, 0]
        assert got[3][1] == 0 and st[1].tolist() == [0, 0, 0, 0, -1, 0, 0, 0] and np.isnan(got[4][1]).all()
        assert st[2][:2].tolist() == [10, 10] and np.isnan(got[4][2][:10]).all() and not got[5][2][:10].any()
        assert got[3][3] >= 50 and st[3][0] == 60
        assert np.array_equal(got[5][3][:30], got[5][3][30:])
        assert st[4][0] == 40 and st[4][2] == 0 and got[3][4] == 0
    finally:
        b.free()


def test_incremental_chain(cs):
    """The six shifted views of the triangulation chain test (a plane Z = Z0 = 10 seen by cameras R = I, f = 200,
    translated in X and Y by the shifts): extraction, the ratio, verify and guided batches, BuildTracks, then
    TriangulateTracks with view 5's set left empty, then AbsolutePoseBatch of view 5 from trackOf and the points.
    Bound: the registered pose moves a point of the plane by less than one pixel when |R - I| <= 1 / f (a rotation
    of one pixel at the centre), |t_xy - t5_xy| <= Z0 / f (one pixel of translation) and |t_z| <= Z0 / (w / 2) (one
    pixel of scale at the image edge); keypoints of these integer shifts are good to about 0.1 px, and the pose
    averages over hundreds of them.  Then TriangulateTracks with all six cameras: no track loses its point."""
    w, h = 960, 540
    img = synth_image(w, h, seed=9)
    shifts = [(0, 0), (3, 5), (-4, 6), (8, -2), (-6, -7), (10, 9)]
    views = [np.ascontiguousarray(np.roll(img, s, axis=(0, 1))) for s in shifts]
    pitch = cs.iAlignUp(w, 128)
    cis = [cs.CudaImage().Allocate(w, h, pitch, False, None, v) for v in views]
    for ci in cis:
        ci.Download()
    ex = cs.Extractor(w, h, 5, 1000, False, batch=6, maxCandidates=16384)
    datas = []
    try:
        ex.submit_device_batch([ci.d_data for ci in cis], pitch, 1.0, 3.0, 0.0)
        counts = ex.wait_batch(6)
        for i in range(6):
            d = cs.SiftData()
            cs.InitSiftData(d, int(counts[i]))
            d._buf.upload(ex.device_points_at(i, int(counts[i])))
            d.numPts = int(counts[i])
            datas.append(d)
    finally:
        ex.close()

    class Empty:
        d_data, numPts = None, 0
    try:
        pairs_idx = list(itertools.combinations(range(6), 2))
        ratio, _, _ = cs.MatchSiftDataRatioBatch(datas, pairs_idx)
        Mv, inl, _, _ = cs.VerifyPairsBatch([(datas[a], datas[b], ratio[k], k) for k, (a, b) in enumerate(pairs_idx)],
                                            "fundamental", 1024, 4.0)
        keep = [k for k in range(len(pairs_idx)) if len(inl[k]) >= 30]
        jobs = [pairs_idx[k] for k in keep]
        guided, _, _ = cs.MatchSiftDataGuidedBatch(datas, jobs, "fundamental", Mv[keep], 4.0)
        sizes = [d.numPts for d in datas]
        offsets, members, trackOf, _, _ = cs.BuildTracks(sizes, [(a, b, g) for (a, b), g in zip(jobs, guided)])
        f, Z0 = 200.0, 10.0
        K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]])
        ts = np.array([[dx * Z0 / f, dy * Z0 / f, 0.0] for dy, dx in shifts])
        five = datas[:5] + [Empty()]
        pts, cnt, _, _, stats, _ = cs.TriangulateTracks(five, K, np.eye(3), ts, offsets, members, numTrials=64,
                                                        maxError=1.0, minTriAngle=0.5, seed=1)
        assert stats[5] > 100
        base = sum(sizes[:5])
        pointOf = trackOf[base:base + sizes[5]]
        R, t, c, err, inlier, st, ms = cs.AbsolutePoseBatch([datas[5]], [pointOf], pts, K, numLoops=256, maxError=1.0)
        assert ms > 0 and c[0] >= 100 and st[0][0] >= c[0]
        assert np.abs(R[0] - np.eye(3)).max() <= 1 / f, R[0]
        assert np.abs(t[0][:2] - ts[5][:2]).max() <= Z0 / f and abs(t[0][2]) <= Z0 / (w / 2), t[0]
        assert inlier[0].sum() == c[0] and (err[0][inlier[0]] < 1.0).all()
        ts2 = ts.copy()
        ts2[5] = t[0]
        Rs2 = np.stack([np.eye(3)] * 5 + [R[0]])
        pts2, cnt2, _, _, stats2, _ = cs.TriangulateTracks(datas, K, Rs2, ts2, offsets, members, numTrials=64,
                                                           maxError=1.0, minTriAngle=0.5, seed=1)
        assert (cnt2[cnt > 0] > 0).all() and stats2[5] >= stats[5]
    finally:
        for d in datas:
            cs.FreeSiftData(d)
