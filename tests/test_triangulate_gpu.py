"""GPU checks of triangulation (cs_triangulate_tracks) against the float64 statement (tests/triangulate_oracle.py):
counts, inlier masks, statistics and point presence exactly, points to 1e-9 of the scene scale, errors to float
rounding, every decision kept away from its boundary (the oracle's Band).  Random scenes with skewed, unequal
intrinsics, arbitrary rolls, pixel noise and 10-30 % outliers over track lengths 2-64 at several numTrials (both
sides of the exhaustive/sampled switch); members behind a camera, tiny baselines, two members of one image, invalid
members, empty and malformed tracks; one 10^5-member track; 10^6 tracks (the oracle on a seeded subset, the rules'
properties on all); sentinels past every output and NULL member outputs; repeated calls and the launch count;
interleaving with tracks, guided and verify calls; and the six-view chain from batched extraction to points."""
import ctypes
import itertools

import numpy as np
import pytest

import triangulate_cases as tc
import triangulate_oracle as to
from cudasift_b200.records import SIFT_DTYPE
from cudasift_b200.synth import synth_image
from test_guided_batch_gpu import _batch as guided_batch
from test_guided_batch_gpu import _mixed, _sift_data
from test_match_batch_gpu import Sets
from test_tracks_gpu import check as tracks_check
from test_tracks_gpu import collection as tracks_collection

pytestmark = pytest.mark.gpu
LAUNCHES = 1
SENTINEL_F = np.float32(-12345.0)
SENTINEL_D = -54321.0
SENTINEL_I = -777


class Scene:
    """Record sets (positions only) and the tracks in device memory."""

    def __init__(self, cs, xy, Ks, Rs, ts, offsets, members):
        self.cs, self.bufs, sets = cs, [], []
        for p in xy:
            rec = np.zeros(len(p), SIFT_DTYPE)
            rec["xpos"], rec["ypos"] = p[:, 0], p[:, 1]
            b = cs.DeviceBuffer(max(rec.nbytes, 8))
            if len(p):
                b.upload(rec)
            self.bufs.append(b)
            sets.append(cs.MatchSet(b.ptr if len(p) else None, len(p)))
        self.sets = (cs.MatchSet * max(len(sets), 1))(*sets)
        self.S = len(xy)
        self.xy, self.Ks, self.Rs, self.ts = xy, np.ascontiguousarray(Ks), np.ascontiguousarray(Rs), np.ascontiguousarray(ts)
        self.offsets = np.asarray(offsets, np.int32)
        self.members = np.asarray(members, np.int32).reshape(-1, 2)
        self.T, self.M = len(self.offsets) - 1, len(self.members)
        self.d_off, self.d_mem = cs.DeviceBuffer(self.offsets.nbytes), cs.DeviceBuffer(max(self.members.nbytes, 8))
        self.d_off.upload(self.offsets)
        if self.M:
            self.d_mem.upload(self.members)
        self.bufs += [self.d_off, self.d_mem]

    def run(self, numTrials=256, maxError=4.0, minTriAngle=1.5, seed=0, memberOutputs=True):
        """One call with one sentinel entry past every output buffer (checked).  Returns (r, points, counts, errors,
        inlier, stats, ms); errors and inlier are None without member outputs."""
        cs, T, M = self.cs, self.T, self.M
        outs = [cs.DeviceBuffer(8 * (3 * T + 1)), cs.DeviceBuffer(4 * (T + 1)), cs.DeviceBuffer(4 * (M + 1)),
                cs.DeviceBuffer(M + 8)]
        try:
            outs[0].upload(np.full(3 * T + 1, SENTINEL_D))
            outs[1].upload(np.full(T + 1, SENTINEL_I, np.int32))
            outs[2].upload(np.full(M + 1, SENTINEL_F, np.float32))
            outs[3].upload(np.full(M + 8, 0xAB, np.uint8))
            stats, ms = np.full(8, 7, np.int64), ctypes.c_double(0.0)
            r = cs.lib().cs_triangulate_tracks(self.sets, self.S, self.Ks.ctypes.data, self.Rs.ctypes.data,
                                               self.ts.ctypes.data, self.d_off.ptr, T, self.d_mem.ptr, M,
                                               numTrials, maxError, minTriAngle, seed, outs[0].ptr, outs[1].ptr,
                                               outs[2].ptr if memberOutputs else None,
                                               outs[3].ptr if memberOutputs else None, stats.ctypes.data,
                                               ctypes.byref(ms))
            assert r >= 0, cs.lib().cs_last_error().decode()
            pts = outs[0].download(np.float64, 3 * T + 1)
            cnt = outs[1].download(np.int32, T + 1)
            err = outs[2].download(np.float32, M + 1)
            inl = outs[3].download(np.uint8, M + 8)
        finally:
            for b in outs:
                b.free()
        assert pts[-1] == SENTINEL_D and cnt[-1] == SENTINEL_I and err[-1] == SENTINEL_F and (inl[M:] == 0xAB).all()
        if not memberOutputs:
            assert (err == SENTINEL_F).all() and (inl == 0xAB).all()
            err, inl = None, None
        else:
            err, inl = err[:M], inl[:M]
        return r, pts[:-1].reshape(T, 3), cnt[:-1], err, inl, stats, ms.value

    def written(self):
        """The members of the well-formed tracks."""
        m = np.zeros(self.M, bool)
        for k in range(self.T):
            lo, hi = int(self.offsets[k]), int(self.offsets[k + 1])
            if 0 <= lo <= hi <= self.M:
                m[lo:hi] = True
        return m

    def free(self):
        for b in self.bufs:
            b.free()


def assert_band(band):
    assert band.e2 > 1e-6 and band.depth > 1e-9 and band.angle > 1e-9, vars(band)


def compare(scene, got, want, tracks=None):
    """The call's outputs for the given tracks (all by default) against the oracle's."""
    r, pts, cnt, err, inl, stats, ms = got
    tracks = np.arange(scene.T) if tracks is None else tracks
    tol = 1e-9 * tc.scale(scene.Ks, scene.Rs, scene.ts)
    assert cnt[tracks].tolist() == want["counts"].tolist()
    has = ~np.isnan(want["points"][:, 0])
    assert np.array_equal(~np.isnan(pts[tracks, 0]), has) and np.isnan(pts[tracks][~has]).all()
    assert np.abs(pts[tracks][has] - want["points"][has]).max(initial=0.0) <= tol
    if err is None:
        return
    m = np.zeros(scene.M, bool)
    for k in tracks:
        lo, hi = int(scene.offsets[k]), int(scene.offsets[k + 1])
        if 0 <= lo <= hi <= scene.M:
            m[lo:hi] = True
    assert np.array_equal(inl[m].astype(bool), want["inlier"][m])
    e, w = err[m], want["errors"][m]
    assert np.array_equal(np.isnan(e), np.isnan(w)) and np.array_equal(np.isinf(e), np.isinf(w))
    f = np.isfinite(w)
    assert np.allclose(e[f], w[f], rtol=2e-6, atol=1e-6)


def check(scene, numTrials=256, maxError=4.0, minTriAngle=1.5, seed=0):
    got = scene.run(numTrials, maxError, minTriAngle, seed)
    want = to.triangulate(scene.xy, scene.Ks, scene.Rs, scene.ts, scene.offsets, scene.members, numTrials, maxError,
                          minTriAngle, seed)
    assert_band(want["band"])
    assert got[0] == want["stats"][5] and got[5].tolist() == want["stats"].tolist(), (got[5], want["stats"])
    compare(scene, got, want)
    m = scene.written()
    assert (got[4][~m] == 0xAB).all() and (got[3][~m] == SENTINEL_F).all()    # nothing of a malformed track
    assert got[6] > 0
    return got, want


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("numTrials", [16, 64, 256])
def test_random_scenes(cs, seed, numTrials):
    scene = Scene(cs, *tc.scene(seed, repeat=0.2)[:6])
    try:
        got, want = check(scene, numTrials, seed=seed * 7 + 1)
        V = np.diff(scene.offsets)
        assert (V * (V - 1) // 2 > numTrials).any() and (V * (V - 1) // 2 <= numTrials).any()
        assert want["stats"][5] > 200 and want["stats"][6] > 0 and want["stats"][4] < want["stats"][3]
    finally:
        scene.free()


def special_scene(seed):
    """A random scene plus: a camera pair one centimetre apart (tracks over just those fail the angle test), a record
    with a NaN position, invalid members of each kind, two members of one image, empty tracks and malformed ones."""
    rng = np.random.default_rng(seed)
    xy, Ks, Rs, ts, offsets, members, _ = tc.scene(seed, numImages=40, numTracks=150, lengths=(2, 30), repeat=0.3)
    xy, offsets, members = [list(map(tuple, p)) for p in xy], list(offsets), [list(m) for m in members]
    S = len(xy)
    C = np.array([0.0, 0.0, -12.0])
    R = tc.look_at(C, np.zeros(3), 0.3)
    Ks = np.concatenate([Ks, [tc.intrinsics(rng)] * 2])
    Rs = np.concatenate([Rs, [R, R]])
    ts = np.concatenate([ts, [-R @ C, -R @ (C + [0.01, 0, 0])]])
    xy += [[], []]

    def add(track):
        members.extend(track)
        offsets.append(len(members))

    for _ in range(20):                                  # tiny baseline
        X = rng.uniform(-1, 1, 3)
        track = []
        for a in (S, S + 1):
            xy[a].append(tuple(tc.project(Ks[a], Rs[a], ts[a], X) + rng.normal(0, 0.3, 2)))
            track.append([a, len(xy[a]) - 1])
        add(track)
    xy[0].append((np.nan, 5.0))
    nanf = len(xy[0]) - 1
    for k in range(20):                                  # invalid members among valid ones
        lo, hi = int(offsets[k]), int(offsets[k + 1])
        add(members[lo:hi] + [[S + 2, 0], [-1, 0], [1, len(xy[1]) + k], [0, nanf]][k % 4:k % 4 + 2])
    add([])
    add([[0, nanf], [S + 5, 0]])                         # no valid member
    add(members[0:1])                                    # one valid member
    a_ = len(members)
    members.extend(members[:6])
    offsets += [-1, a_ + 6, a_ + 6]                      # two malformed tracks, then an empty one
    offsets.append(len(members) + 4)                     # the last one passes numMembers
    xy = [np.array(p, np.float32).reshape(-1, 2) for p in xy]
    return xy, Ks, Rs, ts, np.array(offsets, np.int32), np.array(members, np.int32)


def test_special_cases(cs):
    scene = Scene(cs, *special_scene(5))
    try:
        got, want = check(scene, 64)
        st = want["stats"]
        assert st[1] == 3 and st[2] >= 30 and st[0] == scene.T - 3
        assert np.isinf(want["errors"]).any()                            # members behind a camera
        assert np.isnan(want["points"][150:170]).all()                   # the tiny baselines
        got2 = scene.run(64, memberOutputs=False)
        assert got2[0] == got[0] and got2[5].tolist() == got[5].tolist()
        assert got2[1].tobytes() == got[1].tobytes() and got2[2].tobytes() == got[2].tobytes()
    finally:
        scene.free()


def test_one_long_track(cs):
    """10^5 members of one point over 200 images (many images twice or more), 20 % outliers: the sampled path."""
    rng = np.random.default_rng(9)
    Ks, Rs, ts = tc.cameras(rng, 200)
    X = np.array([0.3, -0.2, 0.4])
    n = 100000
    a = rng.integers(0, 200, n)
    px = np.array([tc.project(Ks[i], Rs[i], ts[i], X) for i in range(200)])[a] + rng.normal(0, 0.05, (n, 2))
    out = rng.random(n) < 0.2
    px[out] = rng.uniform([0, 0], [tc.W, tc.H], (int(out.sum()), 2))
    b = tc.Builder(200)
    b.track([(int(i), b.record(int(i), *p)) for i, p in zip(a, px)])
    xy, offsets, members = b.arrays()
    scene = Scene(cs, xy, Ks, Rs, ts, offsets, members)
    try:
        got, want = check(scene, 256, seed=3)
        assert want["stats"][3] == 256 and got[2][0] > 0.75 * n and np.abs(got[1][0] - X).max() < 1e-3
    finally:
        scene.free()


def test_million_tracks(cs):
    """10^6 tracks of 2-12 views over 1 000 cameras with 10 % outliers: the oracle on 1 500 seeded tracks, and on
    every track the rules' properties."""
    xy, Ks, Rs, ts, offsets, members, X = tc.collection(21, 10 ** 6)
    scene = Scene(cs, xy, Ks, Rs, ts, offsets, members)
    try:
        got = scene.run(256, 4.0, 1.5, 5)
        r, pts, cnt, err, inl, stats, ms = got
        sub = np.sort(np.random.default_rng(4).choice(scene.T, 1500, replace=False))
        want = to.triangulate(xy, Ks, Rs, ts, offsets, members, 256, 4.0, 1.5, 5, tracks=sub)
        assert_band(want["band"])
        compare(scene, got, want, sub)
        has = cnt > 0
        assert r == stats[5] == has.sum() and stats[7] == cnt.sum() and stats[0] == scene.T and stats[1] == 0
        assert (cnt[has] >= 2).all() and np.isnan(pts[~has]).all() and np.isfinite(pts[has]).all()
        per = np.add.reduceat(inl.astype(np.int64), offsets[:-1])
        assert np.array_equal(per, cnt)
        assert (err[inl == 1] <= 4.0).all() and np.isnan(err[np.repeat(~has, np.diff(offsets))]).all()
        assert r > 0.9 * scene.T
    finally:
        scene.free()


def test_repeated_calls_and_launch_count(cs):
    scene = Scene(cs, *special_scene(6))
    try:
        lib = cs.lib()
        before = lib.cs_launch_count()
        a = scene.run(32, seed=4)
        assert lib.cs_launch_count() - before == LAUNCHES
        b = scene.run(32, seed=4)
        for x, y in zip(a[1:6], b[1:6]):
            assert x.tobytes() == y.tobytes()
    finally:
        scene.free()


def test_interleaving_with_other_calls(cs):
    """Triangulation between tracks, guided batch, ratio and verify calls: both sides give the bytes they give alone."""
    arrays, jobs = _mixed()
    S = Sets(cs, arrays)
    keep = []
    sizes, lists = tracks_collection(6)
    scene = Scene(cs, *tc.scene(8, numTracks=200)[:6])
    try:
        (p0, n0), (p1, n1) = S.sets[0], S.sets[1]
        d0, d1 = _sift_data(cs, p0, n0, keep), _sift_data(cs, p1, n1, keep)

        def others():
            c, s, a = guided_batch(cs, S.sets, jobs, 4.0, 1)
            r, _ = cs.MatchSiftDataRatio(d0, d1)
            v = cs.VerifyPairs(d0, d1, r, "fundamental", 512, 4.0, 3)
            t = tracks_check(cs, sizes, lists)
            return (c.tobytes(), s.tobytes(), [x.tobytes() for x in a], r.tobytes(), v[0].tobytes(), v[1].tobytes(),
                    [x.tobytes() for x in t[1:]])

        want = others()
        first = scene.run(64)
        assert others() == want
        again = scene.run(64)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(first[1:6], again[1:6]))
        assert others() == want
    finally:
        scene.free()
        S.free()


def test_end_to_end_collection(cs):
    """The six shifted views of the tracks chain test: ranked batch extraction (N = 1000), the ratio batch, the verify
    batch (F), the guided batch, BuildTracks, then TriangulateTracks with cameras derived from the shifts.

    Model: a fronto-parallel plane Z = Z0 seen by cameras K = [f 0 cx; 0 f cy; 0 0 1], R = I, translated by C_i in X
    and Y only; a point of the plane moves by -f C_i / Z0 pixels, so view i, shifted by (dx, dy), is camera i with
    C_i = -(dx, dy, 0) Z0 / f.  A depth error dZ moves the disparity d = f B / Z by d dZ / Z0; with keypoint precision
    delta (0.1 px assumed for these integer shifts) and the smallest pairwise shift D among any three views, a track
    with at least 3 inliers has |Z - Z0| <= Z0 * 2 delta / D (two observations of error delta each).  It must hold for
    at least 75 % of those tracks.  The rest hold a feature matched within maxError (1 px) of the wrong position: a
    mismatch through the wrap-around band of np.roll, or a repeated texture."""
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
    try:
        pairs_idx = list(itertools.combinations(range(6), 2))
        ratio, _, _ = cs.MatchSiftDataRatioBatch(datas, pairs_idx)
        Mv, inl, _, _ = cs.VerifyPairsBatch([(datas[a], datas[b], ratio[k], k) for k, (a, b) in enumerate(pairs_idx)],
                                            "fundamental", 1024, 4.0)
        keep = [k for k in range(len(pairs_idx)) if len(inl[k]) >= 30]
        jobs = [pairs_idx[k] for k in keep]
        guided, _, _ = cs.MatchSiftDataGuidedBatch(datas, jobs, "fundamental", Mv[keep], 4.0)
        offsets, members, _, _, _ = cs.BuildTracks([d.numPts for d in datas], [(a, b, g) for (a, b), g in
                                                                                zip(jobs, guided)])
        f, Z0 = 200.0, 10.0
        K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]])
        ts = np.array([[dx * Z0 / f, dy * Z0 / f, 0.0] for dy, dx in shifts])        # t = -C
        pts, cnt, err, inlier, stats, ms = cs.TriangulateTracks(datas, K, np.eye(3), ts, offsets, members,
                                                                numTrials=64, maxError=1.0, minTriAngle=0.5, seed=1)
        assert ms > 0 and stats[0] == len(offsets) - 1 and stats[5] > 100
        # the same call against the oracle
        xy = [np.stack([d._buf.download(SIFT_DTYPE, d.numPts)["xpos"], d._buf.download(SIFT_DTYPE, d.numPts)["ypos"]],
                       1) for d in datas]
        want = to.triangulate(xy, [K] * 6, [np.eye(3)] * 6, ts, offsets, members, 64, 1.0, 0.5, 1)
        assert cnt.tolist() == want["counts"].tolist() and stats.tolist() == want["stats"].tolist()
        assert np.array_equal(inlier, want["inlier"])
        D = min(max(np.hypot(shifts[i][0] - shifts[j][0], shifts[i][1] - shifts[j][1])
                    for i, j in itertools.combinations(tri, 2)) for tri in itertools.combinations(range(6), 3))
        bound = Z0 * 2 * 0.1 / D
        three = cnt >= 3
        assert three.sum() > 100
        assert np.mean(np.abs(pts[three, 2] - Z0) <= bound) >= 0.75, (bound, np.percentile(np.abs(pts[three, 2] - Z0),
                                                                                          [50, 90, 99]))
    finally:
        for d in datas:
            cs.FreeSiftData(d)
