"""GPU checks of batched verification (cs_verify_pairs_batch, cs_verify_essential_batch): every job of a mixed batch
equals the single call on that job bit for bit (model, count, inliers, statistics), a few jobs agree with the float64
restatements, several waves issue 8 launches each, jobs do not interact, batch and single calls interleave with the
matchers, and the chain batch extraction -> ratio matching on all pairs -> one batch verification equals the single
calls."""
import copy
import ctypes
import itertools

import numpy as np
import pytest

import essential_oracle as eo
import verify_oracle as vo
from cudasift_b200.synth import synth_descriptors, synth_image
from test_essential_cpu import K1, K2
from test_essential_gpu import planted as planted_e
from test_verify_gpu import planted

pytestmark = pytest.mark.gpu
SIZES = (0, 3, 4, 6, 7, 8, 100, 1000, 5000, 20000)
THRESH = 2.0


def _records(cs, xy):
    r = np.zeros(len(xy), cs.SIFT_DTYPE)
    r["xpos"], r["ypos"] = xy[:, 0], xy[:, 1]
    return r


class Pool:
    """Device buffers of a test: record sets, pair lists and inlier buffers (filled with -7)."""

    def __init__(self, cs):
        self.cs, self.bufs = cs, []

    def put(self, arr):
        arr = np.ascontiguousarray(arr)
        b = self.cs.DeviceBuffer(max(arr.nbytes, 576))
        if arr.nbytes:
            b.upload(arr)
        self.bufs.append(b)
        return b.ptr

    def records(self, xy):
        return self.put(_records(self.cs, xy)), len(xy)

    def pairs(self, p):
        return self.put(np.asarray(p, np.int32).reshape(-1, 2)), len(p)

    def out(self, n):
        return self.put(np.full(2 * max(n, 1), -7, np.int32))

    def free(self):
        for b in self.bufs:
            b.free()


class Job:
    """One job: device records and pairs, a seed, maxInliers (None: numPairs; 0: NULL inliers) and its own inlier
    buffers for the batch and for the single call."""

    def __init__(self, pool, s1, s2, pairs, seed, maxInliers=None, K=(K1, K2)):
        self.s1, self.s2 = s1, s2
        self.pairs, self.np = pool.pairs(pairs) if len(pairs) else (None, 0)
        self.seed = seed
        self.mi = self.np if maxInliers is None else maxInliers
        self.inl_b = pool.out(self.mi) if self.mi else None
        self.inl_s = pool.out(self.mi) if self.mi else None
        self.pool, self.K = pool, K

    def c(self, batch=True):
        return self.cs_job(self.inl_b if batch else self.inl_s)

    def cs_job(self, inl):
        return self.pool.cs.VerifyJob(self.s1[0], self.s1[1], self.s2[0], self.s2[1], self.pairs, self.np, self.seed,
                                      inl, self.mi)

    def inliers(self, count, batch=True):
        b = self.inl_b if batch else self.inl_s
        k = min(count, self.mi)
        if not b or not k:
            return np.zeros((0, 2), np.int32)
        out = np.empty((k, 2), np.int32)
        self.pool.cs.lib().cs_memcpy_d2h(out.ctypes.data, b, out.nbytes)
        return out


def _share(pool, job, seed):
    """A job on another job's device records and pair list, with its own seed and inlier buffers."""
    j = copy.copy(job)
    j.seed = seed
    j.inl_b, j.inl_s = pool.out(j.mi), pool.out(j.mi)
    return j


def _table(cs, jobs):
    t = (cs.VerifyJob * max(len(jobs), 1))()
    for k, j in enumerate(jobs):
        t[k] = j.c(True)
    return t


def batch_pairs(cs, jobs, model, loops):
    J = len(jobs)
    t = _table(cs, jobs)
    models, counts, stats = np.full((J, 9), 7.0), np.full(J, -1, np.int32), np.full((J, 8), 7, np.int64)
    ms = ctypes.c_double(0.0)
    r = cs.lib().cs_verify_pairs_batch(ctypes.addressof(t), J, model, loops, THRESH, models.ctypes.data,
                                       counts.ctypes.data, stats.ctypes.data, ctypes.byref(ms))
    assert r == 0, cs.lib().cs_last_error()
    return models, counts, stats, [j.inliers(int(counts[k])) for k, j in enumerate(jobs)], ms.value


def single_pairs(cs, j, model, loops):
    out = np.zeros(9)
    k = cs.lib().cs_verify_pairs(j.s1[0], j.s1[1], j.s2[0], j.s2[1], j.pairs, j.np, model, loops, THRESH, j.seed,
                                 out.ctypes.data, j.inl_s, j.mi, None)
    assert k >= 0, cs.lib().cs_last_error()
    st = np.array(cs.verify_stats(), np.int64) if j.np else np.zeros(8, np.int64)
    return out, k, st, j.inliers(k, batch=False)


def batch_essential(cs, jobs, loops):
    J = len(jobs)
    t = _table(cs, jobs)
    k1 = np.ascontiguousarray([j.K[0].reshape(9) for j in jobs])
    k2 = np.ascontiguousarray([j.K[1].reshape(9) for j in jobs])
    E, R, tt = np.full((J, 9), 7.0), np.full((J, 9), 7.0), np.full((J, 3), 7.0)
    counts, stats = np.full(J, -1, np.int32), np.full((J, 10), 7, np.int64)
    r = cs.lib().cs_verify_essential_batch(ctypes.addressof(t), J, k1.ctypes.data, k2.ctypes.data, loops, THRESH,
                                           E.ctypes.data, R.ctypes.data, tt.ctypes.data, counts.ctypes.data,
                                           stats.ctypes.data, None)
    assert r == 0, cs.lib().cs_last_error()
    return (E, R, tt), counts, stats, [j.inliers(int(counts[k])) for k, j in enumerate(jobs)]


def single_essential(cs, j, loops):
    E, R, t = np.zeros(9), np.zeros(9), np.zeros(3)
    k1, k2 = np.ascontiguousarray(j.K[0]), np.ascontiguousarray(j.K[1])
    k = cs.lib().cs_verify_essential(j.s1[0], j.s1[1], j.s2[0], j.s2[1], j.pairs, j.np, k1.ctypes.data, k2.ctypes.data,
                                     loops, THRESH, j.seed, E.ctypes.data, R.ctypes.data, t.ctypes.data, j.inl_s, j.mi,
                                     None)
    assert k >= 0, cs.lib().cs_last_error()
    st = np.array(cs.essential_stats(), np.int64) if j.np else np.zeros(10, np.int64)
    return (E, R, t), k, st, j.inliers(k, batch=False)


def _mixed_jobs(cs, pool, model):
    """About 40 jobs: every size of SIZES on a big planted scene's records (shared by many jobs), other scenes, invalid
    pairs and non-finite coordinates, a job whose pairs are all invalid, a set paired with itself, per-job seeds,
    maxInliers below the count and maxInliers == 0 with NULL inliers."""
    planar = model == vo.HOMOGRAPHY
    x1, x2, pairs, _, _, _ = planted(20000, 101, planar)
    A, B = pool.records(x1), pool.records(x2)
    jobs = []
    rng = np.random.default_rng(5)
    for k, n in enumerate(SIZES):                                 # prefixes and random subsets of one pair list
        jobs.append(Job(pool, A, B, pairs[:n], 1000 + k))
        sub = np.sort(rng.choice(20000, n, replace=False))
        jobs.append(Job(pool, A, B, pairs[sub], 2000 + k))
    for k, n in enumerate((500, 3000, 9000)):                     # other scenes
        y1, y2, p, _, _, _ = planted(n, 200 + k, planar)
        jobs.append(Job(pool, pool.records(y1), pool.records(y2), p, 7 * k))
    bad = pairs[:2000].copy()                                     # invalid indices, NaN and inf coordinates
    bad[3] = [-1, 0]; bad[10] = [0, 20000]; bad[20] = [20000, 0]; bad[30] = [2 ** 31 - 1, 5]
    xn = x1.copy()
    xn[pairs[40, 0], 0] = np.nan
    xn[pairs[41, 0], 1] = np.inf
    An = pool.records(xn)
    jobs.append(Job(pool, An, B, bad, 17))
    jobs.append(Job(pool, A, B, np.full((500, 2), -1), 18))        # every pair invalid
    jobs.append(Job(pool, A, A, np.column_stack([np.arange(800)] * 2), 19))      # a set paired with itself
    jobs.append(Job(pool, A, A, pairs[:1500], 20))                # the same set on both sides, a real pair list
    jobs.append(Job(pool, A, B, pairs[:3000], 21, maxInliers=10))  # maxInliers below the count
    jobs.append(Job(pool, A, B, pairs[:3000], 22, maxInliers=0))   # NULL inliers
    jobs.append(Job(pool, A, B, pairs[:3000], 21))                # same pairs as two jobs above, same seed
    jobs.append(_share(pool, jobs[-1], 24))                       # the same device pair list as the job before
    jobs.append(Job(pool, B, A, pairs[:1000, ::-1], 23))           # the views swapped
    for k in range(8):                                            # disjoint slices, per-job seeds
        jobs.append(Job(pool, A, B, pairs[2500 * k:2500 * k + 600 + 300 * k], 3000 + k))
    return jobs, (x1, x2, pairs)


def _check_pairs_equal(cs, jobs, got, model, loops):
    models, counts, stats, inl, _ = got
    for p, j in enumerate(jobs):
        m, k, st, il = single_pairs(cs, j, model, loops)
        assert models[p].tobytes() == m.tobytes(), p
        assert counts[p] == k and np.array_equal(stats[p], st), (p, counts[p], k, stats[p], st)
        assert inl[p].shape == (min(k, j.mi), 2) and np.array_equal(inl[p], il), p
        if not j.np:
            assert not models[p].any() and counts[p] == 0 and not stats[p].any()


@pytest.mark.parametrize("model", [vo.FUNDAMENTAL, vo.HOMOGRAPHY])
def test_mixed_batch_equals_single_calls(cs, model):
    pool = Pool(cs)
    try:
        jobs, (x1, x2, pairs) = _mixed_jobs(cs, pool, model)
        assert len(jobs) == 40
        n0 = cs.lib().cs_launch_count()
        got = batch_pairs(cs, jobs, model, 1024)
        assert cs.lib().cs_launch_count() - n0 == 8                # one wave
        assert got[4] > 0
        _check_pairs_equal(cs, jobs, got, model, 1024)
        models, counts, stats, inl, _ = got
        assert counts[SIZES.index(20000) * 2] > 0.5 * 20000
        bad = 2 * len(SIZES) + 3                                    # the job with invalid pairs and NaN coordinates
        assert stats[bad][1] == 6 and stats[bad][0] == 1994
        assert counts[bad + 1] == 0 and stats[bad + 1][0] == 0 and stats[bad + 1][1] == 500
        # a few jobs against the float64 restatement: the winner's count and the final inliers of the returned model
        for p in (12, 14, 16):                                     # prefixes of 100, 1000 and 5000 pairs
            j = jobs[p]
            sub = pairs[:j.np]
            q = np.column_stack([x1[sub[:, 0]], x2[sub[:, 1]]]).astype(np.float64)
            want, _, _ = vo.slot_models(q, model, 1024, j.seed)
            w = int((vo.residuals(want[stats[p][4]], model, q) < THRESH).sum())
            border = int((np.abs(vo.residuals(want[stats[p][4]], model, q) - THRESH) <= 1e-4 * THRESH).sum())
            assert abs(w - stats[p][5]) <= border, (p, w, stats[p][5])
            r = vo.residuals(models[p].reshape(3, 3), model, q)
            border = int((np.abs(r - THRESH) <= 1e-3 * THRESH).sum())
            assert abs(int((r < THRESH).sum()) - int(counts[p])) <= border, p
    finally:
        pool.free()


def test_permuted_and_repeated_batches(cs):
    pool = Pool(cs)
    try:
        jobs, _ = _mixed_jobs(cs, pool, vo.FUNDAMENTAL)
        a = batch_pairs(cs, jobs, vo.FUNDAMENTAL, 512)
        b = batch_pairs(cs, jobs, vo.FUNDAMENTAL, 512)
        perm = np.random.default_rng(3).permutation(len(jobs))
        c = batch_pairs(cs, [jobs[k] for k in perm], vo.FUNDAMENTAL, 512)
        for p in range(len(jobs)):
            assert a[0][p].tobytes() == b[0][p].tobytes() == c[0][np.nonzero(perm == p)[0][0]].tobytes(), p
        q = np.argsort(perm)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[1], c[1][q]) and np.array_equal(a[2], c[2][q])
        for p in range(len(jobs)):
            assert np.array_equal(a[3][p], b[3][p]) and np.array_equal(a[3][p], c[3][q[p]]), p
    finally:
        pool.free()


def _essential_jobs(cs, pool):
    jobs, scenes = [], []
    for k, (n, motion) in enumerate([(0, "sideways"), (4, "sideways"), (5, "sideways"), (6, "forward"),
                                     (8, "sideways"), (100, "forward"), (1000, "sideways"), (5000, "forward"),
                                     (20000, "sideways")]):
        if n == 0:
            jobs.append(Job(pool, pool.records(np.zeros((3, 2))), pool.records(np.zeros((3, 2))), [], 0))
            scenes.append(None)
            continue
        x1, x2, pairs, _, _, _, _ = planted_e(max(n, 50), 300 + k, motion)
        pairs = pairs[:n]
        A, B = pool.records(x1), pool.records(x2)
        jobs.append(Job(pool, A, B, pairs, 40 + k))
        jobs.append(Job(pool, A, B, pairs, 90 + k, maxInliers=7))
        scenes.append((x1, x2, pairs))
        scenes.append(None)
    x1, x2, pairs, _, _, _, _ = planted_e(3000, 77)
    A, B = pool.records(x1), pool.records(x2)
    Kskew = K2.copy()
    Kskew[0, 1] = 5.0
    for k in range(18):                                            # shared records, per-job K (one with skew), seeds
        jobs.append(Job(pool, A, B, pairs[150 * k:150 * k + 600], 500 + k, K=(K1, Kskew if k == 3 else K2)))
    jobs.append(Job(pool, A, B, pairs[:2000], 9, maxInliers=0))
    bad = pairs[:2000].copy()
    bad[5] = [-3, 0]; bad[9] = [0, 3000]
    xn = x1.copy()
    xn[pairs[50, 0], 0] = np.nan
    jobs.append(Job(pool, pool.records(xn), B, bad, 10))
    jobs.append(Job(pool, A, B, np.full((100, 2), 3000), 11))     # every pair invalid
    jobs.append(Job(pool, A, A, np.column_stack([np.arange(600)] * 2), 12))      # a set paired with itself
    return jobs, scenes


def _check_essential_equal(cs, jobs, got, loops):
    (E, R, t), counts, stats, inl = got
    for p, j in enumerate(jobs):
        (e, r, tt), k, st, il = single_essential(cs, j, loops)
        assert E[p].tobytes() == e.tobytes() and R[p].tobytes() == r.tobytes() and t[p].tobytes() == tt.tobytes(), p
        assert counts[p] == k and np.array_equal(stats[p], st), (p, counts[p], k, stats[p], st)
        assert np.array_equal(inl[p], il), p


def test_essential_batch_equals_single_calls(cs):
    pool = Pool(cs)
    try:
        jobs, scenes = _essential_jobs(cs, pool)
        assert len(jobs) == 39
        n0 = cs.lib().cs_launch_count()
        got = batch_essential(cs, jobs, 1024)
        assert cs.lib().cs_launch_count() - n0 == 8
        _check_essential_equal(cs, jobs, got, 1024)
        (E, R, t), counts, stats, _ = got
        assert counts[-4] > 0 and stats[-3][1] == 3 and counts[-2] == 0 and stats[-2][1] == 100
        # the float64 restatement on a few jobs: the winning slot's count and the final inliers of E
        for p in (11, 13, 15):
            x1, x2, pairs = scenes[p]
            q = np.column_stack([x1[pairs[:, 0]], x2[pairs[:, 1]]]).astype(np.float64)
            want, _, _ = eo.slot_models(q, K1, K2, 1024, jobs[p].seed)
            r = eo.residuals(want[stats[p][4]], K1, K2, q)
            assert abs(int((r < THRESH).sum()) - stats[p][5]) <= int((np.abs(r - THRESH) <= 1e-4 * THRESH).sum()), p
            r = eo.residuals(E[p].reshape(3, 3), K1, K2, q)
            assert abs(int((r < THRESH).sum()) - int(counts[p])) <= int((np.abs(r - THRESH) <= 1e-3 * THRESH).sum()), p
            assert abs(np.linalg.det(R[p].reshape(3, 3)) - 1) < 1e-9 and abs(np.linalg.norm(t[p]) - 1) < 1e-9
    finally:
        pool.free()


def test_several_waves(cs):
    """numLoops = 65536 for E: 10 x 65536 x 76 B per job, so 5 jobs per 256 MiB wave and 3 waves for 12 jobs."""
    pool = Pool(cs)
    try:
        x1, x2, pairs, _, _, _, _ = planted_e(4000, 88)
        A, B = pool.records(x1), pool.records(x2)
        jobs = [Job(pool, A, B, pairs[250 * k:250 * k + 300 + 100 * k], 60 + k) for k in range(12)]
        jobs.insert(4, Job(pool, A, B, [], 0))                    # an empty job launches nothing
        per = (256 << 20) // (10 * 65536 * 76)
        waves = -(-12 // per)
        assert (per, waves) == (5, 3)
        n0 = cs.lib().cs_launch_count()
        got = batch_essential(cs, jobs, 65536)
        assert cs.lib().cs_launch_count() - n0 == 8 * waves
        _check_essential_equal(cs, jobs, got, 65536)
    finally:
        pool.free()


def test_interleaving_with_matchers(cs):
    """Batch and single calls alternate with cs_match_ratio and cs_match_guided on the same device context."""
    pool = Pool(cs)
    try:
        jobs, _ = _mixed_jobs(cs, pool, vo.FUNDAMENTAL)
        jobs = jobs[10:24]
        s1, s2 = synth_descriptors(700, 3), synth_descriptors(650, 4)
        a = batch_pairs(cs, jobs, vo.FUNDAMENTAL, 512)
        q0, _ = cs.match_ratio_host(s1, s2, mode=2)
        F = a[0][-1].reshape(3, 3)
        g0, _ = cs.match_guided_host(s1, s2, "fundamental", F, 50.0)
        one = single_pairs(cs, jobs[5], vo.FUNDAMENTAL, 512)
        for rnd in range(2):
            q, _ = cs.match_ratio_host(s1, s2, mode=2)
            b = batch_pairs(cs, jobs, vo.FUNDAMENTAL, 512)
            g, _ = cs.match_guided_host(s1, s2, "fundamental", F, 50.0)
            o = single_pairs(cs, jobs[5], vo.FUNDAMENTAL, 512)
            assert np.array_equal(q, q0) and np.array_equal(g, g0)
            assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
            assert all(np.array_equal(x, y) for x, y in zip(a[3], b[3]))
            assert o[0].tobytes() == one[0].tobytes() and o[1] == one[1] and np.array_equal(o[3], one[3])
        _check_pairs_equal(cs, jobs, a, vo.FUNDAMENTAL, 512)
    finally:
        pool.free()


def test_end_to_end_all_pairs(cs):
    """Batch extraction of 6 views (ranked, N = 1000), cs_match_ratio on all 15 pairs and one batch verification:
    the same as 15 single calls, through the Python wrappers."""
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
        jobs = []
        for k, (a, b) in enumerate(itertools.combinations(range(6), 2)):
            pairs, _ = cs.MatchSiftDataRatio(datas[a], datas[b])
            jobs.append((datas[a], datas[b], pairs, k))
        assert sum(len(j[2]) > 100 for j in jobs) >= 10
        for model in ("homography", "fundamental"):
            M, inl, st, ms = cs.VerifyPairsBatch(jobs, model, 1024, THRESH)
            assert ms > 0
            for p, (d1, d2, pairs, seed) in enumerate(jobs):
                m, il, _ = cs.VerifyPairs(d1, d2, pairs, model, 1024, THRESH, seed)
                assert M[p].tobytes() == m.tobytes() and np.array_equal(inl[p], il), (model, p)
                assert list(st[p]) == (cs.verify_stats() if len(pairs) else [0] * 8), (model, p)
        K = np.array([[800.0, 0, 480], [0, 800.0, 270], [0, 0, 1]])
        E, R, t, inl, st, _ = cs.VerifyEssentialBatch(jobs, K, K, 1024, THRESH)
        for p, (d1, d2, pairs, seed) in enumerate(jobs):
            e, r, tt, il, _ = cs.VerifyEssential(d1, d2, pairs, K, K, 1024, THRESH, seed)
            assert E[p].tobytes() == e.tobytes() and R[p].tobytes() == r.tobytes() and t[p].tobytes() == tt.tobytes()
            assert np.array_equal(inl[p], il), p
    finally:
        for d in datas:
            cs.FreeSiftData(d)
