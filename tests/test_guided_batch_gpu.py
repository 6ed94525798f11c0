"""GPU checks of batched guided matching (cs_match_guided_batch): every job against its own cs_match_guided call (count,
pair bytes, a sentinel past maxPairs, guided_stats()) on mixed F and H jobs, jagged sizes, empty and 1-row sets, shared
and self-paired sets, rows that scan every candidate and non-finite positions; truncation, permutation and repetition;
several waves with the header's launch count; interleaving with single guided, ratio and verify calls; a few jobs
against the CPU statement; and the collection chain (batched extraction, ratio batch, verify batch, guided batch) on
six shifted views against the per-pair path."""
import ctypes
import itertools

import numpy as np
import pytest

import guided_oracle as go
import knn_oracle as ko
from cudasift_b200.synth import synth_descriptors, synth_image
from test_guided_gpu import planted
from test_match_batch_gpu import SENTINEL, Sets

pytestmark = pytest.mark.gpu
H, F = go.H, go.F
NAMES = {H: "homography", F: "fundamental"}


def _batch(cs, sets, jobs, thresh, cross, ratio=0.8, dist=0.7):
    """jobs: (a, b, maxPairs, model, M).  Returns (counts, stats, pair areas incl. one sentinel entry past maxPairs)."""
    J = len(jobs)
    room = [j[2] + 1 for j in jobs]
    off = np.concatenate([[0], np.cumsum(room)]).astype(int)
    buf = cs.DeviceBuffer(max(int(off[-1]), 1) * 8)
    try:
        buf.upload(np.full(2 * int(off[-1]), SENTINEL, np.int32))
        st = (cs.MatchSet * max(len(sets), 1))(*[cs.MatchSet(p, n) for p, n in sets])
        jt = (cs.MatchJob * max(J, 1))(*[cs.MatchJob(a, b, buf.ptr + 8 * int(off[q]) if m else None, m)
                                         for q, (a, b, m, _, _) in enumerate(jobs)])
        models = np.array([j[3] for j in jobs] or [F], np.int32)
        Ms = np.ascontiguousarray(np.array([np.asarray(j[4], np.float64).reshape(9) for j in jobs] or [np.eye(3).ravel()]))
        counts, stats = np.full(J, -1, np.int32), np.full((J, 4), 7, np.uint64)
        ms = ctypes.c_double(0.0)
        r = cs.lib().cs_match_guided_batch(st, len(sets), jt, J, models.ctypes.data, Ms.ctypes.data, thresh, ratio, dist,
                                           cross, counts.ctypes.data, stats.ctypes.data, ctypes.byref(ms))
        assert r == 0, cs.lib().cs_last_error().decode()
        flat = buf.download(np.int32, 2 * int(off[-1])).reshape(-1, 2)
    finally:
        buf.free()
    return counts, stats, [flat[off[q]:off[q + 1]] for q in range(J)]


def _single(cs, s1, s2, model, M, thresh, cross, dp, ratio=0.8, dist=0.7):
    (p1, n1), (p2, n2) = s1, s2
    m = np.ascontiguousarray(np.asarray(M, np.float64).reshape(9))
    k = cs.lib().cs_match_guided(p1, n1, p2, n2, model, m.ctypes.data, thresh, ratio, dist, cross, dp.ptr, max(n1, 1),
                                 None)
    assert k >= 0, cs.lib().cs_last_error().decode()
    pairs = dp.download(np.int32, 2 * k).reshape(-1, 2) if k else np.zeros((0, 2), np.int32)
    return k, pairs, cs.guided_stats() if n1 and n2 else [0, 0, 0, 0]


def _check(cs, S, jobs, thresh, cross, got=None):
    """Every job of the batch against its single call: count, pairs, the sentinel past maxPairs and the statistics."""
    counts, stats, areas = got if got is not None else _batch(cs, S.sets, jobs, thresh, cross)
    dp = cs.DeviceBuffer(max([n for _, n in S.sets] + [1]) * 8)
    try:
        for q, (a, b, m, model, M) in enumerate(jobs):
            k, pairs, st = _single(cs, S.sets[a], S.sets[b], model, M, thresh, cross, dp)
            w = min(k, m)
            assert counts[q] == k, (q, counts[q], k)
            assert areas[q][:w].tobytes() == pairs[:w].tobytes(), q
            assert (areas[q][w] == SENTINEL).all(), q
            assert [int(x) for x in stats[q]] == [int(x) for x in st], (q, stats[q], st)
    finally:
        dp.free()
    return counts, stats, areas


def _mixed():
    """Record sets and (a, b, maxPairs, model, M) jobs: planted F and H views of jagged sizes, an empty and a 1-row set,
    shared sets, a set against itself, a view with positions beyond 1e12 px (its rows scan every candidate), one with
    non-finite positions, and an H whose |pw| < 1e-12 everywhere."""
    f1, f2, Fm = planted(1000, 1200, False, 11)
    h1, h2, Hm = planted(2000, 1500, True, 12)
    g1, g2, Fg = planted(300, 3100, False, 13)
    far = f1.copy()
    far["xpos"][3], far["ypos"][8] = 2e12, -3e12
    bad = f2.copy()
    bad["xpos"][::7] = np.nan
    bad["ypos"][1::7] = np.inf
    one = h1[:1].copy()
    empty = f1[:0]
    arrays = [f1, f2, h1, h2, g1, g2, far, bad, one, empty]
    tiny = np.array([[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1e-13]])
    jobs = [(0, 1, 1000, F, Fm), (2, 3, 2000, H, Hm), (4, 5, 300, F, Fg), (1, 0, 1200, F, Fm.T), (9, 0, 5, F, Fm),
            (0, 9, 5, H, Hm), (8, 3, 1, H, Hm), (3, 8, 1500, H, np.linalg.inv(Hm)), (2, 2, 2000, H, np.eye(3)),
            (6, 1, 1000, F, Fm), (0, 7, 1000, F, Fm), (2, 3, 2000, H, tiny), (0, 1, 1000, H, Hm), (5, 4, 3100, F, Fg.T),
            (0, 1, 1000, F, Fm)]
    return arrays, jobs


@pytest.mark.parametrize("cross", [0, 1])
def test_mixed_batch_equals_single_calls(cs, cross):
    arrays, jobs = _mixed()
    S = Sets(cs, arrays)
    try:
        counts, stats, _ = _check(cs, S, jobs, 4.0, cross)
        assert counts[0] > 300 and counts[1] > 300 and counts[4] == 0 and counts[5] == 0 and not stats[4].any()
        # the row beyond 1e12 px scans every candidate, and so does the reverse direction over that set; every row
        # under |pw| < 1e-12 does
        assert stats[9][0] >= 1200 + (1000 * 1200 if cross else 0) and stats[11][0] == 2000 * 1500 * (1 + cross)
        assert counts[8] > 1000                                                   # a set against itself under I
    finally:
        S.free()


def test_one_job_does_not_change_its_neighbours(cs):
    """A job whose rows scan every candidate and one with non-finite positions, inserted between two ordinary jobs:
    the neighbours' bytes and statistics are those of the batch without them."""
    arrays, jobs = _mixed()
    S = Sets(cs, arrays)
    try:
        plain = [jobs[0], jobs[1]]
        c0, s0, a0 = _batch(cs, S.sets, plain, 4.0, 1)
        c1, s1, a1 = _batch(cs, S.sets, [jobs[0], jobs[9], jobs[10], jobs[11], jobs[1]], 4.0, 1)
        for q, r in ((0, 0), (1, 4)):
            assert c0[q] == c1[r] and s0[q].tobytes() == s1[r].tobytes() and a0[q].tobytes() == a1[r].tobytes()
    finally:
        S.free()


def test_truncation(cs):
    arrays, jobs = _mixed()
    S = Sets(cs, arrays)
    try:
        short = [(a, b, m, model, M) for (a, b, _, model, M), m in zip(jobs[:4], (0, 1, 17, 250))]
        counts, _, _ = _check(cs, S, short, 4.0, 1)
        assert (counts[1:] > 17).all() and counts[3] > 250
    finally:
        S.free()


def test_permutation_and_repetition(cs):
    arrays, jobs = _mixed()
    S = Sets(cs, arrays)
    try:
        c0, s0, a0 = _batch(cs, S.sets, jobs, 4.0, 1)
        c1, s1, a1 = _batch(cs, S.sets, jobs, 4.0, 1)
        assert c0.tobytes() == c1.tobytes() and s0.tobytes() == s1.tobytes()
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a0, a1))
        perm = np.random.default_rng(3).permutation(len(jobs))
        c2, s2, a2 = _batch(cs, S.sets, [jobs[p] for p in perm], 4.0, 1)
        for q, p in enumerate(perm):
            assert c2[q] == c0[p] and s2[q].tobytes() == s0[p].tobytes() and a2[q].tobytes() == a0[p].tobytes()
    finally:
        S.free()


def _job_bytes(n1, n2, cross):
    """The header's per-job scratch."""
    al = lambda b: -(-b // 256) * 256
    m = n1 if cross else 1
    cap0, cap1 = 2 * n2 + 64, 2 * n1 + 64 if cross else 1
    pieces = [4 * cap0, 4 * cap1, 32 * (n1 + n2), 8 * (n1 + n2), 4 * (cap0 + 1), 4 * (cap0 + 1), 4 * (cap1 + 1),
              4 * (cap1 + 1), 16 * n2, 4 * n2, 16 * n2, 4 * n2, 16 * m, 4 * m, 16 * m, 4 * m, 8 * n1, 8 * n1,
              -(-n1 // 32) * 4, -(-n1 // 1024) * 4]
    if cross:
        pieces += [8 * n2, 8 * n2]
    return 256 + sum(al(p) for p in pieces)


def _waves(ns, jobs, cross):
    """The header's wave rule."""
    waves, total = 0, 0
    for a, b in jobs:
        if ns[a] == 0 or ns[b] == 0:
            continue
        cost = _job_bytes(ns[a], ns[b], cross)
        if waves == 0 or total + cost > 256 << 20:
            waves, total = waves + 1, 0
        total += cost
    return waves


def test_several_waves(cs):
    """45 cross-checked jobs of 30 000 x 30 000 rows over overlapping windows of one buffer, with an empty job among
    them: two waves of seven launches."""
    rng = np.random.default_rng(5)
    recs = synth_descriptors(40000, 78, sift_like=True)
    recs["xpos"], recs["ypos"] = rng.uniform(0, 1920, 40000), rng.uniform(0, 1080, 40000)
    windows = [(200 * k, 30000) for k in range(46)] + [(0, 0)]
    S = Sets(cs, [recs], windows)
    try:
        M = np.array([[1.0, 0, 0.5], [0, 1.0, -0.25], [0, 0, 1.0]])
        pairs = [(1 + k, 2 + k) for k in range(45)]
        pairs[7] = (47, 3)
        jobs = [(a, b, 30000, H, M) for a, b in pairs]
        ns = [n for _, n in S.sets]
        waves = _waves(ns, pairs, True)
        assert waves == 2
        L = cs.lib()
        before = L.cs_launch_count()
        got = _batch(cs, S.sets, jobs, 4.0, 1)
        assert L.cs_launch_count() - before == 7 * waves
        counts, stats, areas = got
        idx = [0, 1, 6, 7, 8, 36, 37, 38, 43, 44]                         # both ends of every wave, the empty job
        _check(cs, S, [jobs[i] for i in idx], 4.0, 1, got=(counts[idx], stats[idx], [areas[i] for i in idx]))
        assert counts[7] == 0 and (np.delete(counts, 7) > 0).all()
        before = L.cs_launch_count()
        _batch(cs, S.sets, jobs[:2] + [(1, 1, 0, F, np.eye(3)[[1, 2, 0]])], 4.0, 0)   # one wave, crossCheck off
        assert L.cs_launch_count() - before == 7
    finally:
        S.free()


def _sift_data(cs, ptr, n, keep):
    d = cs.SiftData()
    d._buf = type("B", (), {"ptr": ptr})()
    d.numPts, d.maxPts = n, n
    keep.append(d)
    return d


def test_interleaving_with_single_calls(cs):
    """Batches between single guided, ratio and verify calls: every single result and guided_stats() is unchanged."""
    arrays, jobs = _mixed()
    S = Sets(cs, arrays)
    keep = []
    try:
        (p0, n0), (p1, n1) = S.sets[0], S.sets[1]
        d0, d1 = _sift_data(cs, p0, n0, keep), _sift_data(cs, p1, n1, keep)
        Fm = jobs[0][4]

        def singles():
            g, _ = cs.MatchSiftDataGuided(d0, d1, "fundamental", Fm, 4.0)
            gs = tuple(cs.guided_stats())
            r, _ = cs.MatchSiftDataRatio(d0, d1)
            v = cs.VerifyPairs(d0, d1, r, "fundamental", 512, 4.0, 3)
            h, _ = cs.MatchSiftDataGuided(S_data[0], S_data[1], "homography", jobs[1][4], 4.0, crossCheck=False)
            return g.tobytes(), gs, r.tobytes(), v[0].tobytes(), v[1].tobytes(), h.tobytes(), tuple(cs.guided_stats())

        S_data = [_sift_data(cs, *S.sets[2], keep), _sift_data(cs, *S.sets[3], keep)]
        want = singles()
        first = _batch(cs, S.sets, jobs, 4.0, 1)
        for rnd in range(2):
            assert singles() == want, rnd
            got = _batch(cs, S.sets, jobs, 4.0, rnd)
            if rnd == 1:
                assert got[0].tobytes() == first[0].tobytes() and got[1].tobytes() == first[1].tobytes()
        assert tuple(cs.guided_stats()) == want[-1]                         # the batch leaves the single call's stats
        _check(cs, S, jobs, 4.0, 1, got=first)
    finally:
        S.free()


def test_jobs_against_cpu_statement(cs):
    """Three jobs' pairs against the CPU statement's lists (tests/guided_oracle.c) and the ratio rule (knn_oracle)."""
    views = [planted(800, 900, False, 21), planted(700, 1000, True, 22), planted(1200, 600, False, 23)]
    arrays, jobs = [], []
    for k, (s1, s2, M) in enumerate(views):
        arrays += [s1, s2]
        jobs.append((2 * k, 2 * k + 1, len(s1), F if k != 1 else H, M))
    S = Sets(cs, arrays)
    try:
        for cross in (0, 1):
            counts, _, areas = _batch(cs, S.sets, jobs, 4.0, cross)
            for q, (a, b, _, model, M) in enumerate(jobs):
                k1 = go.match_knn2_guided(arrays[a], arrays[b], model, M, 4.0)
                k2 = go.match_knn2_guided(arrays[a], arrays[b], model, M, 4.0, reverse=True)
                want, margin = ko.ratio_pairs(*k1, *k2, 0.8, 0.7, cross)
                assert margin > 1e-12
                assert counts[q] == len(want) and np.array_equal(areas[q][:counts[q]], want), (q, cross)
    finally:
        S.free()


def test_end_to_end_collection(cs):
    """Batch extraction of 6 shifted views (ranked, N = 1000), MatchSiftDataRatioBatch over the 15 pairs,
    VerifyPairsBatch, the jobs with at least 30 inliers kept, then MatchSiftDataGuidedBatch: equal to the per-pair path
    (MatchSiftDataRatio, VerifyPairs, MatchSiftDataGuided), for F and H."""
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
        for model in ("fundamental", "homography"):
            vjobs = [(datas[a], datas[b], ratio[k], k) for k, (a, b) in enumerate(pairs_idx)]
            Mv, inl, _, _ = cs.VerifyPairsBatch(vjobs, model, 1024, 4.0)
            keep = [k for k in range(len(pairs_idx)) if len(inl[k]) >= 30]
            assert len(keep) >= 10, model
            guided, stats, ms = cs.MatchSiftDataGuidedBatch(datas, [pairs_idx[k] for k in keep], model, Mv[keep], 4.0)
            assert ms > 0 and stats.shape == (len(keep), 4)
            for q, k in enumerate(keep):
                a, b = pairs_idx[k]
                r, _ = cs.MatchSiftDataRatio(datas[a], datas[b])
                m, _, _ = cs.VerifyPairs(datas[a], datas[b], r, model, 1024, 4.0, k)
                assert m.tobytes() == Mv[k].tobytes(), (model, k)
                g, _ = cs.MatchSiftDataGuided(datas[a], datas[b], model, m, 4.0)
                assert np.array_equal(guided[q], g) and list(stats[q]) == cs.guided_stats(), (model, k)
            assert sum(len(g) for g in guided) >= sum(len(ratio[k]) for k in keep) * 0.9
    finally:
        for d in datas:
            cs.FreeSiftData(d)
