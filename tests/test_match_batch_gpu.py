"""GPU checks of batched ratio matching (cs_match_ratio_batch): every job against its single cs_match_ratio call (count,
pair bytes, cs_match_stats in mode 2, pairs of mode 1), a few against the CPU statement (tests/knn_oracle.c), the
fallback and the bad-input gate per job, truncation, permutation and repetition, several waves with the header's
launch count, interleaving with the single calls, and the collection chain through the Python wrappers."""
import ctypes
import itertools

import numpy as np
import pytest

import knn_oracle
from cudasift_b200.synth import synth_descriptors, synth_image
from test_knn_gpu import RATIOS, _triplicates

pytestmark = pytest.mark.gpu
REC = 576
ALL_EXACT = (1 << 64) - 1
SENTINEL = -7


class Sets:
    """Record arrays in one device buffer; sets[s] is (pointer, n).  windows: extra (offset, n) views of the buffer."""

    def __init__(self, cs, arrays, windows=()):
        self.arrays = list(arrays)
        sizes = [len(a) for a in self.arrays]
        self.offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
        self.buf = cs.DeviceBuffer(max(int(self.offsets[-1]), 1) * REC)
        if self.offsets[-1]:
            self.buf.upload(np.concatenate([a for a in self.arrays if len(a)]))
        self.sets = [(self.buf.ptr + REC * int(o) if n else None, n) for o, n in zip(self.offsets[:-1], sizes)]
        self.recs = list(self.arrays)
        flat = np.concatenate([a for a in self.arrays if len(a)]) if self.offsets[-1] else None
        for o, n in windows:
            self.sets.append((self.buf.ptr + REC * o, n))
            self.recs.append(flat[o:o + n])

    def free(self):
        self.buf.free()


def _batch(cs, sets, jobs, ratio, dist, cross):
    """jobs: (a, b, maxPairs).  Returns (ret, counts, stats, pair areas incl. one sentinel entry past maxPairs)."""
    J = len(jobs)
    room = [m + 1 for _, _, m in jobs]
    off = np.concatenate([[0], np.cumsum(room)]).astype(int)
    buf = cs.DeviceBuffer(max(int(off[-1]), 1) * 8)
    try:
        buf.upload(np.full(2 * int(off[-1]), SENTINEL, np.int32))
        st = (cs.MatchSet * max(len(sets), 1))(*[cs.MatchSet(p, n) for p, n in sets])
        jt = (cs.MatchJob * max(J, 1))(*[cs.MatchJob(a, b, buf.ptr + 8 * int(off[q]) if m else None, m)
                                         for q, (a, b, m) in enumerate(jobs)])
        counts, stats = np.full(J, -1, np.int32), np.full((J, 4), 7, np.uint64)
        ms = ctypes.c_double(0.0)
        r = cs.lib().cs_match_ratio_batch(st, len(sets), jt, J, ratio, dist, cross, counts.ctypes.data,
                                          stats.ctypes.data, ctypes.byref(ms))
        assert r == 0, cs.lib().cs_last_error().decode()
        flat = buf.download(np.int32, 2 * int(off[-1])).reshape(-1, 2)
    finally:
        buf.free()
    return counts, stats, [flat[off[q]:off[q + 1]] for q in range(J)], ms.value


def _single(cs, s1, s2, ratio, dist, cross, mode, dp):
    (p1, n1), (p2, n2) = s1, s2
    k = cs.lib().cs_match_ratio(p1, n1, p2, n2, ratio, dist, cross, dp.ptr, max(n1, 1), mode, None)
    assert k >= 0, cs.lib().cs_last_error().decode()
    pairs = dp.download(np.int32, 2 * k).reshape(-1, 2) if k else np.zeros((0, 2), np.int32)
    return k, pairs, cs.match_stats() if n1 and n2 else [0, 0, 0, 0]


def _check(cs, S, jobs, ratio, dist, cross, got=None, both_modes=True):
    """Every job of the batch against its single calls (mode 2 stats, and the pairs of mode 1)."""
    counts, stats, areas, ms = got or _batch(cs, S.sets, jobs, ratio, dist, cross)
    dp = cs.DeviceBuffer(8 * max(max((n for _, n in S.sets), default=1), 1))
    try:
        for q, (a, b, m) in enumerate(jobs):
            what = "job %d (%d x %d) ratio %g dist %g cross %d" % (q, S.sets[a][1], S.sets[b][1], ratio, dist, cross)
            k, pairs, st = _single(cs, S.sets[a], S.sets[b], ratio, dist, cross, 2, dp)
            assert counts[q] == k, what
            w = min(k, m)
            assert areas[q][:w].tobytes() == pairs[:w].tobytes(), what
            assert (areas[q][w:] == SENTINEL).all(), what
            if S.sets[a][1] and S.sets[b][1]:
                assert list(stats[q][:3]) == list(st[:3]) and stats[q][3] == 2 and st[3] == 2, (what, stats[q], st)
            else:
                assert not stats[q].any(), what
            if both_modes:
                k1, pairs1, _ = _single(cs, S.sets[a], S.sets[b], ratio, dist, cross, 1, dp)
                assert k1 == k and pairs1.tobytes() == pairs.tobytes(), what
    finally:
        dp.free()
    return counts, stats, areas


def _oracle_pairs(s1, s2, ratio, dist, cross):
    k1, k2 = knn_oracle.match_knn2(s1, s2), knn_oracle.match_knn2(s2, s1)
    return knn_oracle.ratio_pairs(*k1, *k2, ratio, dist, cross)[0]


def _mixed_sets():
    sizes = [1, 5, 31, 100, 257, 1000, 1031, 2003]
    arrays = [synth_descriptors(n, 100 + k) for k, n in enumerate(sizes)]
    arrays += [synth_descriptors(1000, 200, sift_like=True), synth_descriptors(1031, 201, sift_like=True),
               synth_descriptors(257, 202, sift_like=True)]
    b = arrays[9]
    b["data"][:400] = arrays[8]["data"][:400] * 0.9 + b["data"][:400] * 0.1
    arrays.append(np.zeros(0, arrays[0].dtype))                    # set 11: empty
    return arrays


def _mixed_jobs():
    full = lambda a, b: 2100                                         # room for every count
    pairs = [(5, 6), (6, 5), (8, 9), (9, 8), (7, 7), (5, 6), (0, 1), (1, 0), (2, 3), (3, 4), (4, 4), (4, 7),
             (7, 2), (8, 10), (10, 8), (11, 5), (5, 11), (11, 11), (3, 9), (0, 7), (9, 9), (6, 7), (2, 2), (10, 6)]
    return [(a, b, full(a, b)) for a, b in pairs]


@pytest.mark.parametrize("cross", [0, 1])
def test_mixed_batch_equals_single_calls(cs, cross):
    """Sizes 1 .. 2003, random and sift_like, shared sets, a set against itself, a repeated job, an empty set and jobs
    below 256 rows, for the four ratio settings."""
    S = Sets(cs, _mixed_sets())
    try:
        jobs = _mixed_jobs()
        for ratio, dist in RATIOS:
            counts, _, areas = _check(cs, S, jobs, ratio, dist, cross)
            assert counts[0] == counts[5] and areas[0].tobytes() == areas[5].tobytes()
            for q in (0, 2, 13):                                    # against the CPU statement
                a, b, _ = jobs[q]
                want = _oracle_pairs(S.recs[a], S.recs[b], ratio, dist, cross)
                assert np.array_equal(areas[q][:counts[q]], want), (q, ratio, dist)
            if (ratio, dist) == RATIOS[0]:
                assert counts[2] > 100
    finally:
        S.free()


def test_fallback_in_many_jobs(cs):
    s1, s2 = _triplicates()
    S = Sets(cs, [s1, s2, synth_descriptors(700, 23)])
    try:
        jobs = [(0, 1, 700), (1, 0, 700), (2, 0, 700), (0, 1, 700), (1, 2, 700), (0, 0, 700)]
        for cross in (0, 1):
            counts, stats, areas = _check(cs, S, jobs, 0.8, 0.7, cross)
            for q in (0, 1, 3):
                assert 0 < stats[q][2] < 700, (q, stats[q])
            want = _oracle_pairs(s1, s2, 0.8, 0.7, cross)
            assert np.array_equal(areas[0][:counts[0]], want)
    finally:
        S.free()


def test_gate_per_job(cs):
    a, b = synth_descriptors(600, 11), synth_descriptors(700, 12)
    big, nan = b.copy(), a.copy()
    big["data"][5, 17] = 8.0
    nan["data"][590, 0] = np.nan
    S = Sets(cs, [a, b, big, nan])
    try:
        jobs = [(0, 1, 700), (0, 2, 700), (1, 0, 700), (3, 1, 700), (0, 0, 700), (1, 1, 700)]
        for cross in (0, 1):
            counts, stats, areas = _check(cs, S, jobs, 0.8, 0.7, cross)
            for q, gated in enumerate([False, True, False, True, False, False]):
                assert (stats[q][2] == ALL_EXACT) == gated, (q, stats[q])
            assert np.array_equal(areas[1][:counts[1]], _oracle_pairs(a, big, 0.8, 0.7, cross))
    finally:
        S.free()


def test_truncation(cs):
    S = Sets(cs, _mixed_sets())
    try:
        full = _batch(cs, S.sets, _mixed_jobs(), 0.8, 0.7, 1)[0]
        jobs = [(a, b, int(full[q]) // 2 if q % 3 else 0) for q, (a, b, _) in enumerate(_mixed_jobs())]
        counts, _, areas = _check(cs, S, jobs, 0.8, 0.7, 1, both_modes=False)
        assert np.array_equal(counts, full)
        assert sum(0 < m < c for (_, _, m), c in zip(jobs, counts)) >= 5
    finally:
        S.free()


def test_permutation_and_repetition(cs):
    S = Sets(cs, _mixed_sets())
    try:
        jobs = _mixed_jobs()
        c0, s0, a0, _ = _batch(cs, S.sets, jobs, 0.8, 0.7, 1)
        c1, s1, a1, _ = _batch(cs, S.sets, jobs, 0.8, 0.7, 1)
        assert c0.tobytes() == c1.tobytes() and s0.tobytes() == s1.tobytes()
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a0, a1))
        perm = np.random.default_rng(3).permutation(len(jobs))
        c2, s2, a2, _ = _batch(cs, S.sets, [jobs[i] for i in perm], 0.8, 0.7, 1)
        assert np.array_equal(c2, c0[perm]) and np.array_equal(s2, s0[perm])
        assert all(a2[q].tobytes() == a0[i].tobytes() for q, i in enumerate(perm))
    finally:
        S.free()


def _waves(ns, jobs, cross):
    """The header's wave rule."""
    set_b = lambda n: -(-n // 128) * 128 * 516
    dir_b = lambda n: -(-n // 128) * 128 * 160 + 24 * n
    waves, used, total = 0, set(), 0
    for a, b, _ in jobs:
        if ns[a] == 0 or ns[b] == 0:
            continue
        def cost(u):
            x = dir_b(ns[a]) + (dir_b(ns[b]) if cross else 0)
            return x + sum(set_b(ns[s]) for s in {a, b} if s not in u)
        if waves == 0 or total + cost(used) > 256 << 20:
            waves, used, total = waves + 1, set(), 0
        total += cost(used)
        used |= {a, b}
    return waves


def test_several_waves(cs):
    """40 cross-checked jobs of 10 000 x 10 000 rows, 80 distinct (overlapping) windows of one buffer: three waves of
    six launches."""
    recs = synth_descriptors(30000, 77)
    windows = [(250 * k, 10000) for k in range(80)]
    S = Sets(cs, [recs], windows)
    try:
        jobs = [(1 + 2 * k, 2 + 2 * k, 10000) for k in range(40)]
        ns = [n for _, n in S.sets]
        waves = _waves(ns, jobs, True)
        assert waves == 3
        L = cs.lib()
        before = L.cs_launch_count()
        got = _batch(cs, S.sets, jobs, 0.8, 0.7, 1)
        assert L.cs_launch_count() - before == 6 * waves
        counts, stats, _ = _check(cs, S, jobs, 0.8, 0.7, 1, got=got, both_modes=False)
        assert (counts > 0).all()
        before = L.cs_launch_count()
        _batch(cs, S.sets, jobs[:2] + [(1, 1, 0)], 0.8, 0.7, 0)        # one wave, crossCheck off: still six
        assert L.cs_launch_count() - before == 6
    finally:
        S.free()


def _sift_data(cs, ptr, n, keep):
    d = cs.SiftData()
    d._buf = type("B", (), {"ptr": ptr})()
    d.numPts, d.maxPts = n, n
    keep.append(d)
    return d


def test_interleaving_with_single_calls(cs):
    """Batch calls between MatchSiftData, mutual, knn, ratio, guided and verification calls (one of them gated): every
    single call's result and match_stats() is the one it gives without the batches."""
    cases = [(300, 400, 1), (512, 333, 2), (1000, 999, 3)]
    arrays = []
    for n1, n2, seed in cases:
        arrays += [synth_descriptors(n1, seed), synth_descriptors(n2, seed + 50)]
    gated = arrays[2].copy()
    gated["data"][7, 7] = -9.0
    arrays.append(gated)
    S = Sets(cs, _mixed_sets() + arrays)
    base = len(_mixed_sets())
    keep = []

    def singles():
        out = []
        for k in range(3):
            s1, s2 = S.recs[base + 2 * k], S.recs[base + 2 * k + 1]
            for a, b in ((s1, s2), (S.recs[-1], s2) if k == 1 else (s1, s2)):
                gi, gs, _ = cs.match_knn2(a, b, mode=2)
                out += [gi.tobytes(), gs.tobytes(), tuple(cs.match_stats())]
            m, _ = cs.match_host(s1, s2, mode=2)
            out += [m.tobytes(), tuple(cs.match_stats())]
            g1, g2, pm, _ = cs.match_mutual_host(s1, s2, mode=2)
            out += [g1.tobytes(), g2.tobytes(), pm.tobytes(), tuple(cs.match_stats())]
            pr, _ = cs.match_ratio_host(s1, s2, 0.8, 0.7, True, 2)
            out += [pr.tobytes(), tuple(cs.match_stats())]
            gi, gs, _ = cs.match_knn2_guided(s1, s2, 1, np.eye(3), 1e4)
            out += [gi.tobytes(), gs.tobytes(), tuple(cs.match_stats())]
            d1 = _sift_data(cs, *S.sets[base + 2 * k], keep)
            d2 = _sift_data(cs, *S.sets[base + 2 * k + 1], keep)
            M, inl, st, _ = cs.VerifyPairsBatch([(d1, d2, pr)], "fundamental", 256, 4.0)
            out += [M.tobytes(), st.tobytes(), tuple(cs.match_stats())]
        return out

    try:
        alone = singles()
        jobs = _mixed_jobs() + [(base + 4, base + 6, 1000), (base, base + 1, 400)]
        first = _batch(cs, S.sets, jobs, 0.8, 0.7, 1)
        mixed = singles()
        again = _batch(cs, S.sets, jobs, 0.8, 0.7, 1)
        assert mixed == alone
        assert first[0].tobytes() == again[0].tobytes() and first[1].tobytes() == again[1].tobytes()
        assert all(x.tobytes() == y.tobytes() for x, y in zip(first[2], again[2]))
        # a batch between every two single calls of one round
        cs_single = [lambda: cs.match_knn2(S.recs[base], S.recs[base + 1], mode=2),
                     lambda: cs.match_knn2(S.recs[-1], S.recs[base + 3], mode=2),
                     lambda: cs.match_host(S.recs[base + 4], S.recs[base + 5], mode=2),
                     lambda: cs.match_ratio_host(S.recs[base + 4], S.recs[base + 5], 0.8, 0.7, True, 2)]
        ref = []
        for f in cs_single:
            r = f()
            ref.append((r[0].tobytes(), tuple(cs.match_stats())))
        for f, (want, st) in zip(cs_single, ref):
            _batch(cs, S.sets, jobs[:6], 0.8, 0.7, 1)
            r = f()
            assert r[0].tobytes() == want and tuple(cs.match_stats()) == st
        _check(cs, S, jobs, 0.8, 0.7, 1, both_modes=False)
    finally:
        S.free()


def test_end_to_end_collection(cs):
    """Batch extraction of 6 views (ranked, N = 1000), MatchSiftDataRatioBatch over the 15 pairs, then
    VerifyPairsBatch: the same pairs, models and inliers as the per-pair path."""
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
        batch, stats, ms = cs.MatchSiftDataRatioBatch(datas, pairs_idx)
        assert ms > 0 and stats.shape == (15, 4) and (stats[:, 3] == 2).all()
        single = [cs.MatchSiftDataRatio(datas[a], datas[b])[0] for a, b in pairs_idx]
        assert all(np.array_equal(x, y) for x, y in zip(batch, single))
        assert sum(len(p) > 100 for p in batch) >= 10
        jobs_b = [(datas[a], datas[b], batch[k], k) for k, (a, b) in enumerate(pairs_idx)]
        jobs_s = [(datas[a], datas[b], single[k], k) for k, (a, b) in enumerate(pairs_idx)]
        Mb, ib, sb, _ = cs.VerifyPairsBatch(jobs_b, "fundamental", 1024, 4.0)
        Ms, is_, ss, _ = cs.VerifyPairsBatch(jobs_s, "fundamental", 1024, 4.0)
        assert Mb.tobytes() == Ms.tobytes() and sb.tobytes() == ss.tobytes()
        assert all(np.array_equal(x, y) for x, y in zip(ib, is_))
        for p, (d1, d2, pairs, seed) in enumerate(jobs_s):
            m, il, _ = cs.VerifyPairs(d1, d2, pairs, "fundamental", 1024, 4.0, seed)
            assert Mb[p].tobytes() == m.tobytes() and np.array_equal(ib[p], il), p
    finally:
        for d in datas:
            cs.FreeSiftData(d)
