"""GPU checks of mutual matching (cs_match_mutual): each direction's five match fields are bit for bit those of a
one-directional MatchSiftData (the oracle, the reference digests, match_host), and the pairs are the numpy
cross-check of those two results, in increasing i."""
import ctypes
import functools
import hashlib

import numpy as np
import pytest

import oracle
import refcases
from cudasift_b200.synth import synth_descriptors, synth_image

pytestmark = pytest.mark.gpu
FIELDS = ("score", "ambiguity", "match", "match_xpos", "match_ypos")
ALL_EXACT = (1 << 64) - 1          # match_stats()[2] when the bad-input gate sent every row the exact way


def _eq(a, b, what):
    for f in FIELDS:
        assert a[f].tobytes() == b[f].tobytes(), "%s: field %s differs in %d rows" % (what, f, int((a[f] != b[f]).sum()))


def cross_check(a, b, minScore=0.0, maxAmbiguity=np.inf):
    """The pairs (i, j) of two finished directions: a[i].match == j, b[j].match == i, score and ambiguity strict."""
    i = np.arange(len(a))
    j = a["match"]
    ok = (j >= 0) & (j < len(b))
    ok &= b["match"][np.where(ok, j, 0)] == i
    ok &= (a["score"] > np.float32(minScore)) & (a["ambiguity"] < np.float32(maxAmbiguity))
    return np.stack([i[ok], j[ok]], axis=1).astype(np.int32)


def _pairs_ok(pairs, a, b, minScore=0.0, maxAmbiguity=np.inf, what=""):
    want = cross_check(a, b, minScore, maxAmbiguity)
    assert pairs.dtype == np.int32 and pairs.shape == want.shape, (what, pairs.shape, want.shape)
    assert np.array_equal(pairs, want), what
    if len(pairs):
        assert (np.diff(pairs[:, 0]) > 0).all() and len(np.unique(pairs[:, 1])) == len(pairs), what


def _tensor(n1, n2, mode):
    return (mode == 2 or (mode == 0 and n1 >= 256 and n2 >= 256)) and n1 >= 32 and n2 >= 32


@functools.lru_cache(maxsize=None)
def _oracle_case(n1, n2):
    s1, s2 = synth_descriptors(n1, 1), synth_descriptors(n2, 2)
    return s1, s2, oracle.match(s1, s2, threads=8), oracle.match(s2, s1, threads=8)


SIZES = [(1, 32), (31, 500), (100, 64), (257, 500), (1000, 1031), (1030, 1060), (2003, 1999), (2000, 2000)]


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("n1,n2", SIZES)
def test_mutual_bit_exact_vs_oracle(cs, n1, n2, mode):
    """Tails [32*floor(n/32), n) inside a tile the other direction reads (100, 500, 1000, 1060, 1999, 2003) and
    outside one (257, 1030, 1031), no tail (32, 64, 2000), and empty reverse directions (n1 < 32)."""
    s1, s2, w1, w2 = _oracle_case(n1, n2)
    g1, g2, pairs, ms = cs.match_mutual_host(s1, s2, mode=mode)
    what = "mode %d %dx%d" % (mode, n1, n2)
    _eq(g1, w1, what + " forward")
    _eq(g2, w2, what + " reverse")
    assert np.array_equal(g1["data"], s1["data"]) and np.array_equal(g2["data"], s2["data"])
    assert np.array_equal(g2["xpos"], s2["xpos"]) and np.array_equal(g1["match_error"], s1["match_error"])
    assert cs.match_stats()[3] == (2 if _tensor(n1, n2, mode) else 1)
    _pairs_ok(pairs, w1, w2, what=what)
    if len(pairs) >= 4:
        sc, am = w1["score"][pairs[:, 0]], w1["ambiguity"][pairs[:, 0]]
        for minScore, maxAmb in ((float(np.median(sc)), np.inf), (0.0, float(np.median(am))),
                                 (float(np.quantile(sc, 0.25)), float(np.quantile(am, 0.75))),
                                 (float(sc.max()), 1.0)):
            _, _, p, _ = cs.match_mutual_host(s1, s2, minScore, maxAmb, mode=mode)
            _pairs_ok(p, w1, w2, minScore, maxAmb, what="%s (%g, %g)" % (what, minScore, maxAmb))


def test_mutual_10000_equals_two_calls_and_reference(cs):
    g = refcases.reference()
    s1, s2 = refcases.match_sets(10000)
    a, _ = cs.match_host(s1, s2, mode=2)
    b, _ = cs.match_host(s2, s1, mode=2)
    g1, g2, pairs, _ = cs.match_mutual_host(s1, s2)
    _eq(g1, a, "forward")
    _eq(g2, b, "reverse")
    st = cs.match_stats()
    assert st[3] == 2 and st[2] < 0.01 * 20000, st
    for f in FIELDS:
        h = hashlib.sha256(np.ascontiguousarray(g1[f]).tobytes()).hexdigest()
        assert h == g["match10000_%s_sha" % f], f
    _pairs_ok(pairs, a, b, what="10000")
    assert len(pairs) > 0


def _quirk_sets():
    s2, s1 = synth_descriptors(640, 5), synth_descriptors(300, 6)
    s1["data"][0] = s2["data"][40]; s2["data"][7] = s2["data"][40]; s2["data"][33] = s2["data"][40]   # Q10 ties
    s1["data"][1] = s2["data"][639]
    s1["data"][2] *= -1                                   # Q11: no positive score
    s1["data"][3] = 0
    s2["data"][10] = 0
    s2["data"][11] *= -1
    a, b = synth_descriptors(500, 11, sift_like=True), synth_descriptors(800, 12, sift_like=True)
    b["data"][100:200] = b["data"][0:100] * np.float32(1.0) + np.float32(1e-7)     # near duplicates
    return [("quirks", s1, s2), ("tail", s1, s2[:630]), ("near duplicates", a, b)]


@pytest.mark.parametrize("mode", [1, 2])
def test_mutual_quirks(cs, mode):
    for what, s1, s2 in _quirk_sets():
        g1, g2, pairs, _ = cs.match_mutual_host(s1, s2, mode=mode)
        w1, w2 = oracle.match(s1, s2, threads=8), oracle.match(s2, s1, threads=8)
        _eq(g1, w1, what + " forward")
        _eq(g2, w2, what + " reverse")
        _pairs_ok(pairs, w1, w2, what=what)


def _triplicates():
    """Three identical candidates in one partition on either side: rows that like them cannot be certified."""
    s1, s2 = synth_descriptors(512, 21), synth_descriptors(640, 22)
    s2["data"][32] = s2["data"][0]
    s2["data"][64] = s2["data"][0]
    s1["data"][:64] = s2["data"][0] * 0.999 + s1["data"][:64] * 0.001
    s1["data"][132] = s1["data"][100]                     # partition 1 of set 1: rows 100, 132, 164
    s1["data"][164] = s1["data"][100]
    s2["data"][100:164] = s1["data"][100] * 0.999 + s2["data"][100:164] * 0.001
    return s1, s2


def test_mutual_fallback_in_both_directions(cs):
    """The per-row fallback runs in each direction as in a single-direction call; the statistics are their sum."""
    for what, s1, s2 in _quirk_sets()[:1] + [("triplicates", *_triplicates())]:
        a, _ = cs.match_host(s1, s2, mode=2)
        sf = cs.match_stats()
        b, _ = cs.match_host(s2, s1, mode=2)
        sr = cs.match_stats()
        g1, g2, pairs, _ = cs.match_mutual_host(s1, s2, mode=2)
        sm = cs.match_stats()
        _eq(g1, a, what + " forward")
        _eq(g2, b, what + " reverse")
        _pairs_ok(pairs, a, b, what=what)
        assert sm[3] == 2 and sm[:3] == [x + y for x, y in zip(sf[:3], sr[:3])], (what, sf, sr, sm)
        if what == "triplicates":
            assert 0 < sf[2] < len(s1) and 0 < sr[2] < len(s2), (sf, sr)
            assert (a["match"][:64] == 0).all() and (b["match"][100:164] == 100).all()


def test_mutual_out_of_range_in_one_set(cs):
    """A value the split-FP16 screening cannot bound, in one set only, sends both directions the exact way."""
    s1, s2 = synth_descriptors(600, 11), synth_descriptors(700, 12)
    s2["data"][5, 17] = 100.0
    g1, g2, pairs, _ = cs.match_mutual_host(s1, s2, mode=2)
    assert cs.match_stats()[2] == ALL_EXACT
    w1, w2 = oracle.match(s1, s2, threads=8), oracle.match(s2, s1, threads=8)
    _eq(g1, w1, "forward")
    _eq(g2, w2, "reverse")
    _pairs_ok(pairs, w1, w2)
    s2 = synth_descriptors(700, 12)
    s1["data"][590, 0] = np.nan                           # in set 1's tail: only its own direction reads it
    e1, e2, ep, _ = cs.match_mutual_host(s1, s2, mode=1)
    g1, g2, pairs, _ = cs.match_mutual_host(s1, s2, mode=2)
    assert cs.match_stats()[2] == ALL_EXACT
    _eq(g1, e1, "nan forward")
    _eq(g2, e2, "nan reverse")
    assert np.array_equal(pairs, ep)
    s1 = synth_descriptors(600, 11)                       # clean again: back on the tensor path
    g1, g2, pairs, _ = cs.match_mutual_host(s1, s2, mode=2)
    assert cs.match_stats()[2] < 0.01 * 1300
    _eq(g1, oracle.match(s1, s2, threads=8), "clean forward")


def test_mutual_ranked_extraction(cs):
    """Two synthetic views through a ranked extractor (N = 1000): non-empty pairs equal to the two-call result."""
    img = synth_image(1920, 1080, seed=7)
    views = [img, np.ascontiguousarray(np.roll(img, (7, 11), axis=(0, 1)))]
    sets = []
    ex = cs.Extractor(1920, 1080, 5, 1000, False, maxCandidates=32768)
    try:
        for v in views:
            ci = cs.CudaImage()
            ci.Allocate(1920, 1080, hostMem=v)
            ci.Download()
            ex.submit_device(ci.d_data, ci.pitch, 1.0, 3.0, 0.0)
            n = ex.wait()
            assert n == 1000
            sets.append(ex.device_points_at(0, n))
    finally:
        ex.close()
    p1, p2 = sets
    for mode in (0, 1, 2):
        a, _ = cs.match_host(p1, p2, mode=mode)
        b, _ = cs.match_host(p2, p1, mode=mode)
        g1, g2, pairs, _ = cs.match_mutual_host(p1, p2, 0.85, 0.95, mode=mode)
        _eq(g1, a, "mode %d forward" % mode)
        _eq(g2, b, "mode %d reverse" % mode)
        _pairs_ok(pairs, a, b, 0.85, 0.95, what="mode %d" % mode)
        assert len(pairs) > 50, len(pairs)


def _device_sets(cs, s1, s2):
    d1 = cs.InitSiftData(cs.SiftData(), max(len(s1), 1), True, True)
    d2 = cs.InitSiftData(cs.SiftData(), max(len(s2), 1), True, True)
    d1._buf.upload(s1); d2._buf.upload(s2)
    d1.numPts, d2.numPts = len(s1), len(s2)
    return d1, d2


def test_mutual_max_pairs_and_sentinel(cs):
    """maxPairs below the total: the total is returned, exactly maxPairs pairs are written, the rest is untouched."""
    s1, s2 = synth_descriptors(700, 31, sift_like=True), synth_descriptors(800, 32, sift_like=True)
    s2["data"][:300] = s1["data"][:300] * 0.98 + s2["data"][:300] * 0.02        # many mutual pairs
    w1, w2 = oracle.match(s1, s2, threads=8), oracle.match(s2, s1, threads=8)
    want = cross_check(w1, w2)
    assert len(want) > 200
    L = cs.lib()
    for mode in (1, 2):
        d1, d2 = _device_sets(cs, s1, s2)
        sentinel = np.full(2 * len(s1), -7, np.int32)
        dp = cs.DeviceBuffer(sentinel.nbytes)
        dp.upload(sentinel)
        ms = ctypes.c_double(0.0)
        room = len(want) // 2
        k = L.cs_match_mutual(d1.d_data, len(s1), d2.d_data, len(s2), 0.0, float("inf"), dp.ptr, room, mode, ctypes.byref(ms))
        assert k == len(want) and ms.value > 0
        got = dp.download(np.int32, 2 * len(s1)).reshape(-1, 2)
        assert np.array_equal(got[:room], want[:room]) and (got[room:] == -7).all()
        _eq(d1._buf.download(cs.SIFT_DTYPE, len(s1)), w1, "device set 1")
        _eq(d2._buf.download(cs.SIFT_DTYPE, len(s2)), w2, "device set 2")
        # maxPairs == 0 with no buffer: only the count
        assert L.cs_match_mutual(d1.d_data, len(s1), d2.d_data, len(s2), 0.0, float("inf"), None, 0, mode, None) == len(want)
        # the host entry point: same rule on a host buffer
        h1, h2 = s1.copy(), s2.copy()
        hp = np.full((len(s1), 2), -7, np.int32)
        k = L.cs_match_mutual_host(h1.ctypes.data, len(h1), h2.ctypes.data, len(h2), 0.0, float("inf"), hp.ctypes.data,
                                   room, mode, None)
        assert k == len(want) and np.array_equal(hp[:room], want[:room]) and (hp[room:] == -7).all()
        _eq(h1, w1, "host set 1")
        _eq(h2, w2, "host set 2")
        dp.free()
        cs.FreeSiftData(d1); cs.FreeSiftData(d2)


def test_mutual_empty_set_writes_nothing(cs):
    s1, s2 = synth_descriptors(300, 41), synth_descriptors(400, 42)
    d1, d2 = _device_sets(cs, s1, s2)
    dp = cs.DeviceBuffer(8 * 300)
    dp.upload(np.full(600, -7, np.int32))
    L = cs.lib()
    for n1, n2 in ((0, 400), (300, 0)):
        assert L.cs_match_mutual(d1.d_data, n1, d2.d_data, n2, 0.0, float("inf"), dp.ptr, 300, 2, None) == 0
    assert d1._buf.download(cs.SIFT_DTYPE, 300).tobytes() == s1.tobytes()
    assert d2._buf.download(cs.SIFT_DTYPE, 400).tobytes() == s2.tobytes()
    assert (dp.download(np.int32, 600) == -7).all()
    g1, g2, pairs, ms = cs.match_mutual_host(s1[:0], s2)
    assert len(pairs) == 0 and ms == 0.0 and g2.tobytes() == s2.tobytes()
    d1.numPts = 0
    pairs, ms = cs.MatchSiftDataMutual(d1, d2)
    assert pairs.shape == (0, 2) and ms == 0.0
    dp.free()


def test_mutual_alternates_with_single_direction(cs):
    """Mutual and plain calls share the matcher's alternating flag areas (a gated call among them): all stay exact."""
    cases = [(300, 400, 1), (512, 333, 2), (1000, 999, 3), (640, 640, 4)]
    for rnd in range(2):
        for n1, n2, seed in cases:
            s1, s2 = synth_descriptors(n1, seed), synth_descriptors(n2, seed + 50)
            if rnd == 1 and seed == 2:
                s1["data"][7, 7] = -9.0                    # gated: every row of both directions the exact way
            w1, w2 = oracle.match(s1, s2, threads=8), oracle.match(s2, s1, threads=8)
            d1, d2 = _device_sets(cs, s1, s2)
            pairs, ms = cs.MatchSiftDataMutual(d1, d2, mode=2)
            _eq(d1.h_data[:n1], w1, "mutual set 1 %d" % seed)
            _eq(d2.h_data[:n2], w2, "mutual set 2 %d" % seed)
            _pairs_ok(pairs, w1, w2, what="alternation %d" % seed)
            d1._buf.upload(s1)
            cs.MatchSiftData(d1, d2, mode=2)
            _eq(d1.h_data[:n1], w1, "single %d" % seed)
            assert cs.match_stats()[3] == 2
            cs.FreeSiftData(d1); cs.FreeSiftData(d2)
