"""GPU checks of two-nearest-neighbour matching: cs_match_knn2 bit for bit against the CPU statement
(tests/knn_oracle.c) on both paths, its tie to the unmodified reference's MatchSiftData digests, ties and degenerate
rows, the exact fallback and the bad-input gate, and the ratio-test pairs of cs_match_ratio against a float64 numpy
restatement built from the oracle's lists."""
import ctypes
import functools
import hashlib

import numpy as np
import pytest

import knn_oracle
import oracle
import refcases
from cudasift_b200.synth import synth_descriptors, synth_image

pytestmark = pytest.mark.gpu
ALL_EXACT = (1 << 64) - 1          # match_stats()[2] when the bad-input gate sent every row the exact way
FIELDS = ("score", "ambiguity", "match", "match_xpos", "match_ypos")


def _eq(gi, gs, wi, ws, what):
    assert np.array_equal(gi, wi), "%s: idx differs in %d rows" % (what, int((gi != wi).any(1).sum()))
    assert gs.tobytes() == ws.tobytes(), "%s: score differs in %d rows" % (what, int((gs != ws).any(1).sum()))


@functools.lru_cache(maxsize=None)
def _case(n1, n2):
    s1, s2 = synth_descriptors(n1, 1), synth_descriptors(n2, 2)
    return s1, s2, knn_oracle.match_knn2(s1, s2)


SIZES = [(1, 1), (5, 3), (31, 500), (100, 64), (257, 500), (1000, 1031), (2003, 1999), (2000, 2000)]


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("n1,n2", SIZES)
def test_knn2_bit_exact_vs_oracle(cs, n1, n2, mode):
    """n2 not a multiple of 4, 32 or 128 (1, 3, 500, 1031, 1999) and a multiple (64, 2000)."""
    s1, s2, (wi, ws) = _case(n1, n2)
    gi, gs, ms = cs.match_knn2(s1, s2, mode=mode)
    _eq(gi, gs, wi, ws, "mode %d %dx%d" % (mode, n1, n2))
    st = cs.match_stats()
    assert st[3] == mode and ms > 0
    if mode == 2 and n1 >= 100:
        assert st[2] < max(2, 0.01 * n1), st


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("n", [2000, 10000])
def test_knn2_ties_to_reference_digests(cs, n):
    """With n2 % 32 == 0 the reference's MatchSiftData visits every candidate, so score1 is its score and (without
    exact ties) j1 its match: the digests of the unmodified reference's output."""
    g = refcases.reference()
    s1, s2 = refcases.match_sets(n)
    s2 = s2[:32 * (n // 32)]
    for mode in (0, 2):
        idx, score, _ = cs.match_knn2(s1, s2, mode=mode)
        st = cs.match_stats()
        assert st[3] == 2 and st[2] < 0.01 * n, st
        j1 = idx[:, 0]
        ok = j1 >= 0
        xpos = np.where(ok, s2["xpos"][np.where(ok, j1, 0)], np.float32(0)).astype(np.float32)
        ypos = np.where(ok, s2["ypos"][np.where(ok, j1, 0)], np.float32(0)).astype(np.float32)
        assert _digest(score[:, 0].copy()) == g["match%d_score_sha" % n]
        assert _digest(j1.astype(np.int32)) == g["match%d_match_sha" % n]
        assert _digest(xpos) == g["match%d_match_xpos_sha" % n]
        assert _digest(ypos) == g["match%d_match_ypos_sha" % n]


def _degenerate_sets():
    s1, s2 = synth_descriptors(300, 5), synth_descriptors(640, 6)
    s2["data"][:, 127] = -np.abs(s2["data"][:, 127]) - np.float32(0.01)
    s2["data"][600, 127] = 0.5
    s2["data"][5] = s2["data"][4]; s1["data"][0] = s2["data"][4]          # inside one group
    s2["data"][64] = s2["data"][32]; s1["data"][1] = s2["data"][32]       # inside one partition (groups 8 and 16)
    s2["data"][33] = s2["data"][7]; s1["data"][2] = s2["data"][7]         # across partitions (groups 8 and 1)
    s1["data"][3] = 0                                                     # no positive score
    s1["data"][5] = 0
    s1["data"][5, 127] = 1.0                                              # one positive candidate: j = 600
    return s1, s2


@pytest.mark.parametrize("mode", [1, 2])
def test_knn2_ties_and_degenerate_rows(cs, mode):
    s1, s2 = _degenerate_sets()
    wi, ws = knn_oracle.match_knn2(s1, s2)
    gi, gs, _ = cs.match_knn2(s1, s2, mode=mode)
    _eq(gi, gs, wi, ws, "mode %d" % mode)
    for r, (a, b) in enumerate([(4, 5), (32, 64), (7, 33)]):
        assert tuple(gi[r]) == (a, b) and gs[r, 0] == gs[r, 1] > 0, (r, gi[r], gs[r])
    assert tuple(gi[3]) == (-1, -1) and tuple(gs[3]) == (0.0, 0.0)
    assert tuple(gi[5]) == (600, -1) and gs[5, 0] == np.float32(0.5) and gs[5, 1] == 0.0


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


def test_knn2_fallback_in_both_directions(cs):
    s1, s2 = _triplicates()
    for a, b in ((s1, s2), (s2, s1)):
        gi, gs, _ = cs.match_knn2(a, b, mode=2)
        st = cs.match_stats()
        assert st[3] == 2 and 0 < st[2] < len(a), st
        _eq(gi, gs, *knn_oracle.match_knn2(a, b), what="triplicates")
    gi, _, _ = cs.match_knn2(s1, s2, mode=2)
    assert (gi[:64, 0] == 0).all() and (gi[:64, 1] == 32).all()


def test_knn2_gate(cs):
    """A value the split-FP16 screening cannot bound, in one set, sends every row the exact way."""
    s1, s2 = synth_descriptors(600, 11), synth_descriptors(700, 12)
    for what, a, b in (("big", s1, s2.copy()), ("nan", s1.copy(), s2)):
        if what == "big":
            b["data"][5, 17] = 8.0
        else:
            a["data"][590, 0] = np.nan
        ei, es, _ = cs.match_knn2(a, b, mode=1)
        gi, gs, _ = cs.match_knn2(a, b, mode=2)
        assert cs.match_stats()[2] == ALL_EXACT, what
        _eq(gi, gs, ei, es, what + " vs mode 1")
        _eq(gi, gs, *knn_oracle.match_knn2(a, b), what=what + " vs oracle")
    gi, gs, _ = cs.match_knn2(s1, s2, mode=2)               # clean again: back on the tensor path
    assert cs.match_stats()[2] < 0.01 * 600
    _eq(gi, gs, *knn_oracle.match_knn2(s1, s2), what="clean")


def _device(cs, recs):
    d = cs.DeviceBuffer(max(recs.nbytes, 576))
    d.upload(recs)
    return d


RATIOS = [(0.8, 0.7), (0.6, 0.5), (0.9, 1.6), (1.0, 0.3)]


def _ratio_sets():
    a, b = synth_descriptors(700, 31, sift_like=True), synth_descriptors(800, 32, sift_like=True)
    b["data"][:300] = a["data"][:300] * 0.9 + b["data"][:300] * 0.1
    norm = np.linalg.norm(b["data"], axis=1, keepdims=True)
    b["data"] = (b["data"] / np.maximum(norm, 1e-6)).astype(np.float32)
    return a, b


@pytest.mark.parametrize("mode", [1, 2])
def test_ratio_pairs_vs_numpy(cs, mode):
    s1, s2 = _ratio_sets()
    k1, k2 = knn_oracle.match_knn2(s1, s2), knn_oracle.match_knn2(s2, s1)
    L = cs.lib()
    d1, d2 = _device(cs, s1), _device(cs, s2)
    n1, n2 = len(s1), len(s2)
    dp = cs.DeviceBuffer(8 * n1)
    try:
        for maxRatio, maxDistance in RATIOS:
            for cross in (0, 1):
                want, margin = knn_oracle.ratio_pairs(*k1, *k2, maxRatio, maxDistance, cross)
                assert margin > 1e-12, (maxRatio, maxDistance, cross, margin)
                what = "mode %d (%g, %g) cross %d" % (mode, maxRatio, maxDistance, cross)
                got, ms = cs.match_ratio_host(s1, s2, maxRatio, maxDistance, bool(cross), mode)
                assert np.array_equal(got, want), what
                assert cs.match_stats()[3] == mode and ms > 0
                if len(want):
                    assert (np.diff(want[:, 0]) > 0).all()
                    if cross:
                        assert len(np.unique(want[:, 1])) == len(want)
                # device entry point: sentinel past maxPairs, the total returned, maxPairs == 0 gives only the count
                dp.upload(np.full(2 * n1, -7, np.int32))
                room = len(want) // 2
                k = L.cs_match_ratio(d1.ptr, n1, d2.ptr, n2, maxRatio, maxDistance, cross, dp.ptr, room, mode, None)
                assert k == len(want), what
                out = dp.download(np.int32, 2 * n1).reshape(-1, 2)
                assert np.array_equal(out[:room], want[:room]) and (out[room:] == -7).all(), what
                assert L.cs_match_ratio(d1.ptr, n1, d2.ptr, n2, maxRatio, maxDistance, cross, None, 0, mode, None) == len(want)
                hp = np.full((n1, 2), -7, np.int32)
                k = L.cs_match_ratio_host(s1.ctypes.data, n1, s2.ctypes.data, n2, maxRatio, maxDistance, cross,
                                          hp.ctypes.data, room, mode, None)
                assert k == len(want) and np.array_equal(hp[:room], want[:room]) and (hp[room:] == -7).all(), what
        some, _ = knn_oracle.ratio_pairs(*k1, *k2, 0.8, 0.7, 1)
        assert len(some) > 100
        assert d1.download(cs.SIFT_DTYPE, n1).tobytes() == s1.tobytes()
        assert d2.download(cs.SIFT_DTYPE, n2).tobytes() == s2.tobytes()
        pairs, _ = cs.MatchSiftDataRatio(_sift_data(cs, d1, n1), _sift_data(cs, d2, n2), mode=mode)
        assert np.array_equal(pairs, knn_oracle.ratio_pairs(*k1, *k2, 0.8, 0.7, 1)[0])
    finally:
        for b in (d1, d2, dp):
            b.free()


def _sift_data(cs, buf, n):
    d = cs.SiftData()
    d._buf, d.numPts, d.maxPts = buf, n, n
    return d


def test_records_unmodified_and_self_match(cs):
    s1, s2 = synth_descriptors(900, 41), synth_descriptors(1100, 42)
    d1, d2 = _device(cs, s1), _device(cs, s2)
    idx, sc = cs.DeviceBuffer(8 * 1100), cs.DeviceBuffer(8 * 1100)
    L = cs.lib()
    try:
        for mode in (1, 2):
            assert L.cs_match_knn2(d1.ptr, 900, d2.ptr, 1100, idx.ptr, sc.ptr, mode, None) == 0
            _eq(idx.download(np.int32, 1800).reshape(-1, 2), sc.download(np.float32, 1800).reshape(-1, 2),
                *knn_oracle.match_knn2(s1, s2), what="device mode %d" % mode)
            assert L.cs_match_ratio(d1.ptr, 900, d2.ptr, 1100, 0.8, 0.7, 1, None, 0, mode, None) >= 0
            assert d1.download(cs.SIFT_DTYPE, 900).tobytes() == s1.tobytes()
            assert d2.download(cs.SIFT_DTYPE, 1100).tobytes() == s2.tobytes()
            # a set against itself, and against an overlapping window of itself
            assert L.cs_match_knn2(d2.ptr, 1100, d2.ptr, 1100, idx.ptr, sc.ptr, mode, None) == 0
            gi = idx.download(np.int32, 2200).reshape(-1, 2)
            gs = sc.download(np.float32, 2200).reshape(-1, 2)
            _eq(gi, gs, *knn_oracle.match_knn2(s2, s2), what="self mode %d" % mode)
            assert L.cs_match_knn2(d2.ptr + 100 * 576, 1000, d2.ptr, 1100, idx.ptr, sc.ptr, mode, None) == 0
            _eq(idx.download(np.int32, 2000).reshape(-1, 2), sc.download(np.float32, 2000).reshape(-1, 2),
                *knn_oracle.match_knn2(s2[100:], s2), what="window mode %d" % mode)
            k = L.cs_match_ratio(d2.ptr, 1100, d2.ptr, 1100, 0.8, 0.7, 1, None, 0, mode, None)
            assert k >= 0
            assert d2.download(cs.SIFT_DTYPE, 1100).tobytes() == s2.tobytes()
    finally:
        for b in (d1, d2, idx, sc):
            b.free()


def test_knn_alternates_with_match_and_mutual(cs):
    """knn / ratio, MatchSiftData and mutual calls share the matcher's workspace and flag areas (a gated call among
    them): all stay exact."""
    cases = [(300, 400, 1), (512, 333, 2), (1000, 999, 3), (640, 640, 4)]
    for rnd in range(2):
        for n1, n2, seed in cases:
            s1, s2 = synth_descriptors(n1, seed), synth_descriptors(n2, seed + 50)
            if rnd == 1 and seed == 2:
                s1["data"][7, 7] = -9.0                    # gated
            k1, k2 = knn_oracle.match_knn2(s1, s2), knn_oracle.match_knn2(s2, s1)
            gi, gs, _ = cs.match_knn2(s1, s2, mode=2)
            _eq(gi, gs, *k1, what="knn %d" % seed)
            m, _ = cs.match_host(s1, s2, mode=2)
            w = oracle.match(s1, s2, threads=8)
            assert all(m[f].tobytes() == w[f].tobytes() for f in FIELDS), seed
            pairs, _ = cs.match_ratio_host(s1, s2, 0.8, 0.7, True, 2)
            assert np.array_equal(pairs, knn_oracle.ratio_pairs(*k1, *k2, 0.8, 0.7, 1)[0]), seed
            g1, g2, _, _ = cs.match_mutual_host(s1, s2, mode=2)
            assert all(g1[f].tobytes() == w[f].tobytes() for f in FIELDS), seed
            gi, gs, _ = cs.match_knn2(s2, s1, mode=2)
            _eq(gi, gs, *k2, what="knn reverse %d" % seed)


def test_ratio_purpose_shifted_views(cs):
    """Two synthetic 1920x1080 views, the second rolled by (7, 11) pixels, through a ranked extractor (N = 1000): with
    COLMAP's defaults and cross-check most pairs carry the true shift."""
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
        pairs, _ = cs.match_ratio_host(p1, p2, mode=mode)
        k1, k2 = knn_oracle.match_knn2(p1, p2), knn_oracle.match_knn2(p2, p1)
        assert np.array_equal(pairs, knn_oracle.ratio_pairs(*k1, *k2, 0.8, 0.7, 1)[0]), mode
        assert len(pairs) > 400, len(pairs)
        a, b = p1[pairs[:, 0]], p2[pairs[:, 1]]
        tol = np.maximum(2.0, a["subsampling"])
        good = (np.abs(b["xpos"] - a["xpos"] - 11) <= tol) & (np.abs(b["ypos"] - a["ypos"] - 7) <= tol)
        assert good.mean() >= 0.95, (mode, len(pairs), good.mean())
