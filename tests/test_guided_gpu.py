"""GPU checks of guided matching: cs_match_knn2_guided bit for bit against the CPU statement
(tests/guided_oracle.c) on planted two-view sets, forward motion, candidates on the admissible boundary and
degenerate positions; the reverse direction through the cross-checked pairs; the two limits (a model that admits
everything, one that admits nothing); monotonicity after verification on two shifted views; the culling statistics;
reproducibility and interleaving with the other matchers; the launch counts of single calls."""
import functools

import numpy as np
import pytest

import guided_oracle as go
import knn_oracle as ko
from cudasift_b200.synth import synth_descriptors
from test_verify_cpu import planted_views
from test_verify_gpu import _shifted_views, _sift_data

pytestmark = pytest.mark.gpu
W, H_ = 1920, 1080
NAMES = {go.H: "homography", go.F: "fundamental"}


def _eq(gi, gs, wi, ws, what):
    assert np.array_equal(gi, wi), "%s: idx differs in %d rows" % (what, int((gi != wi).any(1).sum()))
    assert gs.tobytes() == ws.tobytes(), "%s: score differs in %d rows" % (what, int((gs != ws).any(1).sum()))


def _records(xy, seed):
    r = synth_descriptors(len(xy), seed, sift_like=True)
    r["xpos"], r["ypos"] = xy[:, 0], xy[:, 1]
    return r


@functools.lru_cache(maxsize=None)
def planted(n1, n2, planar, seed):
    """Two views of one scene: n true correspondences (descriptors of set 2 a noisy copy, positions with 0.5 px noise)
    and the rest of each set random in the image.  Returns (s1, s2, model 3x3)."""
    rng = np.random.default_rng(seed)
    n = min(n1, n2) // 2
    x1, x2, F, H = planted_views(4 * n, seed, planar)
    inside = (x1 >= 0).all(1) & (x1 < [W, H_]).all(1) & (x2 >= 0).all(1) & (x2 < [W, H_]).all(1)
    x1, x2 = x1[inside][:n], x2[inside][:n] + rng.normal(0, 0.5, (n, 2))
    p1 = np.concatenate([x1, rng.uniform([0, 0], [W, H_], (n1 - n, 2))]).astype(np.float32)
    p2 = np.concatenate([x2, rng.uniform([0, 0], [W, H_], (n2 - n, 2))]).astype(np.float32)
    s1, s2 = _records(p1, seed + 1), _records(p2, seed + 2)
    s2["data"][:n] = s1["data"][:n] * 0.8 + s2["data"][:n] * 0.2
    perm = rng.permutation(n2)
    return s1, s2[perm], (H if planar else F)


def _check_both(cs, s1, s2, model, M, t, what):
    """Forward lists bit for bit; the reverse direction through the cross-checked pairs at several ratio settings."""
    gi, gs, _ = cs.match_knn2_guided(s1, s2, NAMES[model], M, t)
    k1 = go.match_knn2_guided(s1, s2, model, M, t)
    _eq(gi, gs, *k1, what=what)
    k2 = go.match_knn2_guided(s1, s2, model, M, t, reverse=True)
    for ratio, dist in ((0.8, 0.7), (1.0, 3.0)):
        want, margin = ko.ratio_pairs(*k1, *k2, ratio, dist, 1)
        got, _ = cs.match_guided_host(s1, s2, NAMES[model], M, t, ratio, dist, True)
        if margin > 1e-12:
            assert np.array_equal(got, want), (what, ratio, dist)
    st = cs.guided_stats()                      # the last call was cross-checked
    assert st[0] >= st[1] and st[2] >= int((k1[0][:, 0] >= 0).sum()) and st[3] >= int((k2[0][:, 0] >= 0).sum()), what
    return k1, k2


@pytest.mark.parametrize("model", [go.F, go.H])
@pytest.mark.parametrize("n1,n2", [(1000, 1200), (5000, 5000)])
@pytest.mark.parametrize("t", [1.0, 4.0, 16.0])
def test_planted_bit_exact(cs, model, n1, n2, t):
    s1, s2, M = planted(n1, n2, model == go.H, 11)
    _check_both(cs, s1, s2, model, M, t, "%s %dx%d t=%g" % (NAMES[model], n1, n2, t))


def test_forward_motion_epipole_at_centre(cs):
    K = np.array([[1400.0, 0, 960], [0, 1400.0, 540], [0, 0, 1]])
    tx = np.array([[0, -1.0, 0], [1.0, 0, 0], [0, 0, 0]])             # t = (0, 0, 1), R = I
    F = np.linalg.inv(K).T @ tx @ np.linalg.inv(K)
    rng = np.random.default_rng(3)
    X = np.column_stack([rng.uniform(-4, 4, 3000), rng.uniform(-2.5, 2.5, 3000), rng.uniform(6, 14, 3000)])
    p1, p2 = X @ K.T, (X + [0, 0, -1.0]) @ K.T
    x1 = (p1[:, :2] / p1[:, 2:]).astype(np.float32)
    x2 = (p2[:, :2] / p2[:, 2:] + rng.normal(0, 0.5, (3000, 2))).astype(np.float32)
    x1[:5] = [960, 540]                                                # on the epipole: a = 0
    s1, s2 = _records(x1, 4), _records(x2, 5)
    s2["data"][:2000] = s1["data"][:2000] * 0.8 + s2["data"][:2000] * 0.2
    for t in (1.0, 4.0):
        _check_both(cs, s1, s2, go.F, F, t, "forward motion t=%g" % t)


def test_candidates_on_the_boundary(cs):
    """Set-2 points at t * (1 -/+ 1e-6) from the predicted point (H) or the epipolar line (F)."""
    rng = np.random.default_rng(9)
    n = 3000
    _, _, F, _ = planted_views(10, 2, False)
    _, _, _, H = planted_views(10, 3, True)
    x1 = rng.uniform([0, 0], [W, H_], (n, 2))
    h1 = np.column_stack([x1, np.ones(n)])
    for model, M in ((go.H, H), (go.F, F)):
        for t in (1.0, 4.0):
            s = np.where(np.arange(n) % 2 == 0, 1 - 1e-6, 1 + 1e-6) * t
            if model == go.H:
                p = h1 @ M.T
                ang = rng.uniform(0, 2 * np.pi, n)
                x2 = p[:, :2] / p[:, 2:] + s[:, None] * np.column_stack([np.cos(ang), np.sin(ang)])
            else:
                l = h1 @ M.T
                nrm = np.hypot(l[:, 0], l[:, 1])
                foot = rng.uniform(0, W, n)
                on = np.column_stack([foot, -(l[:, 0] * foot + l[:, 2]) / l[:, 1]])
                x2 = on + s[:, None] * (l[:, :2] / nrm[:, None])
            s1, s2 = _records(x1.astype(np.float32), 20), _records(x2.astype(np.float32), 21)
            s2["data"] = s1["data"] * 0.7 + s2["data"] * 0.3
            _check_both(cs, s1, s2, model, M, t, "boundary %s t=%g" % (NAMES[model], t))


def test_degenerate_positions(cs):
    rng = np.random.default_rng(13)
    _, _, F, _ = planted_views(10, 4, False)
    _, _, _, H = planted_views(10, 5, True)
    Hw = H.copy()
    Hw[2] = [1e-3, 0, -0.9]                                           # pw <= 0 on most of the image
    one = np.tile([[700.5, 300.25]], (5000, 1))
    far = np.concatenate([rng.uniform([0, 0], [W, H_], (999, 2)), [[1e7, 500.0]]])
    neg = rng.uniform([-3000, -2000], [100, 100], (1500, 2))
    bad = rng.uniform([0, 0], [W, H_], (800, 2))
    bad[::7, 0] = np.nan
    bad[1::7, 1] = np.inf
    bad[2::7, 0] = -np.inf
    cases = [("one pixel", one, one), ("1e7 px", far, far[::-1].copy()), ("negative", neg, neg + 3.0),
             ("nan/inf", bad, bad[::-1].copy()), ("n = 1", far[:1], far[:1] + 1.0), ("n1 = 1", far[:1], far),
             ("n2 = 1", far, far[5:6])]
    for what, a, b in cases:
        s1, s2 = _records(a.astype(np.float32), 30), _records(b.astype(np.float32), 31)
        m = min(len(s1), len(s2))
        s2["data"][:m] = s1["data"][:m] * 0.7 + s2["data"][:m] * 0.3
        for model, M in ((go.F, F), (go.H, H), (go.H, Hw)):
            for t in (4.0, 300.0):
                _check_both(cs, s1, s2, model, M, t, "%s %s t=%g" % (what, NAMES[model], t))


def test_admits_everything_and_nothing(cs):
    s1, s2 = synth_descriptors(700, 41), synth_descriptors(900, 42)
    rng = np.random.default_rng(1)
    s1["xpos"], s1["ypos"] = rng.uniform(0, W, 700), rng.uniform(0, H_, 700)
    s2["xpos"], s2["ypos"] = rng.uniform(0, W, 900), rng.uniform(0, H_, 900)
    gi, gs, _ = cs.match_knn2_guided(s1, s2, "homography", np.eye(3), 1e5)
    for mode in (1, 2):
        _eq(gi, gs, *cs.match_knn2(s1, s2, mode=mode)[:2], what="everything mode %d" % mode)
    want, _ = cs.match_ratio_host(s1, s2)
    got, _ = cs.match_guided_host(s1, s2, "homography", np.eye(3), 1e5)
    assert np.array_equal(got, want)
    assert cs.guided_stats()[:2] == [700 * 900 * 2, 700 * 900 * 2]
    T = np.array([[1, 0, 1e6], [0, 1, 0], [0, 0, 1.0]])                # everything predicted 1e6 px away
    for model, M in (("homography", T), ("fundamental", np.array([[0, 0, 0], [0, 0, 0], [0, 0, 1.0]]))):
        gi, gs, _ = cs.match_knn2_guided(s1, s2, model, M, 4.0)
        assert (gi == -1).all() and (gs == 0).all(), model
        pairs, _ = cs.match_guided_host(s1, s2, model, M, 4.0)
        st = cs.guided_stats()
        assert len(pairs) == 0 and st[1] == 0 and st[2] == 0 and st[3] == 0, (model, st)


def test_pairs_vs_oracle_lists(cs):
    s1, s2, M = planted(2000, 2500, False, 17)
    k1 = go.match_knn2_guided(s1, s2, go.F, M, 4.0)
    k2 = go.match_knn2_guided(s1, s2, go.F, M, 4.0, reverse=True)
    d1, d2 = _sift_data(cs, s1), _sift_data(cs, s2)
    try:
        for ratio, dist in ((0.8, 0.7), (0.6, 0.5), (0.9, 1.6)):
            for cross in (False, True):
                want, margin = ko.ratio_pairs(*k1, *k2, ratio, dist, cross)
                if margin < 1e-12:
                    continue
                got, ms = cs.MatchSiftDataGuided(d1, d2, "fundamental", M, 4.0, ratio, dist, cross)
                assert np.array_equal(got, want) and ms > 0, (ratio, dist, cross)
                host, _ = cs.match_guided_host(s1, s2, "fundamental", M, 4.0, ratio, dist, cross)
                assert np.array_equal(host, want)
        assert len(ko.ratio_pairs(*k1, *k2, 0.8, 0.7, 1)[0]) > 500
        assert d1._buf.download(cs.SIFT_DTYPE, len(s1)).tobytes() == s1.tobytes()
    finally:
        cs.FreeSiftData(d1)
        cs.FreeSiftData(d2)


def test_monotonic_after_verification(cs):
    """ratio -> VerifyPairs -> MatchSiftDataGuided on two shifted views: every ratio pair the predicate admits is a
    guided pair (its best candidate stays admissible, its second best can only get worse), and every guided pair
    satisfies the predicate."""
    p1, p2 = _shifted_views(cs)
    d1, d2 = _sift_data(cs, p1), _sift_data(cs, p2)
    try:
        pairs, _ = cs.MatchSiftDataRatio(d1, d2)
        for model in ("homography", "fundamental"):
            M, inl, _ = cs.VerifyPairs(d1, d2, pairs, model=model)
            g, _ = cs.MatchSiftDataGuided(d1, d2, model, M, 4.0)
            code = cs.GEOM_MODELS[model]
            adm = go.admissible_c(code, M, 4.0, p1["xpos"][pairs[:, 0]], p1["ypos"][pairs[:, 0]],
                                  p2["xpos"][pairs[:, 1]], p2["ypos"][pairs[:, 1]])
            gs = {tuple(r) for r in g}
            assert all(tuple(r) in gs for r in pairs[adm]), model
            assert go.admissible_c(code, M, 4.0, p1["xpos"][g[:, 0]], p1["ypos"][g[:, 0]], p2["xpos"][g[:, 1]],
                                   p2["ypos"][g[:, 1]]).all(), model
            assert len(g) >= adm.sum() and len(g) > 400, (model, len(g), adm.sum())
    finally:
        cs.FreeSiftData(d1)
        cs.FreeSiftData(d2)


def test_culling(cs):
    """F at 4 px on 5000 x 5000 points of a 1920x1080 view: the grid aims at 2 candidates per cell, so a cell is
    about c = sqrt(1920 * 1080 * 2 / 5000) = 29 px wide.  A strip of half-width ~4-8 px crosses every cell column in at
    most 1 + 2 * 8 / c + (slope <= 1) < 3 cells, about 3 * c / 1080 of the candidates: evaluations stay below
    4 * c / 1080 (11 %) of n1 * n2 per direction."""
    s1, s2, F = planted(5000, 5000, False, 11)
    _, _ = cs.match_guided_host(s1, s2, "fundamental", F, 4.0)
    st = cs.guided_stats()
    c = np.sqrt(W * H_ * 2 / 5000)
    assert st[1] <= st[0] <= 2 * 4 * c / H_ * 5000 * 5000, (st, c)
    assert st[1] > 0 and st[2] > 2000 and st[3] > 2000, st


def test_reproducible_host_equals_device_and_interleaving(cs):
    s1, s2, F = planted(3000, 3000, False, 23)
    t1, t2 = synth_descriptors(600, 51), synth_descriptors(700, 52)
    d1, d2 = _sift_data(cs, s1), _sift_data(cs, s2)
    try:
        a, _ = cs.MatchSiftDataGuided(d1, d2, "fundamental", F, 4.0)
        sa = cs.guided_stats()
        li, ls, _ = cs.match_knn2_guided(s1, s2, "fundamental", F, 4.0)
        m0, _ = cs.match_host(t1, t2, mode=2)
        q0, _ = cs.match_ratio_host(t1, t2, mode=2)
        v0 = cs.VerifyPairs(d1, d2, a, model="fundamental", numLoops=512)
        for rnd in range(3):
            b, _ = cs.MatchSiftDataGuided(d1, d2, "fundamental", F, 4.0)
            assert np.array_equal(a, b) and cs.guided_stats() == sa
            m, _ = cs.match_host(t1, t2, mode=2 if rnd % 2 == 0 else 1)
            h, _ = cs.match_guided_host(s1, s2, "fundamental", F, 4.0)
            assert np.array_equal(h, a) and cs.guided_stats() == sa
            q, _ = cs.match_ratio_host(t1, t2, mode=2)
            v = cs.VerifyPairs(d1, d2, a, model="fundamental", numLoops=512)
            gi, gs, _ = cs.match_knn2_guided(s1, s2, "fundamental", F, 4.0)
            assert m.tobytes() == m0.tobytes() and np.array_equal(q, q0)
            assert v[0].tobytes() == v0[0].tobytes() and np.array_equal(v[1], v0[1])
            _eq(gi, gs, li, ls, "round %d" % rnd)
        assert cs.guided_stats()[3] == 0                                  # a one-way call
    finally:
        cs.FreeSiftData(d1)
        cs.FreeSiftData(d2)


def test_single_call_launches(cs):
    """A single call runs as one job of the batch waves: 7 launches for cs_match_guided with or without the cross-check
    (both directions' knn in one launch), 5 for cs_match_knn2_guided (no ratio test or pair writes)."""
    s1, s2, F = planted(1000, 1200, False, 11)
    L = cs.lib()
    for cross in (False, True):
        before = L.cs_launch_count()
        pairs, _ = cs.match_guided_host(s1, s2, "fundamental", F, 4.0, crossCheck=cross)
        assert L.cs_launch_count() - before == 7 and len(pairs) > 0, cross
    before = L.cs_launch_count()
    cs.match_knn2_guided(s1, s2, "fundamental", F, 4.0)
    assert L.cs_launch_count() - before == 5
