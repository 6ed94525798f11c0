"""GPU checks of geometric verification (cs_verify_pairs): every minimal-solver slot against the float64 restatement
(tests/verify_oracle.py), planted fundamental matrices and homographies with noise and outliers, the chain ranked
extraction -> ratio matching -> verification on two shifted views, reproducibility, edge cases and interleaving with
the matchers."""
import ctypes
import functools

import numpy as np
import pytest

import verify_oracle as vo
from cudasift_b200.synth import synth_descriptors, synth_image
from test_verify_cpu import planted_views

pytestmark = pytest.mark.gpu
W, H_ = 1920, 1080


def _records(cs, xy):
    r = np.zeros(len(xy), cs.SIFT_DTYPE)
    r["xpos"], r["ypos"] = xy[:, 0], xy[:, 1]
    return r


def planted(n, seed, planar, sigma=0.5, outliers=0.4):
    """n pairs of two 1920x1080 views: inliers with Gaussian noise, uniform outliers.  The pairs are (k, perm[k]) in a
    shuffled order of set 2.  Returns (x1, x2 float32 [n, 2], pairs, inlier mask, F, H)."""
    rng = np.random.default_rng(seed)
    x1, x2, F, H = planted_views(4 * n, seed, planar)
    inside = (x1 >= 0).all(1) & (x1 < [W, H_]).all(1) & (x2 >= 0).all(1) & (x2 < [W, H_]).all(1)
    x1, x2 = x1[inside][:n], x2[inside][:n]
    assert len(x1) == n
    x2 = x2 + rng.normal(0, sigma, x2.shape)
    out = rng.random(n) < outliers
    x2[out] = rng.uniform([0, 0], [W, H_], (out.sum(), 2))
    perm = rng.permutation(n)
    s2 = np.empty_like(x2)
    s2[perm] = x2
    pairs = np.column_stack([np.arange(n), perm]).astype(np.int32)
    return x1.astype(np.float32), s2.astype(np.float32), pairs, ~out, F, H


class Dev:
    """Device copies of two record sets and a pair list."""

    def __init__(self, cs, r1, r2, pairs):
        self.cs, self.n1, self.n2, self.np = cs, len(r1), len(r2), len(pairs)
        self.b = [cs.DeviceBuffer(max(r1.nbytes, 576)), cs.DeviceBuffer(max(r2.nbytes, 576)),
                  cs.DeviceBuffer(max(8 * len(pairs), 8)), cs.DeviceBuffer(max(8 * len(pairs), 8))]
        self.b[0].upload(r1)
        self.b[1].upload(r2)
        if len(pairs):
            self.b[2].upload(np.ascontiguousarray(pairs, np.int32))

    def verify(self, model, loops, thresh, seed, maxInliers=None):
        mi = self.np if maxInliers is None else maxInliers
        out = np.zeros(9)
        k = self.cs.lib().cs_verify_pairs(self.b[0].ptr, self.n1, self.b[1].ptr, self.n2, self.b[2].ptr, self.np, model,
                                          loops, thresh, seed, out.ctypes.data, self.b[3].ptr, mi, None)
        assert k >= 0, self.cs.lib().cs_last_error()
        return k, out.reshape(3, 3), self.b[3].download(np.int32, 2 * min(k, mi)).reshape(-1, 2)

    def models(self, model, loops, thresh, seed):
        M, C, N = np.zeros((3 * loops, 9)), np.zeros(3 * loops, np.int32), np.zeros(5)
        v = self.cs.lib().cs_verify_models(self.b[0].ptr, self.n1, self.b[1].ptr, self.n2, self.b[2].ptr, self.np, model,
                                           loops, thresh, seed, M.ctypes.data, C.ctypes.data, N.ctypes.data)
        assert v >= 0, self.cs.lib().cs_last_error()
        return v, M, C, N

    def free(self):
        for b in self.b:
            b.free()


def _coords(x1, x2, pairs):
    return np.column_stack([x1[pairs[:, 0]], x2[pairs[:, 1]]]).astype(np.float64)


@pytest.mark.parametrize("model", [vo.FUNDAMENTAL, vo.HOMOGRAPHY])
def test_solver_parity_slot_by_slot(cs, model):
    x1, x2, pairs, _, _, _ = planted(600, 5, model == vo.HOMOGRAPHY, outliers=0.3)
    thresh, loops, seed = 2.0, 1024, 77
    d = Dev(cs, _records(cs, x1), _records(cs, x2), pairs)
    try:
        v, M, C, N = d.models(model, loops, thresh, seed)
    finally:
        d.free()
    p = _coords(x1, x2, pairs)
    assert v == len(p)
    want, smp, (c1, c2, s) = vo.slot_models(p, model, loops, seed)
    assert np.allclose(N, [c1[0], c1[1], c2[0], c2[1], s], rtol=1e-12, atol=0)
    live_g, live_w = ~np.isnan(M[:, 0]), ~np.isnan(want[:, 0])
    assert live_g.sum() > 0.9 * loops
    either = live_g | live_w
    agree = np.zeros(len(M), bool)
    for k in np.nonzero(live_g & live_w)[0]:
        agree[k] = vo.same_model(M[k], want[k], model) < 1e-6
    assert agree.sum() >= 0.995 * either.sum(), (agree.sum(), either.sum())
    for k in np.nonzero(agree)[0]:
        r = vo.residuals(want[k], model, p)
        w = int((r < thresh).sum())
        border = int((np.abs(r - thresh) <= 1e-4 * thresh).sum())
        assert abs(int(C[k]) - w) <= border, (k, C[k], w, border)
    assert (C[~live_g] == 0).all()


def _sampson_rms(F, p):
    return float(np.sqrt(np.mean(vo.residuals(F, vo.FUNDAMENTAL, p) ** 2)))


def test_planted_fundamental(cs):
    x1, x2, pairs, good, _, _ = planted(2000, 21, False)
    d = Dev(cs, _records(cs, x1), _records(cs, x2), pairs)
    try:
        k, F, inl = d.verify(vo.FUNDAMENTAL, 4096, 2.0, 0)
        st = cs.verify_stats()
        _, M, _, _ = d.models(vo.FUNDAMENTAL, 4096, 2.0, 0)
    finally:
        d.free()
    assert k == len(inl) == st[7] and st[0] == 2000 and st[1] == 0 and st[4] >= 0
    assert (np.diff(inl[:, 0]) > 0).all()                                   # input order
    got = np.zeros(2000, bool)
    got[inl[:, 0]] = True
    assert np.array_equal(pairs[got], inl)
    assert got[good].mean() >= 0.97, got[good].mean()
    assert got[~good].mean() <= 0.03, got[~good].mean()
    p = _coords(x1, x2, pairs)
    minimal = M[st[4]]
    assert _sampson_rms(F, p[good]) <= _sampson_rms(minimal, p[good]) * (1 + 1e-9)
    assert abs(np.linalg.norm(F) - 1) < 1e-12 and F.reshape(-1)[np.argmax(np.abs(F))] > 0
    try:
        import cv2
    except ImportError:
        return
    _, mask = cv2.findFundamentalMat(p[:, :2], p[:, 2:], cv2.FM_RANSAC, 2.0, 0.999)
    assert k >= 0.97 * int(mask.sum()), (k, int(mask.sum()))


def test_planted_homography(cs):
    x1, x2, pairs, good, _, H = planted(2000, 31, True)
    d = Dev(cs, _records(cs, x1), _records(cs, x2), pairs)
    try:
        k, Hg, inl = d.verify(vo.HOMOGRAPHY, 4096, 2.0, 0)
    finally:
        d.free()
    got = np.zeros(2000, bool)
    got[inl[:, 0]] = True
    assert got[good].mean() >= 0.97 and got[~good].mean() <= 0.03, (got[good].mean(), got[~good].mean())
    assert Hg[2, 2] == 1.0
    corners = np.array([[0, 0, 1], [W, 0, 1], [0, H_, 1], [W, H_, 1]], np.float64)
    a, b = corners @ Hg.T, corners @ H.T
    assert np.abs(a[:, :2] / a[:, 2:] - b[:, :2] / b[:, 2:]).max() < 1.0


@functools.lru_cache(maxsize=None)
def _shifted_views(cs):
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
            assert ex.wait() == 1000
            sets.append(ex.device_points_at(0, 1000))
    finally:
        ex.close()
    return sets[0], sets[1]


def _sift_data(cs, recs):
    d = cs.SiftData()
    cs.InitSiftData(d, len(recs))
    d._buf.upload(recs)
    d.numPts = len(recs)
    return d


def test_end_to_end_shifted_views(cs):
    """Ranked extraction (N = 1000) -> cross-checked ratio matching -> verification, on two views rolled by (7, 11).
    An odd shift does not survive downsampling, so the coarse octaves' keypoints move by more than the shift: the median
    error of the pairs is 0 px at subsampling 1, 0.6 px at 2, 1.9 px at 8 and 4 px at 16.  With COLMAP's 4 px the
    least-squares H therefore extrapolates to the image corners within about 1-1.7 px, and the bound here is 2 px."""
    p1, p2 = _shifted_views(cs)
    d1, d2 = _sift_data(cs, p1), _sift_data(cs, p2)
    try:
        pairs, _ = cs.MatchSiftDataRatio(d1, d2)
        assert len(pairs) > 400
        Hm, inl, ms = cs.VerifyPairs(d1, d2, pairs, model="homography")
        assert ms > 0
        corners = np.array([[0, 0, 1], [W, 0, 1], [0, H_, 1], [W, H_, 1]], np.float64)
        q = corners @ Hm.T
        assert np.abs(q[:, :2] / q[:, 2:] - (corners[:, :2] + [11, 7])).max() < 2.0, Hm
        a, b = p1[pairs[:, 0]], p2[pairs[:, 1]]
        shifted = (np.abs(b["xpos"] - a["xpos"] - 11) <= 1.0) & (np.abs(b["ypos"] - a["ypos"] - 7) <= 1.0)
        kept = {tuple(r) for r in inl}
        hit = np.array([tuple(r) in kept for r in pairs])
        assert hit[shifted].mean() >= 0.99, (hit[shifted].mean(), shifted.sum())
        Fm, inlF, _ = cs.VerifyPairs(d1, d2, pairs, model="fundamental")
        assert len(inlF) >= 0.95 * len(pairs), (len(inlF), len(pairs))
        # the host variant gives the same bytes
        Hh, inlh, _ = cs.verify_pairs_host(p1, p2, pairs, model="homography")
        assert Hh.tobytes() == Hm.tobytes() and np.array_equal(inlh, inl)
    finally:
        cs.FreeSiftData(d1)
        cs.FreeSiftData(d2)


@pytest.mark.parametrize("model", [vo.FUNDAMENTAL, vo.HOMOGRAPHY])
def test_reproducible_and_host_equals_device(cs, model):
    x1, x2, pairs, _, _, _ = planted(3000, 41, model == vo.HOMOGRAPHY)
    r1, r2 = _records(cs, x1), _records(cs, x2)
    d = Dev(cs, r1, r2, pairs)
    try:
        a = d.verify(model, 2048, 3.0, 12345)
        sa = cs.verify_stats()
        b = d.verify(model, 2048, 3.0, 12345)
        assert cs.verify_stats() == sa
        c = d.verify(model, 2048, 3.0, 999)
    finally:
        d.free()
    assert a[0] == b[0] and a[1].tobytes() == b[1].tobytes() and np.array_equal(a[2], b[2])
    h = cs.verify_pairs_host(r1, r2, pairs, model, 2048, 3.0, 12345)
    assert cs.verify_stats() == sa
    assert h[0].tobytes() == a[1].tobytes() and np.array_equal(h[1], a[2])
    assert c[0] > 0.5 * len(pairs)                      # another seed: another sample sequence, a similar answer
    assert 0 < sa[2] <= 2048 and sa[3] >= sa[2] and sa[6] in (0, 1)
    assert sa[7] >= sa[5] if sa[6] else sa[7] == sa[5]           # a refit is kept only when it has no fewer inliers


def test_edge_cases(cs):
    L = cs.lib()
    x1, x2, pairs, _, _, _ = planted(500, 51, False, outliers=0.2)
    r1, r2 = _records(cs, x1), _records(cs, x2)
    # too few valid pairs: 3 for H, 6 for F
    for model, n in ((vo.HOMOGRAPHY, 3), (vo.FUNDAMENTAL, 6)):
        M, inl, _ = cs.verify_pairs_host(r1, r2, pairs[:n], model, 64, 2.0, 0)
        st = cs.verify_stats()
        assert len(inl) == 0 and not M.any() and st[0] == n and st[2] == 0 and st[4] == -1 and st[7] == 0
    # all pairs at one point; collinear points in both images
    one = _records(cs, np.tile([[100.0, 200.0]], (50, 1)))
    for model in (vo.HOMOGRAPHY, vo.FUNDAMENTAL):
        M, inl, _ = cs.verify_pairs_host(one, one, np.column_stack([np.arange(50)] * 2), model, 256, 2.0, 0)
        assert len(inl) == 0 and not M.any() and cs.verify_stats()[2] == 0
    t = np.linspace(0, 1, 60)
    line1 = _records(cs, np.column_stack([100 + 1500 * t, 100 + 800 * t]))
    line2 = _records(cs, np.column_stack([120 + 1400 * t, 90 + 850 * t]))
    lp = np.column_stack([np.arange(60)] * 2)
    M, inl, _ = cs.verify_pairs_host(line1, line2, lp, vo.HOMOGRAPHY, 256, 2.0, 0)
    assert len(inl) == 0 and not M.any() and cs.verify_stats()[2] == 0
    M, inl, _ = cs.verify_pairs_host(line1, line2, lp, vo.FUNDAMENTAL, 256, 2.0, 0)
    assert len(inl) <= 60
    # out-of-range indices and NaN coordinates: excluded and counted
    bad = pairs.copy()
    bad[3] = [-1, 0]; bad[10] = [0, 500]; bad[20] = [500, 0]; bad[30] = [2 ** 31 - 1, 5]
    rn = r1.copy()
    rn["xpos"][40] = np.nan
    rn["ypos"][41] = np.inf
    M, inl, _ = cs.verify_pairs_host(rn, r2, bad, vo.FUNDAMENTAL, 1024, 2.0, 0)
    st = cs.verify_stats()
    assert st[0] == 494 and st[1] == 6 and st[7] == len(inl) > 300
    assert not set(map(tuple, inl)) & {(-1, 0), (0, 500), (500, 0), (2 ** 31 - 1, 5)}
    assert not ({40, 41} & set(inl[:, 0].tolist()))
    # maxInliers below the count: only that many written, the total returned
    d = Dev(cs, r1, r2, pairs)
    try:
        k, _, full = d.verify(vo.FUNDAMENTAL, 1024, 2.0, 0)
        d.b[3].upload(np.full(2 * len(pairs), -7, np.int32))
        k2, _, part = d.verify(vo.FUNDAMENTAL, 1024, 2.0, 0, maxInliers=10)
        rest = d.b[3].download(np.int32, 2 * len(pairs)).reshape(-1, 2)
        assert k2 == k > 10 and np.array_equal(part, full[:10]) and (rest[10:] == -7).all()
        out = np.full(9, 3.0)
        assert L.cs_verify_pairs(d.b[0].ptr, 500, d.b[1].ptr, 500, d.b[2].ptr, 500, 2, 64, 2.0, 0, out.ctypes.data,
                                 None, 0, None) > 0
        # numPairs == 0
        assert L.cs_verify_pairs(d.b[0].ptr, 500, d.b[1].ptr, 500, None, 0, 2, 64, 2.0, 0, out.ctypes.data, None, 0,
                                 None) == 0 and not out.any()
        # numLoops at both ends
        for model in (vo.FUNDAMENTAL, vo.HOMOGRAPHY):
            for loops in (1, 65536):
                k, M, inl = d.verify(model, loops, 2.0, 3)
                st = cs.verify_stats()
                assert st[2] <= loops and k == len(inl) and np.isfinite(M).all()
                if loops == 65536 and model == vo.FUNDAMENTAL:        # the scene is not planar: H has few inliers
                    assert k > 300
    finally:
        d.free()


def test_interleaving_with_matchers(cs):
    """Verify calls alternate with MatchSiftData and ratio matching: the scratch areas do not disturb each other."""
    x1, x2, pairs, _, _, _ = planted(1500, 61, False)
    r1, r2 = _records(cs, x1), _records(cs, x2)
    s1, s2 = synth_descriptors(700, 3), synth_descriptors(650, 4)
    v0 = cs.verify_pairs_host(r1, r2, pairs, "fundamental", 1024, 2.0, 0)
    h0 = cs.verify_pairs_host(r1, r2, pairs, "homography", 256, 2.0, 0)
    m0, _ = cs.match_host(s1, s2, mode=2)
    q0, _ = cs.match_ratio_host(s1, s2, mode=2)
    for rnd in range(3):
        q, _ = cs.match_ratio_host(s1, s2, mode=2)
        v = cs.verify_pairs_host(r1, r2, pairs, "fundamental", 1024, 2.0, 0)
        m, _ = cs.match_host(s1, s2, mode=2 if rnd % 2 == 0 else 1)
        h = cs.verify_pairs_host(r1, r2, pairs, "homography", 256, 2.0, 0)
        assert np.array_equal(q, q0) and m.tobytes() == m0.tobytes()
        assert v[0].tobytes() == v0[0].tobytes() and np.array_equal(v[1], v0[1])
        assert h[0].tobytes() == h0[0].tobytes() and np.array_equal(h[1], h0[1])
