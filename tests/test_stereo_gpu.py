"""GPU checks of dense reconstruction against tests/stereo_oracle.py: the cost at every pixel, the start draws, every
half-step replayed, accuracy against the rendered truth, fusion, undistortion, determinism and batching."""
import numpy as np
import pytest

import cudasift_b200 as cs
import stereo_cases as sc
import stereo_oracle as so
from test_stereo_cpu import DEPTH_FRACTION, NORMAL_MEDIAN_DEG, accuracy

pytestmark = pytest.mark.gpu

COST_BOUND = 2e-3          # the header's FP32 bound on a view cost, which bounds the mean of topK of them too
R, STEP, TOPK = 3, 1, 2


@pytest.fixture(scope="module")
def small():
    Ks, Rs, ts, views = sc.render(6, 160, 120, seed=1)
    images = [v[0] for v in views]
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(6)]) if b != a][:4], 3.0, 12.0) for a in range(6)]
    return Ks, Rs, ts, views, images, jobs


def _pm(small, n, jobs=None, **kw):
    Ks, Rs, ts, _, images, js = small
    return cs.PatchMatchStereo(images, Ks, Rs, ts, js if jobs is None else jobs, windowRadius=R, windowStep=STEP,
                               numIterations=n, topK=TOPK, seed=3, **kw)


def _job(small, p):
    Ks, Rs, ts, _, _, jobs = small
    a, s, lo, hi = jobs[p]
    return so.Job(Ks, Rs, ts, a, s, lo, hi)


def test_start_equals_the_draws(small):
    d, n, c, stats, _ = _pm(small, 0)
    for p in (0, 3):
        job = _job(small, p)
        H, W = d[p].shape
        y, x = [v.reshape(-1) for v in np.mgrid[0:H, 0:W]]
        z, nn = so.random_hyp(3, job, W, x, y, 0, 0)
        assert np.all(np.abs(d[p].reshape(-1) - z) <= np.spacing(z))
        assert np.all(np.abs(n[p].reshape(-1, 3) - nn) <= np.spacing(np.abs(nn)) + 1e-12)
    assert np.all(stats[:, 0] == 160 * 120)


def test_cost_at_every_pixel(small):
    d, n, c, stats, _ = _pm(small, 2)
    Ks, Rs, ts, _, images, jobs = small
    for p in (1, 4):
        job = _job(small, p)
        H, W = d[p].shape
        y, x = [v.reshape(-1) for v in np.mgrid[0:H, 0:W]]
        oc, _, mar = so.cost(images, job, x, y, d[p].reshape(-1), n[p].reshape(-1, 3), R, STEP, TOPK)
        diff = np.abs(oc - c[p].reshape(-1))
        assert mar.mean() < 0.01, mar.mean()
        assert np.all(diff[~mar] <= COST_BOUND), diff[~mar].max()
        assert np.all(np.isfinite(d[p])) and np.all(np.isfinite(n[p]))
        assert stats[p, 2] == int((c[p] >= 2).sum())


def _check_half(small, p, before, after, it, colour):
    """The GPU's pixels of `colour` in `after` are admissible choices of the oracle's half-step from `before`."""
    _, _, _, _, images, _ = small
    job = _job(small, p)
    _, opt = so.half_step(images, job, before, it, colour, 3, R, STEP, TOPK, eps=2 * COST_BOUND)
    x, y = opt["x"], opt["y"]
    gz, gn = after[0][y, x], after[1][y, x]
    same = (np.abs(opt["z"] - gz[None]) <= 1e-5 * np.abs(gz[None])) & \
        np.all(np.abs(opt["n"] - gn[None]) <= 1e-5, axis=-1)
    ok = np.any(same & opt["admissible"], axis=0)
    marginal = np.any(opt["marginal"] & opt["admissible"], axis=0)
    assert np.all(ok | marginal), (it, colour, int((~ok & ~marginal).sum()))
    return marginal.mean()


def test_every_half_step_replayed(small):
    runs = [_pm(small, n) for n in range(5)]
    fr = []
    for nIt in range(4):
        for p in (0, 5):
            Sn = (runs[nIt][0][p], runs[nIt][1][p], runs[nIt][2][p])
            Sn1 = (runs[nIt + 1][0][p], runs[nIt + 1][1][p], runs[nIt + 1][2][p])
            fr.append(_check_half(small, p, Sn, Sn1, nIt + 1, 0))
            H, W = Sn[0].shape
            even = ((np.add.outer(np.arange(H), np.arange(W))) & 1) == 0
            mid = tuple(np.where(even[..., None] if a.ndim == 3 else even, b, a) for a, b in zip(Sn, Sn1))
            fr.append(_check_half(small, p, mid, Sn1, nIt + 1, 1))
    print("marginal fraction per half-step:", ["%.4f" % f for f in fr])
    assert max(fr) < 0.01


def test_accuracy_at_640x480():
    Ks, Rs, ts, views = sc.render(8, 640, 480, seed=2)
    a, sources = 3, [2, 4, 1, 5, 0, 6, 7]
    d, n, c, stats, ms = cs.PatchMatchStereo([v[0] for v in views], Ks, Rs, ts, [(a, sources, 3.0, 12.0)])
    frac, med = accuracy(views, Ks, Rs, ts, a, sources, d[0], n[0])
    print("640x480: %.3f within 1 %%, median normal error %.1f deg, %.1f ms" % (frac, med, ms))
    assert frac >= DEPTH_FRACTION and med <= NORMAL_MEDIAN_DEG


def test_fusion(small):
    Ks, Rs, ts, views, images, jobs = small
    d, n, c, _, _ = _pm(small, 6)
    args = dict(maxCost=0.5, minConsistent=2, maxReprojError=2.0, maxDepthError=0.01, maxNormalErrorDeg=10.0)
    xyz, nrm, inten, src, total, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, d, n, c, **args)
    assert total == len(xyz) > 0
    rows = so.fuse(images, Ks, Rs, ts, jobs, d, n, c, *args.values())
    want = {(r[0], r[1]): (r[3], r[4], r[5]) for r in rows if r[2]}
    sure = {(r[0], r[1]) for r in rows if r[6] > 1e-6}
    got = {(int(a), int(p)): k for k, (a, p) in enumerate(src)}
    assert list(got) == sorted(got)
    assert {k for k in got if k in sure} == {k for k in want if k in sure}
    for key, k in got.items():
        if key in want:
            X, N, I = want[key]
            assert np.allclose(xyz[k], X, rtol=1e-5, atol=1e-5 * 10) and np.allclose(nrm[k], N, atol=1e-5)
            assert abs(inten[k] - I) <= 1e-5 * max(1.0, abs(I))
    near = 0
    sceneDepth = max(float(v[1].max()) for v in views)
    for (a, p), k in got.items():
        z = Rs[a][2] @ xyz[k] + ts[a][2]
        near += abs(z - views[a][1].reshape(-1)[p]) <= 0.005 * sceneDepth
    print("fusion: %d points, %.3f within 0.5 %% of the scene depth" % (len(got), near / len(got)))
    assert near >= 0.95 * len(got), near / len(got)
    half = total // 2
    xyz2, _, _, src2, total2, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, d, n, c, maxPoints=half, **args)
    assert total2 == total and len(src2) == half
    assert np.array_equal(src2, src[:half]) and np.array_equal(xyz2, xyz[:half])


def test_undistortion():
    rng = np.random.default_rng(4)
    Ks, Rs, ts = sc.cameras(3, 200, 150, seed=5)
    dists = np.array([[-0.12, 0.03], [0.08, -0.02], [0.0, 0.0]])
    imgs = [rng.uniform(0, 255, (150, 200)).astype(np.float32) for _ in range(3)]
    out, outside, _ = cs.UndistortImages(imgs, Ks, dists)
    for a in range(3):
        ref, n = so.undistort(imgs[a], Ks[a], dists[a])
        assert np.max(np.abs(out[a] - ref)) <= 1e-3 and outside[a] == n
    assert np.array_equal(out[2][1:-1, 1:-1], imgs[2][1:-1, 1:-1])  # the header's 1-pixel border aside
    tex = sc._texture()
    for a in range(2):
        pin = sc.cast(Ks[a], Rs[a], ts[a], 200, 150, tex=tex)[0]
        dis = sc.cast(Ks[a], Rs[a], ts[a], 200, 150, dist=dists[a], tex=tex)[0]
        und = cs.UndistortImages([dis], Ks[a], dists[a])[0][0]
        inner = (slice(20, -20), slice(25, -25))
        assert np.median(np.abs(und[inner] - pin[inner])) < 2.0


def test_undistortion_of_65536_images():
    """The header's largest image count in one call (more images than a grid's z extent)."""
    import ctypes
    N, w, h = 65536, 4, 3
    rng = np.random.default_rng(6)
    imgs = rng.uniform(0, 255, (N, h, w)).astype(np.float32)
    K = np.array([[3.0, 0.2, 1.5], [0, 2.8, 1.0], [0, 0, 1]])
    dist = np.array([0.3, -0.1])
    src, dst = cs.DeviceBuffer(imgs.nbytes), cs.DeviceBuffer(imgs.nbytes)
    try:
        src.upload(imgs)
        table = (cs.StereoImage * N)(*[cs.StereoImage(src.ptr + 4 * w * h * a, w, h, w) for a in range(N)])
        outs = (ctypes.c_void_p * N)(*[dst.ptr + 4 * w * h * a for a in range(N)])
        Ks, dists = np.ascontiguousarray(np.broadcast_to(K, (N, 3, 3))), np.ascontiguousarray(np.broadcast_to(dist, (N, 2)))
        outside = np.zeros(N, np.int64)
        assert cs.lib().cs_undistort_images(table, N, Ks.ctypes.data, dists.ctypes.data, outs, outside.ctypes.data,
                                            None) == 0, cs.lib().cs_last_error()
        got = dst.download(np.float32, imgs.size).reshape(N, h, w)
    finally:
        src.free()
        dst.free()
    for a in (0, 65534, 65535):
        ref, n = so.undistort(imgs[a], K, dist)
        assert np.max(np.abs(got[a] - ref)) <= 1e-3 and outside[a] == n


def test_determinism_batching_and_launches():
    Ks, Rs, ts = sc.cameras(6, 160, 120, seed=1)
    tex = sc._texture()
    S = np.diag([0.8, 0.8, 1.0])
    Ks = np.array([K if a < 3 else S @ K for a, K in enumerate(Ks)])
    images = [sc.cast(Ks[a], Rs[a], ts[a], 160 if a < 3 else 128, 120 if a < 3 else 96, tex=tex)[0] for a in range(6)]
    jobs = [(a, [b for b in range(6) if b != a][:3], 3.0, 12.0) for a in range(6)]
    L = cs.lib()
    c0 = L.cs_launch_count()
    first = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs, windowRadius=2, numIterations=3, seed=9)
    assert L.cs_launch_count() - c0 == 2 + 2 * 3
    again = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs, windowRadius=2, numIterations=3, seed=9)
    for k in range(3):
        for p in range(6):
            assert first[k][p].tobytes() == again[k][p].tobytes()
    for p in range(6):
        alone = cs.PatchMatchStereo(images, Ks, Rs, ts, [jobs[p]], windowRadius=2, numIterations=3, seed=9)
        for k in range(3):
            assert alone[k][0].tobytes() == first[k][p].tobytes(), (p, k)
    c0 = L.cs_launch_count()
    cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, *first[:3])
    cs.UndistortImages(images, Ks, np.zeros(2))
    assert L.cs_launch_count() - c0 == 3


def test_end_to_end_on_library_outputs():
    """extract -> MatchSiftDataRatioBatch -> BuildTracks -> TriangulateTracks -> SelectStereoViews -> PatchMatchStereo
    -> FuseDepthMaps on a rendered scene with known cameras.

    The pixel convention is checked twice.  First directly: Gaussian blobs rendered at known sub-pixel centres, pixel
    (col, row) holding the blob's value at (col, row), are extracted at those centres within 0.05 px; a half-pixel
    offset between the records and the images would miss by 0.5.  Then through the chain: with the true cameras, the
    triangulated tracks reproject onto their records.  That second check alone would not see an offset shared by
    every image, which acts like a shift of every principal point."""
    rng = np.random.default_rng(0)
    yy, xx = np.mgrid[0:256, 0:320].astype(np.float64)
    blob = np.full((256, 320), 60.0)
    centres = []
    while len(centres) < 8:
        c = rng.uniform(30, [290, 226])
        if all(np.hypot(*(c - d)) >= 40 for d in centres):
            centres.append(c)
            blob += 150.0 * np.exp(-((xx - c[0]) ** 2 + (yy - c[1]) ** 2) / (2 * 3.0 ** 2))
    rec = cs.extract_host(blob.astype(np.float32), numOctaves=5, initBlur=1.0, thresh=3.0)
    for c in centres:
        d = np.hypot(rec["xpos"] - c[0], rec["ypos"] - c[1])
        assert d.min() <= 0.05, (c, d.min())

    Ks, Rs, ts, views = sc.render(8, 640, 480, seed=2, texels=96)
    images = [v[0] for v in views]
    datas = []
    try:
        for im in images:
            r = cs.extract_host(im, numOctaves=5, initBlur=1.0, thresh=3.0)
            d = cs.InitSiftData(cs.SiftData(), max(len(r), 1))
            d._buf.upload(r)
            d.numPts = len(r)
            datas.append(d)
        assert min(d.numPts for d in datas) > 200
        pairs = [(a, b) for a in range(8) for b in range(a + 1, 8)]
        ratio, _, _ = cs.MatchSiftDataRatioBatch(datas, pairs)
        offsets, members, _, _, _ = cs.BuildTracks([d.numPts for d in datas],
                                                   [(a, b, p) for (a, b), p in zip(pairs, ratio)])
        pts, cnt, err, inlier, stats, _ = cs.TriangulateTracks(datas, Ks, Rs, ts, offsets, members)
        recs = [d._buf.download(cs.SIFT_DTYPE, d.numPts) for d in datas]
    finally:
        for d in datas:
            cs.FreeSiftData(d)
    good = np.isfinite(pts[:, 0])
    assert good.sum() > 300, good.sum()
    # the records against the projections of their tracks' points under the true cameras
    res = []
    for k in np.nonzero(good)[0]:
        for m in range(offsets[k], offsets[k + 1]):
            if not inlier[m]:
                continue
            a, f = members[m]
            u = Ks[a] @ (Rs[a] @ pts[k] + ts[a])
            res.append(u[:2] / u[2] - (recs[a]["xpos"][f], recs[a]["ypos"][f]))
    res = np.array(res)
    print("end to end: %d points, %d inlier observations, median reprojection error %.3f px, mean residual %s" %
          (good.sum(), len(res), np.median(np.hypot(*res.T)), res.mean(0)))
    assert np.median(np.hypot(*res.T)) <= 1.0 and np.all(np.abs(res.mean(0)) <= 0.15)

    jobs = cs.SelectStereoViews(Ks, Rs, ts, offsets, members, pts)
    assert sorted(j[0] for j in jobs) == list(range(8))
    d, n, c, _, _ = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs)
    for p, (a, sources, lo, hi) in enumerate(jobs):
        frac, med = accuracy(views, Ks, Rs, ts, a, list(sources), d[p], n[p])
        print("image %d: depth range %.2f..%.2f, %.3f within 1 %%, median normal error %.1f deg" % (a, lo, hi, frac,
                                                                                                   med))
        assert frac >= DEPTH_FRACTION and med <= NORMAL_MEDIAN_DEG
    xyz, _, _, src, total, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, d, n, c)
    sceneDepth = max(float(v[1][np.isfinite(v[1])].max()) for v in views)
    z = np.array([Rs[a][2] @ xyz[k] + ts[a][2] for k, (a, _) in enumerate(src)])
    zt = np.array([views[a][1].reshape(-1)[p] for a, p in src])
    near = np.mean(np.abs(z - zt) <= 0.005 * sceneDepth)
    print("end to end fusion: %d points, %.3f within 0.5 %% of the scene depth" % (total, near))
    assert total > 0 and near >= 0.95
