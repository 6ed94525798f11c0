"""GPU checks of PatchMatch stereo with geometric consistency (cs_patch_match_stereo_geometric) against
tests/stereo_geom_oracle.py: the start from the priors, the cost at every pixel, every half-step replayed, accuracy
and cross-map consistency at 640 x 480, fusion on library outputs, determinism, batching and launches."""
import ctypes

import numpy as np
import pytest

import cudasift_b200 as cs
import stereo_cases as sc
import stereo_geom_oracle as sg
import stereo_oracle as so
from test_stereo_cpu import DEPTH_FRACTION, NORMAL_MEDIAN_DEG, accuracy

pytestmark = pytest.mark.gpu

COST_BOUND = 2e-3          # the header's FP32 bound on a view cost; g is float64 rounded once, so it holds for the sum
R, STEP, TOPK, SEED = 3, 1, 2, 3


@pytest.fixture(scope="module")
def small():
    Ks, Rs, ts, views = sc.render(6, 160, 120, seed=1)
    images = [v[0] for v in views]
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(6)]) if b != a][:4], 3.0, 12.0) for a in range(6)]
    photo = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs, windowRadius=R, windowStep=STEP, numIterations=2, topK=TOPK,
                                seed=SEED)
    return Ks, Rs, ts, views, images, jobs, photo


def _geo(small, n, lam=0.3, gmax=3.0, depth=None, normal=None):
    Ks, Rs, ts, _, images, jobs, photo = small
    return cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, photo[0] if depth is None else depth,
                                        photo[1] if normal is None else normal, windowRadius=R, windowStep=STEP,
                                        numIterations=n, topK=TOPK, geomWeight=lam, geomMaxError=gmax, seed=SEED)


def _job(small, p):
    Ks, Rs, ts, _, _, jobs, _ = small
    a, s, lo, hi = jobs[p]
    return sg.GeomJob(Ks, Rs, ts, a, s, lo, hi)


def _priors(jobs, depth, normal):
    return {int(j[0]): (depth[p], normal[p]) for p, j in enumerate(jobs)}


def _grid(H, W):
    return [v.reshape(-1) for v in np.mgrid[0:H, 0:W]]


def test_zero_weight_and_no_iterations(small):
    """lambda = 0, 0 iterations: every prior that the start rule takes comes back as its bytes, and the cost is the
    photometric call's, bit for bit (the two cost functions share st_view_cost and fmaf(0, g, c) = c)."""
    Ks, Rs, ts, _, images, jobs, photo = small
    d, n, c, stats, _ = _geo(small, 0, lam=0.0)
    for p in range(len(jobs)):
        job = _job(small, p)
        H, W = d[p].shape
        y, x = _grid(H, W)
        take = sg.start_rule(job, photo[0][p], photo[1][p], x, y).reshape(H, W)
        assert stats[p, 4] == int((~take).sum())
        assert d[p][take].tobytes() == photo[0][p][take].tobytes()
        assert n[p][take].tobytes() == photo[1][p][take].tobytes()
        assert c[p][take].tobytes() == photo[2][p][take].tobytes()
        assert stats[p, 0] == H * W and stats[p, 2] == int((c[p] >= 2).sum())
    print("pixels started from a draw:", stats[:, 4].tolist())


def test_start_rule(small):
    Ks, Rs, ts, _, images, jobs, photo = small
    depth, normal = [a.copy() for a in photo[0]], [a.copy() for a in photo[1]]
    p = 2
    job = _job(small, p)
    poison = [(5, 7), (5, 8), (5, 9), (60, 80), (119, 159)]
    depth[p][5, 7] = np.nan
    depth[p][5, 8] = 0.0
    depth[p][5, 9] = 2 * job.dmax
    normal[p][60, 80] = -normal[p][60, 80]
    normal[p][119, 159] *= 1.01
    d, n, c, stats, _ = _geo(small, 0, depth=depth, normal=normal)
    H, W = d[p].shape
    y, x = _grid(H, W)
    take = sg.start_rule(job, depth[p], normal[p], x, y)
    for yy, xx in poison:
        assert not take[yy * W + xx]
    z, nn = so.random_hyp(SEED, job, W, x, y, sg.IT0, 0)
    drawn = ~take
    assert stats[p, 4] == int(drawn.sum())
    assert np.all(np.abs(d[p].reshape(-1)[drawn] - z[drawn]) <= np.spacing(z[drawn]))
    assert np.all(np.abs(n[p].reshape(-1, 3)[drawn] - nn[drawn]) <= np.spacing(np.abs(nn[drawn])) + 1e-12)
    assert d[p].reshape(-1)[take].tobytes() == depth[p].reshape(-1)[take].tobytes()
    # the start's costs and counts against the oracle
    pri = {a: v[0] for a, v in _priors(jobs, depth, normal).items()}
    oc, inv, cap, mar = sg.cost(images, job, pri, x, y, d[p].reshape(-1), n[p].reshape(-1, 3), R, STEP, TOPK, 0.3, 3.0)
    assert mar.mean() < 0.01 and np.all(np.abs(oc - c[p].reshape(-1))[~mar] <= COST_BOUND)
    assert abs(stats[p, 1] - int(inv.sum())) <= int(mar.sum()) * len(job.sources)
    assert abs(stats[p, 3] - int(cap.sum())) <= int(mar.sum()) * len(job.sources)


def test_cost_at_every_pixel(small):
    Ks, Rs, ts, _, images, jobs, photo = small
    d, n, c, stats, _ = _geo(small, 2)
    pri = {a: v[0] for a, v in _priors(jobs, photo[0], photo[1]).items()}
    for p in (1, 4):
        job = _job(small, p)
        H, W = d[p].shape
        y, x = _grid(H, W)
        oc, _, _, mar = sg.cost(images, job, pri, x, y, d[p].reshape(-1), n[p].reshape(-1, 3), R, STEP, TOPK, 0.3, 3.0)
        diff = np.abs(oc - c[p].reshape(-1))
        print("job %d: marginal %.4f, max cost difference %.2e" % (p, mar.mean(), diff[~mar].max()))
        assert mar.mean() < 0.01, mar.mean()
        assert np.all(diff[~mar] <= COST_BOUND), diff[~mar].max()
        assert np.all(np.isfinite(d[p])) and np.all(np.isfinite(n[p]))
        assert stats[p, 2] == int((c[p] >= 2).sum())


def _check_half(small, p, before, after, it, colour):
    _, _, _, _, images, jobs, photo = small
    job = _job(small, p)
    priors = _priors(jobs, photo[0], photo[1])
    _, opt = sg.half_step(images, job, priors, before, it, colour, SEED, R, STEP, TOPK, 0.3, 3.0, eps=2 * COST_BOUND)
    x, y = opt["x"], opt["y"]
    gz, gn = after[0][y, x], after[1][y, x]
    same = (np.abs(opt["z"] - gz[None]) <= 1e-5 * np.abs(gz[None])) & \
        np.all(np.abs(opt["n"] - gn[None]) <= 1e-5, axis=-1)
    ok = np.any(same & opt["admissible"], axis=0)
    marginal = np.any(opt["marginal"] & opt["admissible"], axis=0)
    assert np.all(ok | marginal), (it, colour, int((~ok & ~marginal).sum()))
    return marginal.mean()


def test_every_half_step_replayed(small):
    runs = [_geo(small, n) for n in range(5)]
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


def test_accuracy_and_consistency_at_640x480():
    """8 views, every view a job: 5 photometric iterations, then 5 geometric ones with the defaults and, as the other
    arm, the same call with lambda = 0.  Consistency (the fraction of a map's pixels with g <= 1 px in >= 2 sources,
    against the photometric maps) is what the term optimises and what fusion counts."""
    Ks, Rs, ts, views = sc.render(8, 640, 480, seed=2)
    images = [v[0] for v in views]
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(8)], kind="stable") if b != a], 3.0, 12.0)
            for a in range(8)]
    photo = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs)
    priors = _priors(jobs, photo[0], photo[1])
    arms = {}
    for lam in (0.3, 0.0):
        d, n, c, stats, ms = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, photo[0], photo[1], geomWeight=lam)
        rows = []
        for p, (a, sources, lo, hi) in enumerate(jobs):
            frac, med = accuracy(views, Ks, Rs, ts, a, sources, d[p], n[p])
            cons = sg.consistency(sg.GeomJob(Ks, Rs, ts, a, sources, lo, hi), priors, d[p])
            rows.append((frac, med, cons))
        arms[lam] = np.array(rows)
        print("lambda %.1f, %.1f ms: depth fraction %s, median normal error %s, consistency %s" % (
            lam, ms, np.round(arms[lam][:, 0], 3).tolist(), np.round(arms[lam][:, 1], 1).tolist(),
            np.round(arms[lam][:, 2], 3).tolist()))
    photo_rows = np.array([accuracy(views, Ks, Rs, ts, a, s, photo[0][p], photo[1][p]) for p, (a, s, _, _) in
                           enumerate(jobs)])
    print("photometric: depth fraction %s, median normal error %s" % (np.round(photo_rows[:, 0], 3).tolist(),
                                                                     np.round(photo_rows[:, 1], 1).tolist()))
    g = arms[0.3]
    assert np.all(g[:, 0] >= DEPTH_FRACTION) and np.all(g[:, 1] <= NORMAL_MEDIAN_DEG), g
    assert g[:, 2].mean() > arms[0.0][:, 2].mean(), (g[:, 2], arms[0.0][:, 2])


def test_end_to_end_with_the_geometric_pass():
    """extract -> MatchSiftDataRatioBatch -> BuildTracks -> TriangulateTracks -> SelectStereoViews -> PatchMatchStereo
    -> PatchMatchStereoGeometric -> FuseDepthMaps on the scene of test_end_to_end_on_library_outputs, against the same
    chain with lambda = 0 before fusion."""
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
        pairs = [(a, b) for a in range(8) for b in range(a + 1, 8)]
        ratio, _, _ = cs.MatchSiftDataRatioBatch(datas, pairs)
        offsets, members, _, _, _ = cs.BuildTracks([d.numPts for d in datas],
                                                   [(a, b, p) for (a, b), p in zip(pairs, ratio)])
        pts, _, _, _, _, _ = cs.TriangulateTracks(datas, Ks, Rs, ts, offsets, members)
    finally:
        for d in datas:
            cs.FreeSiftData(d)
    jobs = cs.SelectStereoViews(Ks, Rs, ts, offsets, members, pts)
    assert sorted(j[0] for j in jobs) == list(range(8))
    d, n, c, _, _ = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs)
    sceneDepth = max(float(v[1][np.isfinite(v[1])].max()) for v in views)
    out = {}
    for lam in (0.3, 0.0):
        dg, ng, cg, _, _ = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, d, n, geomWeight=lam)
        for p, (a, sources, _, _) in enumerate(jobs):
            frac, med = accuracy(views, Ks, Rs, ts, a, list(sources), dg[p], ng[p])
            print("lambda %.1f image %d: %.3f within 1 %%, median normal error %.1f deg" % (lam, a, frac, med))
        xyz, _, _, src, total, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, dg, ng, cg)
        z = np.array([Rs[a][2] @ xyz[k] + ts[a][2] for k, (a, _) in enumerate(src)])
        zt = np.array([views[a][1].reshape(-1)[p] for a, p in src])
        out[lam] = (total, float(np.mean(np.abs(z - zt) <= 0.005 * sceneDepth)))
        print("lambda %.1f fusion: %d points, %.3f within 0.5 %% of the scene depth" % ((lam,) + out[lam]))
    assert out[0.3][1] >= 0.95
    assert out[0.3][0] > out[0.0][0], out


def _geometric_raw(images, Ks, Rs, ts, priors, jobs, n, seed):
    """cs_patch_match_stereo_geometric through the C ABI: priors {image: (depth, normal)} for any images, so a subset of
    the jobs can run with every prior.  Returns (depth, normal, cost) lists."""
    S = len(images)
    arrs, bufs, table = cs._upload_images(images)
    maps = []
    try:
        pri = (cs.DepthPrior * S)()
        for a, (pd, pn) in priors.items():
            b = [cs.DeviceBuffer(pd.nbytes), cs.DeviceBuffer(pn.nbytes)]
            bufs += b
            b[0].upload(np.ascontiguousarray(pd, np.float32))
            b[1].upload(np.ascontiguousarray(pn, np.float32))
            pri[a] = cs.DepthPrior(b[0].ptr, b[1].ptr)
        shapes = [im.shape for im in arrs]
        parsed, jt, maps = cs._stereo_jobs(jobs, shapes, lambda p, sh: [cs.DeviceBuffer(4 * sh[0] * sh[1]),
                                                                        cs.DeviceBuffer(12 * sh[0] * sh[1]),
                                                                        cs.DeviceBuffer(4 * sh[0] * sh[1])])
        K, R_, t = (np.ascontiguousarray(np.asarray(v, np.float64)) for v in (Ks, Rs, ts))
        r = cs.lib().cs_patch_match_stereo_geometric(table, S, K.ctypes.data, R_.ctypes.data, t.ctypes.data, pri, jt,
                                                     len(parsed), 2, 1, n, 3, 0.3, 3.0, seed, None, None)
        assert r == 0, cs.lib().cs_last_error()
        res = [[], [], []]
        for (ref, _, _, _), m in zip(parsed, maps):
            h, w = shapes[ref]
            for k, sz in enumerate((h * w, 3 * h * w, h * w)):
                res[k].append(m[k].download(np.float32, sz))
    finally:
        for b in bufs + [b for m in maps for b in m]:
            b.free()
    return res


def test_determinism_batching_and_launches():
    Ks, Rs, ts = sc.cameras(6, 160, 120, seed=1)
    tex = sc._texture()
    S = np.diag([0.8, 0.8, 1.0])
    Ks = np.array([K if a < 3 else S @ K for a, K in enumerate(Ks)])
    images = [sc.cast(Ks[a], Rs[a], ts[a], 160 if a < 3 else 128, 120 if a < 3 else 96, tex=tex)[0] for a in range(6)]
    jobs = [(a, [b for b in range(6) if b != a][:3], 3.0, 12.0) for a in range(6)]
    photo = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs, windowRadius=2, numIterations=2, seed=9)
    L = cs.lib()
    c0 = L.cs_launch_count()
    first = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, photo[0], photo[1], windowRadius=2,
                                         numIterations=3, seed=9)
    assert L.cs_launch_count() - c0 == 2 + 2 * 3
    again = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, photo[0], photo[1], windowRadius=2,
                                         numIterations=3, seed=9)
    for k in range(4):
        for p in range(6):
            assert first[k][p].tobytes() == again[k][p].tobytes()
    for p in range(6):
        assert first[3][p, 2] == int((first[2][p] >= 2).sum())
    # each job alone, with every image's prior, through the C ABI
    priors = _priors(jobs, photo[0], photo[1])
    batch = _geometric_raw(images, Ks, Rs, ts, priors, jobs, 3, 9)
    for k in range(3):
        for p in range(6):
            assert batch[k][p].tobytes() == first[k][p].tobytes(), (p, k)
    for p in range(6):
        alone = _geometric_raw(images, Ks, Rs, ts, priors, [jobs[p]], 3, 9)
        for k in range(3):
            assert alone[k][0].tobytes() == first[k][p].tobytes(), (p, k)
    c0 = L.cs_launch_count()
    cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, photo[0], photo[1], windowRadius=2, numIterations=0)
    assert L.cs_launch_count() - c0 == 2
