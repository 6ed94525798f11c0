"""CPU checks of dense reconstruction: the oracle's full PatchMatch loop reaches the accuracy bounds the GPU test uses,
SelectStereoViews picks the expected neighbours and ranges, every documented CS_E_ARG of cs_undistort_images,
cs_patch_match_stereo and cs_fuse_depth_maps is returned naming its argument, and every forbidden overlap is rejected
and named (with no device present)."""
import ctypes

import numpy as np
import pytest

import cudasift_b200 as cs
import stereo_cases as sc
import stereo_oracle as so
from test_arg_ranges_cpu import BASE, MSG, _buf, _layout, _share

CS_E_ARG = -2
# Accuracy bounds of the GPU test at 640 x 480 with the defaults.  test_oracle_loop_reaches_the_bounds at 160 x 120
# (r = 3, 3 iterations) gave 0.66 of the pixels seen by two or more sources within 1 % depth error and a median normal
# error of 24 degrees; the GPU at 640 x 480 with the defaults gave 0.53 and 29 degrees on an H100 (random starts
# propagate over more pixels there in the same 5 iterations).  The bounds leave a margin below both runs.
DEPTH_FRACTION = 0.45
NORMAL_MEDIAN_DEG = 35.0


def accuracy(views, Ks, Rs, ts, a, sources, depth, normal):
    """(fraction of the pixels seen by >= 2 sources within 1 % depth error, median normal error in degrees)."""
    vis = sum(sc.visible_in(views, Ks, Rs, ts, a, b) for b in sources) >= 2
    with np.errstate(invalid="ignore"):               # infinite true depth where the ray misses the scene
        err = np.abs(depth - views[a][1]) / views[a][1]
    ang = np.degrees(np.arccos(np.clip(np.sum(normal * views[a][2], -1), -1, 1)))
    return float((err[vis] <= 0.01).mean()), float(np.median(ang[vis]))


def test_oracle_loop_reaches_the_bounds():
    Ks, Rs, ts, views = sc.render(6, 160, 120, seed=1)
    job = so.Job(Ks, Rs, ts, 2, [1, 3, 0, 4], 3.0, 12.0)
    d, n, c = so.run([v[0] for v in views], job, 0, 3, 1, 3, 2)
    frac, med = accuracy(views, Ks, Rs, ts, 2, [1, 3, 0, 4], d, n)
    assert frac >= DEPTH_FRACTION + 0.15 and med <= NORMAL_MEDIAN_DEG - 8, (frac, med)
    assert np.all(np.isfinite(d)) and np.all((c >= 0) & (c <= 2))


def test_draws_and_hypotheses_follow_the_header():
    u = so.draw(7, 3, np.arange(100), 0, 1)
    assert np.all((u >= 0) & (u < 1)) and len(np.unique(u)) == 100
    # the counter family: ((ref 2^24 + pix) 64 + it) 16 + slot
    assert so.draw(7, 0, 1, 0, 0) == so.draw(7, 0, 0, 64, 0) and so.draw(7, 0, 0, 0, 16) == so.draw(7, 0, 0, 1, 0)
    Ks, Rs, ts = sc.cameras(3, 64, 48)
    job = so.Job(Ks, Rs, ts, 0, [1, 2], 2.0, 9.0)
    y, x = [a.reshape(-1) for a in np.mgrid[0:48, 0:64]]
    z, n = so.random_hyp(5, job, 64, x, y, 0, 0)
    assert np.all((z >= 2.0) & (z <= 9.0))
    assert np.all(np.sum(n * so.rays(job, x, y), -1) < 0)
    assert np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-6)


def test_select_stereo_views_on_a_known_layout():
    # 4 cameras on a line looking down +z; tracks seen by chosen image sets
    Ks = np.array([[100.0, 0, 50], [0, 100, 40], [0, 0, 1]])
    Rs = np.stack([np.eye(3)] * 4)
    ts = np.array([[-a * 1.0, 0, 0] for a in range(4)])       # centres at x = a
    pts, groups = [], []
    rng = np.random.default_rng(0)
    spec = [((0, 1), 5), ((0, 2), 3), ((1, 2), 4), ((2, 3), 2), ((0, 3), 3)]
    for imgs, k in spec:
        for _ in range(k):
            pts.append([1.5 + rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.uniform(8, 12)])
            groups.append(imgs)
    pts.append([1.0, 0.0, 1e4])                                 # seen by 0 and 1 at a tiny angle: not counted
    groups.append((0, 1))
    pts.append([np.nan] * 3)                                     # no point
    groups.append((1, 3))
    offsets = np.concatenate([[0], np.cumsum([len(g) for g in groups])])
    members = np.array([[a, k] for k, g in enumerate(groups) for a in g])
    jobs = cs.SelectStereoViews(Ks, Rs, ts, offsets, members, np.array(pts), numSources=2, minTriAngle=1.0)
    got = {a: list(s) for a, s, _, _ in jobs}
    assert got == {0: [1, 2], 1: [0, 2], 2: [1, 0], 3: [0, 2]}, got
    for a, _, lo, hi in jobs:
        z = np.array([p[2] for p, g in zip(pts, groups) if a in g and np.isfinite(p[2])])
        assert lo == pytest.approx(0.75 * np.percentile(z, 1)) and hi == pytest.approx(1.25 * np.percentile(z, 99))


# ---- argument checks -------------------------------------------------------------------------------------------------

K = np.array([[80.0, 0.5, 32], [0, 82, 24], [0, 0, 1]])
R0 = np.eye(3)


class Scene:
    """A call's host arguments over fake (never dereferenced) device addresses."""

    def __init__(self, n=3, w=64, h=48):
        self.n, self.w, self.h = n, w, h
        self.Ks = np.ascontiguousarray(np.stack([K] * n))
        self.Rs = np.ascontiguousarray(np.stack([R0] * n))
        self.ts = np.ascontiguousarray(np.array([[-0.3 * a, 0, 0] for a in range(n)]))
        self.images = (cs.StereoImage * n)(*[cs.StereoImage(0x10000000 * (a + 1), w, h, w) for a in range(n)])
        self.src = [np.array([b for b in range(n) if b != a], np.int32) for a in range(n)]
        self.jobs = (cs.StereoJob * n)(*[cs.StereoJob(a, self.src[a].ctypes.data, n - 1, 2.0, 9.0,
                                                       0x80000000 + 0x1000000 * (3 * a), 0x80000000 + 0x1000000 * (3 * a + 1),
                                                       0x80000000 + 0x1000000 * (3 * a + 2)) for a in range(n)])

    def pm(self, r=3, step=1, iters=2, topK=2, n=None, jobs=None, numJobs=None):
        return cs.lib().cs_patch_match_stereo(self.images, self.n if n is None else n, self.Ks.ctypes.data,
                                              self.Rs.ctypes.data, self.ts.ctypes.data,
                                              self.jobs if jobs is None else jobs,
                                              self.n if numJobs is None else numJobs, r, step, iters, topK, 0, None,
                                              None)

    def fuse(self, maxCost=0.5, minC=2, rep=2.0, dep=0.01, nrm=10.0, maxPoints=0, outs=(None,) * 4):
        return cs.lib().cs_fuse_depth_maps(self.images, self.n, self.Ks.ctypes.data, self.Rs.ctypes.data,
                                           self.ts.ctypes.data, self.jobs, self.n, maxCost, minC, rep, dep, nrm,
                                           *outs, maxPoints, None, None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    for w in words:
        assert w in msg, (w, msg)


def test_patch_match_argument_checks():
    s = Scene()
    _rejects(s.pm(r=0), "windowRadius")
    _rejects(s.pm(r=8), "windowRadius")
    _rejects(s.pm(r=3, step=2), "windowStep")
    _rejects(s.pm(r=2, step=3), "windowStep")
    _rejects(s.pm(iters=33), "numIterations")
    _rejects(s.pm(topK=0), "topK")
    _rejects(s.pm(topK=3), "jobs[0]", "topK")
    _rejects(s.pm(n=0), "numImages")
    _rejects(s.pm(numJobs=-1), "numJobs")
    s.images[1].width = 1
    _rejects(s.pm(), "images[1]", "width")
    s = Scene()
    s.images[2].pitch = 10
    _rejects(s.pm(), "images[2]", "pitch")
    s = Scene()
    s.images[0].d_img = None
    _rejects(s.pm(), "images[0].d_img")
    s = Scene()
    s.Ks[1, 2, 2] = 2.0
    _rejects(s.pm(), "Ks[1]")
    s = Scene()
    s.Rs[2] *= 2
    _rejects(s.pm(), "Rs[2]")
    s = Scene()
    s.ts[0, 1] = np.nan
    _rejects(s.pm(), "ts[0]")
    for field, value, words in [("ref", 5, ("jobs[1]", "ref")), ("numSources", 0, ("jobs[1]", "numSources")),
                                ("numSources", 33, ("jobs[1]", "numSources")), ("sources", None, ("jobs[1]", "sources")),
                                ("depthMin", 0.0, ("jobs[1]", "depthMin")), ("depthMax", 1.0, ("jobs[1]", "depthMin")),
                                ("depthMax", float("inf"), ("jobs[1]", "depthMax")),
                                ("d_cost", None, ("jobs[1]", "d_cost")), ("d_depth", 0x80000002, ("jobs[1]", "aligned"))]:
        s = Scene()
        setattr(s.jobs[1], field, value)
        _rejects(s.pm(), *words)
    s = Scene()
    s.jobs[2].ref = 0
    _rejects(s.pm(), "jobs[2]", "already the ref of jobs[0]")
    s = Scene()
    s.src[1][0] = 1
    _rejects(s.pm(), "jobs[1]", "sources[0]")
    s = Scene()
    s.src[1][1] = s.src[1][0]
    _rejects(s.pm(), "jobs[1]", "sources[1] repeats sources[0]")


def test_fuse_and_undistort_argument_checks():
    s = Scene()
    _rejects(s.fuse(maxCost=2.5), "maxCost")
    _rejects(s.fuse(minC=0), "minConsistent")
    _rejects(s.fuse(rep=0.0), "maxReprojError")
    _rejects(s.fuse(dep=float("nan")), "maxDepthError")
    _rejects(s.fuse(nrm=181.0), "maxNormalErrorDeg")
    _rejects(s.fuse(maxPoints=-1), "maxPoints")
    _rejects(s.fuse(maxPoints=4), "d_xyz")
    _rejects(s.fuse(maxPoints=4, outs=(0x1000, 0x2000, 0x3000, 0x4004)), "d_source")
    s.jobs[0].numSources = 0
    _rejects(s.fuse(), "jobs[0]", "numSources")
    L = cs.lib()
    s = Scene()
    outs = (ctypes.c_void_p * 3)(0x90000000, 0x91000000, 0x92000000)
    dists = np.zeros((3, 2))
    _rejects(L.cs_undistort_images(s.images, -1, s.Ks.ctypes.data, None, outs, None, None), "numImages")
    _rejects(L.cs_undistort_images(s.images, 3, s.Ks.ctypes.data, None, None, None, None), "d_out")
    dists[2, 1] = np.inf
    _rejects(L.cs_undistort_images(s.images, 3, s.Ks.ctypes.data, dists.ctypes.data, outs, None, None), "dists[2]")
    outs[1] = 0x91000002
    _rejects(L.cs_undistort_images(s.images, 3, s.Ks.ctypes.data, None, outs, None, None), "d_out[1]")
    s.Ks[0, 0, 0] = -1
    outs[1] = 0x91000000
    _rejects(L.cs_undistort_images(s.images, 3, s.Ks.ctypes.data, None, outs, None, None), "Ks[0]")
    assert L.cs_undistort_images(None, 0, None, None, None, None, None) == 0


# ---- overlaps --------------------------------------------------------------------------------------------------------

def _stereo_layout(rng, call):
    """Ranges of one dense call over random images and jobs: (sizes, forbidden, make)."""
    I = int(rng.integers(2, 4))
    dims = [(int(rng.integers(2, 6)), int(rng.integers(2, 5))) for _ in range(I)]
    pitch = [w + int(rng.integers(0, 3)) for w, _ in dims]
    sizes = {"images[%d].d_img" % a: 4 * ((h - 1) * pitch[a] + w) for a, (w, h) in enumerate(dims)}
    J = int(rng.integers(1, I + 1)) if call != "undistort" else 0
    refs = [int(v) for v in rng.permutation(I)[:J]]
    maps = ["d_depth", "d_normal", "d_cost"]
    for p, a in enumerate(refs):
        w, h = dims[a]
        for k, m in enumerate(maps):
            sizes["jobs[%d].%s" % (p, m)] = 4 * w * h * (3 if k == 1 else 1)
    if call == "undistort":
        outs = ["d_out[%d]" % a for a in range(I)]
        for a, (w, h) in enumerate(dims):
            sizes[outs[a]] = 4 * w * h
    elif call == "fuse":
        P = int(rng.integers(1, 6))
        outs = ["d_xyz", "d_normal", "d_intensity", "d_source"]
        sizes.update(d_xyz=12 * P, d_normal=12 * P, d_intensity=4 * P, d_source=8 * P)
    else:
        outs = [x for x in sizes if x.startswith("jobs[")]
    written = set(outs)
    Ks = np.ascontiguousarray(np.stack([K] * I))
    Rs = np.ascontiguousarray(np.stack([R0] * I))
    ts = np.zeros((I, 3))
    srcs = [np.array([b for b in range(I) if b != a], np.int32) for a in refs]

    def make(at):
        ims = (cs.StereoImage * I)(*[cs.StereoImage(at["images[%d].d_img" % a], w, h, pitch[a])
                                    for a, (w, h) in enumerate(dims)])
        L = cs.lib()
        if call == "undistort":
            o = (ctypes.c_void_p * I)(*[at["d_out[%d]" % a] for a in range(I)])
            return L.cs_undistort_images(ims, I, Ks.ctypes.data, None, o, None, None)
        jt = (cs.StereoJob * J)(*[cs.StereoJob(a, srcs[p].ctypes.data, I - 1, 1.0, 5.0,
                                               *[at["jobs[%d].%s" % (p, m)] for m in maps])
                                  for p, a in enumerate(refs)])
        if call == "fuse":
            return L.cs_fuse_depth_maps(ims, I, Ks.ctypes.data, Rs.ctypes.data, ts.ctypes.data, jt, J, 0.5, 1, 2.0,
                                        0.01, 10.0, *[at[x] for x in outs], sizes["d_source"] // 8, None, None)
        return L.cs_patch_match_stereo(ims, I, Ks.ctypes.data, Rs.ctypes.data, ts.ctypes.data, jt, J, 1, 1, 1, 1, 0,
                                       None, None)

    return sizes, (lambda a, b: a in written or b in written), make


@pytest.mark.parametrize("call", ["undistort", "patch_match", "fuse"])
def test_every_stereo_overlap_is_rejected_and_named(call):
    rng = np.random.default_rng(sum(map(ord, call)))
    for _ in range(200):
        sizes, forbidden, make = _stereo_layout(rng, call)
        at = _layout(rng, sizes, forbidden)
        # 4-byte alignment is what the dense calls ask of every buffer but d_source
        r = make({x: BASE + v for x, v in at.items()})
        msg = cs.lib().cs_last_error().decode()
        assert r == CS_E_ARG, (call, r, msg)
        m = MSG.match(msg)
        assert m, (call, msg)
        _, a, b = m.groups()
        assert a in sizes and b in sizes, (call, msg, sorted(sizes))
        assert forbidden(a, b) and _share((at[a], sizes[a]), (at[b], sizes[b])), (call, msg, at, sizes)
    assert not _buf.any()
