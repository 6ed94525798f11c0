"""CPU checks of PatchMatch stereo with geometric consistency (cs_patch_match_stereo_geometric): the photometric
kernels are the parent's instruction for instruction, the oracle's geometric error is near 0 on rendered truth, what
the term does to one map is measured on the oracle, and every documented CS_E_ARG is returned naming its argument,
the overlap of an output with a prior included (with no device present)."""
import ctypes
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import stereo_cases as sc
import stereo_geom_oracle as sg
import stereo_oracle as so
from cudasift_b200 import build
from test_arg_ranges_cpu import BASE, MSG, _buf, _layout, _share
from test_bundle_intrinsics_cpu import _sass
from test_stereo_cpu import CS_E_ARG, DEPTH_FRACTION, NORMAL_MEDIAN_DEG, Scene, _rejects, accuracy

# ---- the photometric and fusion kernels are the parent's, instruction for instruction ----

# sha256 of the normalised `cuobjdump -sass` of stereo.o's kernels before the geometric pass was added, from nvcc 12.9
# (V12.9.86) with the library's flags.
SASS = {"pm_start_kernel": "58e9c533943825c3b4003913356e51154e32bad79750c3d2bfe6268bd11a52d3",
        "pm_half_kernel": "96b2db22a46d16692acf42e616689977c1efc705de16d650d7b8e0e2cc2febe8",
        "pm_final_kernel": "46ede5052409921831dd344b2402e91fe6a0ed903463f585fd27ea9e32fa64fd",
        "fuse_flags_kernel": "60976be97a1067aa834f685ba2625c628ffc6dc43f7c1b6bff5e8bbc60f46116",
        "fuse_write_kernel": "82af28748beffdfd4928efd4fea22ebd2ca8a1e7a7d1bdd7995e9a500ce2f487"}


def test_photometric_kernels_are_unchanged():
    nvcc = build.nvcc_path()
    if nvcc is None or "V12.9.86" not in subprocess.run([nvcc, "--version"], stdout=subprocess.PIPE,
                                                        text=True).stdout:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    build.build_library()
    fs = _sass(os.path.join(build.OBJDIR, "stereo.o"))
    for name, digest in SASS.items():
        key = [f for f in fs if re.search(r"\d+%sE" % name, f)]
        assert len(key) == 1, (name, sorted(fs))
        assert hashlib.sha256("\n".join(fs[key[0]]).encode()).hexdigest() == digest, name
    assert any(re.search(r"\d+pm_geom_half_kernelE", f) for f in fs)


# ---- the oracle's geometric error ----

def _truth_priors(views, n):
    """Every view's true depth (0 where the ray misses) and normal as its prior."""
    return {a: (np.where(np.isfinite(views[a][1]), views[a][1], 0.0).astype(np.float32),
                views[a][2].astype(np.float32)) for a in range(n)}


@pytest.mark.parametrize("size", [(160, 120), (640, 480)])
def test_geometric_error_on_rendered_truth(size):
    W, H = size
    Ks, Rs, ts, views = sc.render(6, W, H, seed=1)
    priors = _truth_priors(views, 6)
    job = sg.GeomJob(Ks, Rs, ts, 2, [1, 3, 0], 3.0, 12.0)
    y, x = [a.reshape(-1) for a in np.mgrid[0:H, 0:W]]
    z = priors[2][0].reshape(-1)
    hit = z > 0
    for k, s in enumerate(job.sources):
        g, capped, _ = sg.geom_error(job, k, priors[s][0], x[hit], y[hit], z[hit], 3.0)
        vis = sc.visible_in(views, Ks, Rs, ts, 2, s).reshape(-1)[hit]
        med, below = float(np.median(g[vis])), float(np.mean(g[vis] < 0.5))
        print("%dx%d source %d: median g %.3f px, %.4f below 0.5 px" % (W, H, s, med, below))
        assert med < 0.05 and below >= 0.99, (s, med, below)
    # gmax where the prior is 0, NaN or missing
    for bad in (0.0, np.nan):
        d = np.full_like(priors[1][0], bad)
        g, capped, _ = sg.geom_error(job, 0, d, x[hit], y[hit], z[hit], 3.0)
        assert np.all(g == 3.0) and np.all(capped)
    g, capped, _ = sg.geom_error(job, 0, None, x[hit], y[hit], z[hit], 2.5)
    assert np.all(g == 2.5) and np.all(capped)


def test_zero_weight_is_the_photometric_cost():
    Ks, Rs, ts, views = sc.render(4, 64, 48, seed=1)
    images = [v[0] for v in views]
    priors = _truth_priors(views, 4)
    job = sg.GeomJob(Ks, Rs, ts, 2, [1, 3, 0], 3.0, 12.0)
    y, x = [a.reshape(-1) for a in np.mgrid[0:48, 0:64]]
    z, n = so.random_hyp(4, job, 64, x, y, 0, 0)
    c0, inv0, m0 = so.cost(images, job, x, y, z, n, 3, 1, 2)
    c, inv, cap, m = sg.cost(images, job, {a: p[0] for a, p in priors.items()}, x, y, z, n, 3, 1, 2, 0.0, 3.0)
    assert np.array_equal(c, c0) and np.array_equal(inv, inv0)
    assert np.all(cap <= 3 - inv)
    # the start takes a valid prior bit for bit, and draws at iteration 32 elsewhere
    pd, pn = priors[2][0].copy(), priors[2][1].copy()
    pd[0, :5] = [np.nan, 0.0, 50.0, 5.0, 5.0]
    pn[0, 3] = -pn[0, 3]
    pn[0, 4] *= 1.01
    take = sg.start_rule(job, pd, pn, x, y).reshape(48, 64)
    assert not take[0, :5].any() and take[pd > 0].mean() > 0.9


# ---- what the term does to one map ----

# 160 x 120, r = 3, topK = 2: 3 photometric iterations on ref 2 and on each of its sources [1, 3, 0] (each with its 3
# nearest views), then 3 more on ref 2 from its photometric map with the sources' photometric maps as priors, under
# the header's rule (an invalid view costs 2 + lambda g).  The oracle gave (fraction of the pixels seen by >= 2 sources
# within 1 % depth error, median normal error, fraction of pixels with g <= 1 px in >= 2 sources):
#   photometric, 3 iterations:          0.655, 24.0 deg, 0.666
#   lambda = 0 (3 more, photometric):   0.790,  6.2 deg, 0.682
#   lambda = 0.3 (COLMAP's default):    0.795, 10.2 deg, 0.741
# The term raises the agreement between the maps, which is what fusion counts.  It does not make one map more accurate
# than further photometric iterations do, and the median normal gets worse.  The normal error follows lambda: 6.2, 8.3,
# 10.2 and 12.2 degrees at lambda = 0, 0.1, 0.3 and 1 (gmax 3), and 10.1 and 10.2 degrees at gmax 1 and 10 (lambda 0.3).
# It is there on the pixels whose depth is within 1 % too (4.5 degrees at lambda 0, 8.4 at 0.3).  g depends on the
# depth alone (X = z ray), so the term cannot tell normals apart: it lowers the weight of the photometric cost, the only
# part that can, and a candidate that brings the depth toward the sources' maps wins with whatever normal it carries.
def _nearest(a, n=6, k=3):
    return [b for b in np.argsort([abs(b - a) for b in range(n)], kind="stable") if b != a][:k]


def test_geometric_pass_on_one_map():
    Ks, Rs, ts, views = sc.render(6, 160, 120, seed=1)
    images = [v[0] for v in views]
    ref, sources = 2, [1, 3, 0]
    photo = {}
    for a in [ref] + sources:
        photo[a] = so.run(images, so.Job(Ks, Rs, ts, a, _nearest(a), 3.0, 12.0), 0, 3, 1, 3, 2)
    priors = {a: (photo[a][0], photo[a][1]) if a in photo else None for a in range(6)}
    job = sg.GeomJob(Ks, Rs, ts, ref, sources, 3.0, 12.0)
    rows = {"photometric": photo[ref][:2]}
    for lam in (0.0, 0.3):
        rows[lam] = sg.run(images, job, priors, 0, 3, 1, 3, 2, lam, 3.0)[:2]
    res = {}
    for key, (d, n) in rows.items():
        frac, med = accuracy(views, Ks, Rs, ts, ref, sources, d, n)
        res[key] = (frac, med, sg.consistency(job, priors, d))
        print("%s: %.3f within 1 %%, median normal error %.1f deg, consistency %.3f" % ((key,) + res[key]))
    assert res[0.3][0] >= DEPTH_FRACTION and res[0.3][1] <= NORMAL_MEDIAN_DEG, res[0.3]


# ---- argument checks ----

class GeomScene(Scene):
    def __init__(self, n=3, w=64, h=48):
        super().__init__(n, w, h)
        self.priors = (cs.DepthPrior * n)(*[cs.DepthPrior(0xA0000000 + 0x1000000 * (2 * a),
                                                          0xA0000000 + 0x1000000 * (2 * a + 1)) for a in range(n)])

    def geo(self, r=3, step=1, iters=2, topK=2, lam=0.3, gmax=3.0, priors=True, numJobs=None):
        return cs.lib().cs_patch_match_stereo_geometric(self.images, self.n, self.Ks.ctypes.data, self.Rs.ctypes.data,
                                                        self.ts.ctypes.data, self.priors if priors else None,
                                                        self.jobs, self.n if numJobs is None else numJobs, r, step,
                                                        iters, topK, lam, gmax, 0, None, None)


def test_geometric_argument_checks():
    s = GeomScene()
    _rejects(s.geo(iters=32), "numIterations must be in [0, 31]")
    _rejects(s.geo(iters=-1), "numIterations")
    _rejects(s.geo(r=0), "windowRadius")
    _rejects(s.geo(r=3, step=2), "windowStep")
    _rejects(s.geo(topK=3), "jobs[0]", "topK")
    _rejects(s.geo(priors=False), "priors")
    assert s.geo(priors=False, numJobs=0) == 0
    _rejects(s.geo(lam=-0.1), "geomWeight")
    _rejects(s.geo(lam=float("inf")), "geomWeight")
    _rejects(s.geo(gmax=0.0), "geomMaxError")
    _rejects(s.geo(gmax=float("nan")), "geomMaxError")
    s.priors[1].d_depth = None
    _rejects(s.geo(), "jobs[1]", "priors[1]")
    s = GeomScene()
    s.priors[2].d_normal = None
    _rejects(s.geo(), "jobs[2]", "priors[2]")
    s = GeomScene()
    s.priors[0].d_normal = 0xA0000002
    _rejects(s.geo(), "priors[0]", "aligned")
    s = GeomScene()
    s.jobs[1].d_cost = None
    _rejects(s.geo(), "jobs[1]", "d_cost")
    s = GeomScene()
    s.ts[0, 1] = np.nan
    _rejects(s.geo(), "ts[0]")


def test_output_overlapping_a_prior_is_rejected_and_named():
    s = GeomScene()
    s.priors[0].d_depth = s.jobs[1].d_normal + 4
    _rejects(s.geo(), "jobs[1].d_normal and priors[0].d_depth overlap")
    s = GeomScene()
    s.priors[2].d_normal = s.jobs[2].d_depth
    _rejects(s.geo(), "jobs[2].d_depth and priors[2].d_normal overlap")


def _geom_layout(rng):
    """Ranges of one geometric call over random images, jobs and priors: (sizes, forbidden, make).  Every ref has a
    prior; another image has one or not."""
    I = int(rng.integers(2, 4))
    dims = [(int(rng.integers(2, 6)), int(rng.integers(2, 5))) for _ in range(I)]
    pitch = [w + int(rng.integers(0, 3)) for w, _ in dims]
    sizes = {"images[%d].d_img" % a: 4 * ((h - 1) * pitch[a] + w) for a, (w, h) in enumerate(dims)}
    J = int(rng.integers(1, I + 1))
    refs = [int(v) for v in rng.permutation(I)[:J]]
    maps = ["d_depth", "d_normal", "d_cost"]
    for p, a in enumerate(refs):
        w, h = dims[a]
        for k, m in enumerate(maps):
            sizes["jobs[%d].%s" % (p, m)] = 4 * w * h * (3 if k == 1 else 1)
    written = set(sizes) - {"images[%d].d_img" % a for a in range(I)}
    has = [a in refs or rng.random() < 0.5 for a in range(I)]
    for a, (w, h) in enumerate(dims):
        if has[a]:
            sizes["priors[%d].d_depth" % a], sizes["priors[%d].d_normal" % a] = 4 * w * h, 12 * w * h
    Ks = np.ascontiguousarray(np.stack([np.array([[80.0, 0.5, 32], [0, 82, 24], [0, 0, 1]])] * I))
    Rs = np.ascontiguousarray(np.stack([np.eye(3)] * I))
    ts = np.zeros((I, 3))
    srcs = [np.array([b for b in range(I) if b != a], np.int32) for a in refs]

    def make(at):
        ims = (cs.StereoImage * I)(*[cs.StereoImage(at["images[%d].d_img" % a], w, h, pitch[a])
                                    for a, (w, h) in enumerate(dims)])
        pri = (cs.DepthPrior * I)(*[cs.DepthPrior(at["priors[%d].d_depth" % a], at["priors[%d].d_normal" % a])
                                    if has[a] else cs.DepthPrior(None, None) for a in range(I)])
        jt = (cs.StereoJob * J)(*[cs.StereoJob(a, srcs[p].ctypes.data, I - 1, 1.0, 5.0,
                                               *[at["jobs[%d].%s" % (p, m)] for m in maps])
                                  for p, a in enumerate(refs)])
        return cs.lib().cs_patch_match_stereo_geometric(ims, I, Ks.ctypes.data, Rs.ctypes.data, ts.ctypes.data, pri,
                                                        jt, J, 1, 1, 1, 1, 0.3, 3.0, 0, None, None)

    return sizes, (lambda a, b: a in written or b in written), make


def test_every_geometric_overlap_is_rejected_and_named():
    rng = np.random.default_rng(1732)
    for _ in range(200):
        sizes, forbidden, make = _geom_layout(rng)
        at = _layout(rng, sizes, forbidden)
        r = make({x: BASE + v for x, v in at.items()})
        msg = cs.lib().cs_last_error().decode()
        assert r == CS_E_ARG, (r, msg)
        m = MSG.match(msg)
        assert m, msg
        _, a, b = m.groups()
        assert a in sizes and b in sizes, (msg, sorted(sizes))
        assert forbidden(a, b) and _share((at[a], sizes[a]), (at[b], sizes[b])), (msg, at, sizes)
    assert not _buf.any()
