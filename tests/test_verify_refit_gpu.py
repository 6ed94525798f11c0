"""GPU checks of step 7 of verification (vp_refit_kernel: the refit, the keep rule, the final mask, the output model and,
for E, the pose) against the float64 restatements (tests/verify_oracle.py, tests/essential_oracle.py).  Each case runs
the models entry point and the verify entry point with the same arguments, takes the device's own winning slot and
normalisation, and restates everything after it in float64: the minimal model's inliers, the refit, the keep rule
(kept unless it has fewer inliers), the returned model, the final inlier list and the pose.  The cases cover both
branches of the keep rule and its tie, the inlier counts where a refit starts (4 for H, 8 for F and E), valid-pair
counts around the kernels' CTA and word sizes with invalid pairs interleaved, badly conditioned scenes, and a batch of
every case against its single calls.

The case generators are plain functions: tests/test_verify_refit_cpu.py checks each case's preconditions without a GPU.

Inlier decisions on the device are FP32 on normalised coordinates, here float64 on pixels: they may differ only for
pairs whose residual lies within BAND of the threshold, and every assertion that compares decisions first asserts that
no pair lies there.  Where the restatement's normal matrix has a clustered spectrum (second-smallest eigenvalue below
CLUSTERED of the largest) its smallest eigenvector is not determined to any useful precision, and the model itself is
not compared: the checks there are the rules applied to the device's own output."""
import ctypes
import functools
import math
from collections import namedtuple

import numpy as np
import pytest

import essential_oracle as eo
import verify_oracle as vo
from test_essential_cpu import K1, K2, calibrated_views
from test_verify_cpu import planted_views

pytestmark = pytest.mark.gpu
W, H_ = 1920, 1080
BAND = 1e-4              # relative half-width of the threshold band where FP32 and float64 decisions may differ
CLUSTERED = 1e-6         # lambda2 / lambda_max below this: the refit's eigenvector is not compared
MODEL_TOL = 1e-9         # kept refit against the restatement's refit (unit Frobenius norm)
SLOT_TOL = 1e-12         # a dropped refit: the winning slot's model, denormalised on the device and on the host
POSE_TOL = 1e-9
NEAR_ZERO = 1e-9         # cheirality quantities this close to zero (relative) could be decided either way
SIZES = (7, 8, 9, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 4097, 262145)
ESSENTIAL = 3            # the kind of an essential case (F and H use vo.FUNDAMENTAL and vo.HOMOGRAPHY)
KINDS = {"F": vo.FUNDAMENTAL, "H": vo.HOMOGRAPHY, "E": ESSENTIAL}
MIN_REFIT = {vo.FUNDAMENTAL: 8, vo.HOMOGRAPHY: 4, ESSENTIAL: 8}
SAMPLE = {vo.FUNDAMENTAL: 7, vo.HOMOGRAPHY: 4, ESSENTIAL: 5}
PER_SAMPLE = {vo.FUNDAMENTAL: 3, vo.HOMOGRAPHY: 3, ESSENTIAL: eo.SLOTS}

# A case: records x1, x2 (float32 [n, 2]), the pair list, the call's arguments, intrinsics (E), the planted model in
# pixels (F or H; E for an essential case), the planted inliers among the pairs (valid, not an outlier) and what the
# case is for:
#   exact     every pair fits exactly: both fits take every pair, the refit ties and is kept
#   drop      the refit has fewer inliers than the minimal model and is dropped
#   tiny      a threshold so small that each slot has only its own sample as inliers
#   clustered the refit's normal matrix has a clustered spectrum
#   whole     the whole call is also restated from scratch (numLoops <= 512)
#   rotation  pure rotation: t is noise, the pose is not compared
Case = namedtuple("Case", "name kind x1 x2 pairs loops thresh seed K1 K2 truth good tags")


# ---- scenes ------------------------------------------------------------------------------------------------------------
def fh_views(n, seed, planar, kind):
    """n exact correspondences inside both 1920x1080 views of planted_views, and the planted model of kind."""
    x1, x2, F, H = planted_views(4 * n + 64, seed, planar)
    inside = (x1 >= 0).all(1) & (x1 < [W, H_]).all(1) & (x2 >= 0).all(1) & (x2 < [W, H_]).all(1)
    x1, x2 = x1[inside][:n], x2[inside][:n]
    assert len(x1) == n
    return x1, x2, (H if kind == vo.HOMOGRAPHY else F)


def e_views(n, seed, motion="sideways", planar=False, Ka=K1, Kb=K2):
    """n exact correspondences of calibrated_views, moved to the intrinsics Ka, Kb (x' = Ka K1^-1 x), and E."""
    x1, x2, _, _, E = calibrated_views(n, seed, motion, planar)
    move = lambda x, Kn, Ko: (np.column_stack([x, np.ones(len(x))]) @ (Kn @ np.linalg.inv(Ko)).T)[:, :2]   # noqa: E731
    return move(x1, np.asarray(Ka), K1), move(x2, np.asarray(Kb), K2), E


def perturb(x1, x2, seed, sigma, outliers, box=((0, 0), (W, H_))):
    """Gaussian noise on image 2, then a fraction of uniform outliers in box; the mask of the others."""
    rng = np.random.default_rng(seed + 7919)
    x2 = x2 + rng.normal(0, sigma, x2.shape)
    out = rng.random(len(x2)) < outliers
    x2[out] = rng.uniform(box[0], box[1], (out.sum(), 2))
    return x1, x2, ~out


def assemble(x1, x2, good, seed, invalid=0.0):
    """Records, a pair list and its planted inliers: set 2 shuffled, pairs (k, perm[k]); with invalid > 0 about that
    fraction of invalid pairs interleaved at random positions, cycling through an index below 0, i = n1, j = n2,
    j = 2^31 - 1, a NaN coordinate in set 1 and an infinite one in set 2 (one extra record at the end of each set)."""
    rng = np.random.default_rng(seed + 104729)
    n = len(x1)
    perm = rng.permutation(n)
    s2 = np.empty_like(x2)
    s2[perm] = x2
    pairs = np.column_stack([np.arange(n), perm])
    r1, r2 = np.asarray(x1, np.float64), s2
    if invalid > 0:
        r1 = np.vstack([r1, [[np.nan, 5.0]]])
        r2 = np.vstack([r2, [[7.0, np.inf]]])
        m = max(1, int(round(invalid * n)))
        bad = []
        for q in range(m):
            i, j = int(rng.integers(n)), int(rng.integers(n))
            bad.append([(-1, j), (n + 1, j), (i, n + 1), (i, 2 ** 31 - 1), (n, j), (i, n)][q % 6])
        at = np.sort(rng.choice(n + m, m, replace=False))
        full, g = np.zeros((n + m, 2), np.int64), np.zeros(n + m, bool)
        keep = np.ones(n + m, bool)
        keep[at] = False
        full[keep], full[at], g[keep] = pairs, bad, good
        pairs, good = full, g
    return r1.astype(np.float32), r2.astype(np.float32), pairs.astype(np.int32), good


def fh_case(name, kind, n, seed, planar, sigma=0.5, outliers=0.1, invalid=0.1, loops=1024, thresh=2.0, tags=()):
    x1, x2, truth = fh_views(n, seed, planar, kind)
    x1, x2, good = perturb(x1, x2, seed, sigma, outliers)
    r1, r2, pairs, good = assemble(x1, x2, good, seed, invalid)
    return Case(name, kind, r1, r2, pairs, loops, thresh, seed, None, None, truth, good, frozenset(tags))


def e_case(name, n, seed, motion="sideways", planar=False, Ka=K1, Kb=K2, sigma=0.5, outliers=0.1, invalid=0.1,
           loops=1024, thresh=2.0, tags=()):
    x1, x2, E = e_views(n, seed, motion, planar, Ka, Kb)
    x1, x2, good = perturb(x1, x2, seed, sigma, outliers)
    r1, r2, pairs, good = assemble(x1, x2, good, seed, invalid)
    return Case(name, ESSENTIAL, r1, r2, pairs, loops, thresh, seed, np.asarray(Ka, np.float64),
                np.asarray(Kb, np.float64), E, good, frozenset(tags))


def shrunk(name, kind, seed, width, origin):
    """A planted scene (1 500 pairs, 0.5 px noise, 10 % outliers, thresh 2 px, 10 % invalid pairs) mapped into a
    width-pixel square at origin in both images, the noise and the threshold scaled alike."""
    planar = kind == vo.HOMOGRAPHY
    k = width / W
    x1, x2, truth = fh_views(1500, seed, planar, kind)
    A = np.array([[k, 0, origin[0]], [0, k, origin[1]], [0, 0, 1]])
    Ai = np.linalg.inv(A)
    truth = A @ truth @ Ai if planar else Ai.T @ truth @ Ai
    x1, x2 = x1 * k + origin, x2 * k + origin
    x1, x2, good = perturb(x1, x2, seed, 0.5 * k, 0.1, (origin, (origin[0] + width, origin[1] + width * H_ / W)))
    r1, r2, pairs, good = assemble(x1, x2, good, seed, 0.1)
    return Case(name, kind, r1, r2, pairs, 1024, 2.0 * k, seed, None, None, truth, good, frozenset())


# H with H[2][2] = 0: the origin of image 1 maps to the line at infinity, so the pixel-space output's scaling divides by
# a refitted H[2][2] that is noise around zero
H_AT_INFINITY = np.array([[1.2, 0.1, 0.0], [-0.05, 1.1, 0.0], [8e-4, 4e-4, 0.0]])


def h22_zero(name, seed):
    rng = np.random.default_rng(seed)
    x1 = rng.uniform([400, 300], [1500, 1000], (1500, 2))
    q = np.column_stack([x1, np.ones(len(x1))]) @ H_AT_INFINITY.T
    x1, x2, good = perturb(x1, q[:, :2] / q[:, 2:], seed, 0.3, 0.1, ((0, 0), (2000, 2000)))
    r1, r2, pairs, good = assemble(x1, x2, good, seed, 0.1)
    return Case(name, vo.HOMOGRAPHY, r1, r2, pairs, 1024, 2.0, seed, None, None, H_AT_INFINITY, good, frozenset())


def repeated(name, kind, seed, copies=100, others=40):
    """One correspondence (the pair list's first) repeated copies times among others, 0.5 px noise."""
    if kind == ESSENTIAL:
        x1, x2, truth = e_views(others, seed)
    else:
        x1, x2, truth = fh_views(others, seed, kind == vo.HOMOGRAPHY, kind)
    x1, x2, good = perturb(x1, x2, seed, 0.5, 0.0)
    r1, r2, pairs, good = assemble(x1, x2, good, seed)
    rng = np.random.default_rng(seed)
    at = np.sort(rng.choice(others + copies, copies, replace=False))
    full = np.zeros((others + copies, 2), np.int32)
    keep = np.ones(others + copies, bool)
    keep[at] = False
    full[keep], full[at] = pairs, pairs[0]
    Ka, Kb = (K1, K2) if kind == ESSENTIAL else (None, None)
    return Case(name, kind, r1, r2, full, 4096, 2.0, seed, Ka, Kb, truth, np.ones(len(full), bool), frozenset())


def tiny_threshold(name, kind, seed, n, loops, sigma, tags=()):
    """Threshold 0.01 px, sigma px of noise, no outliers: every live slot's inliers are its own sample (the seed chosen
    so that no other pair lies within 10 times the threshold of any slot's model)."""
    if kind == ESSENTIAL:
        return e_case(name, n, seed, sigma=sigma, outliers=0.0, invalid=0.0, loops=loops, thresh=0.01, tags=tags)
    return fh_case(name, kind, n, seed, kind == vo.HOMOGRAPHY, sigma=sigma, outliers=0.0, invalid=0.0, loops=loops,
                   thresh=0.01, tags=tags)


SKEWED = np.array([[1400.0, 25.0, 900.0], [0.0, 1450.0, 560.0], [0.0, 0.0, 1.0]])


def _builders():
    """name -> a function building the case.  Seeds tagged "drop" were chosen so that the refit loses inliers."""
    F, Hm = vo.FUNDAMENTAL, vo.HOMOGRAPHY
    b = {}
    # valid-pair counts: 0.3 px of noise (no pair within BAND of 2 px even among 262 145), 10 % outliers, 10 % invalid
    for n in SIZES:
        b[f"F-n{n}"] = functools.partial(fh_case, f"F-n{n}", F, n, 1000 + n, False, 0.3)
        b[f"H-n{n}"] = functools.partial(fh_case, f"H-n{n}", Hm, n, 2000 + n, True, 0.3)
        b[f"E-n{n}"] = functools.partial(e_case, f"E-n{n}", n, 3000 + n, sigma=0.3)
    for n in (4, 5, 6):
        b[f"H-n{n}"] = functools.partial(fh_case, f"H-n{n}", Hm, n, 2000 + n, True, 0.3)
    b["E-n5"] = functools.partial(e_case, "E-n5", 5, 3005, sigma=0.3)
    b["E-n6"] = functools.partial(e_case, "E-n6", 6, 3006, sigma=0.3)
    # the keep rule: exact data ties (kept), noisy scenes with outliers drop the refit
    for n in (8, 600):
        b[f"F-exact{n}"] = functools.partial(fh_case, f"F-exact{n}", F, n, 11 + n, False, 0.0, 0.0, 0.0, 512,
                                             tags=("exact", "whole"))
        b[f"E-exact{n}"] = functools.partial(e_case, f"E-exact{n}", n, 13 + n, sigma=0.0, outliers=0.0, invalid=0.0,
                                             loops=512, tags=("exact", "whole"))
    b["H-exact4"] = functools.partial(fh_case, "H-exact4", Hm, 4, 15, True, 0.0, 0.0, 0.0, 512, tags=("exact",))
    b["H-exact600"] = functools.partial(fh_case, "H-exact600", Hm, 600, 17, True, 0.0, 0.0, 0.0, 512,
                                        tags=("exact", "whole"))
    b["F-drop"] = functools.partial(fh_case, "F-drop", F, 2000, DROP_SEEDS["F"], False, 0.5, 0.4, 0.0, 512,
                                    tags=("drop", "whole"))
    b["H-drop"] = functools.partial(fh_case, "H-drop", Hm, 2000, DROP_SEEDS["H"], True, 0.5, 0.4, 0.0, 512,
                                    tags=("drop", "whole"))
    b["E-drop"] = functools.partial(e_case, "E-drop", 2000, DROP_SEEDS["E"], sigma=0.5, outliers=0.4, invalid=0.0,
                                    loops=512, tags=("drop", "whole"))
    # where a refit starts
    for k, kind, n, loops, sigma in (("F", F, 12, 8, 50.0), ("H", Hm, 40, 16, 30.0), ("E", ESSENTIAL, 12, 4, 50.0)):
        b[f"{k}-tiny"] = functools.partial(tiny_threshold, f"{k}-tiny", kind, TINY_SEEDS[k], n, loops, sigma,
                                           tags=("tiny",))
    # conditioning
    b["F-far"] = functools.partial(shrunk, "F-far", F, 41, 200.0, (40000.0, 30000.0))
    b["H-far"] = functools.partial(shrunk, "H-far", Hm, 42, 200.0, (40000.0, 30000.0))
    b["F-small"] = functools.partial(shrunk, "F-small", F, 43, 4.0, (50.0, 40.0))
    b["H-small"] = functools.partial(shrunk, "H-small", Hm, 44, 4.0, (50.0, 40.0))
    b["F-planar"] = functools.partial(fh_case, "F-planar", F, 2000, 45, True, outliers=0.0, tags=("clustered",))
    b["H-h22"] = functools.partial(h22_zero, "H-h22", 46)
    for k, kind in (("F", F), ("H", Hm), ("E", ESSENTIAL)):
        b[f"{k}-repeated"] = functools.partial(repeated, f"{k}-repeated", kind, 47)
    # E specifics (the degenerate scenes without outliers: an outlier that happens to fit lifts the spectrum)
    b["E-forward"] = functools.partial(e_case, "E-forward", 2000, 51, "forward")
    b["E-planar"] = functools.partial(e_case, "E-planar", 2000, 52, planar=True, outliers=0.0, tags=("clustered",))
    b["E-rotation"] = functools.partial(e_case, "E-rotation", 1000, 53, "rotation", outliers=0.0,
                                        tags=("rotation", "clustered"))
    b["E-sameK"] = functools.partial(e_case, "E-sameK", 1500, 54, Ka=K1, Kb=K1)
    b["E-skew"] = functools.partial(e_case, "E-skew", 1500, 55, Ka=SKEWED, Kb=K2)
    return b


DROP_SEEDS = {"F": 23, "H": 85, "E": 24}
TINY_SEEDS = {"F": 62, "H": 61, "E": 61}
BUILDERS = _builders()
NAMES = list(BUILDERS)


@functools.lru_cache(maxsize=None)
def case(name):
    return BUILDERS[name]()


def tags(name):
    """A case's tags without building it."""
    return frozenset(BUILDERS[name].keywords.get("tags", ()))


# ---- the restatement from the device's winning slot ---------------------------------------------------------------------
def valid(c):
    ok, xy = vo.valid_mask(c.x1[:, 0], c.x1[:, 1], c.x2[:, 0], c.x2[:, 1], c.pairs, len(c.x1), len(c.x2))
    return ok, xy[ok]


def residuals(c, M, p):
    if c.kind == ESSENTIAL:
        return eo.residuals(M, c.K1, c.K2, p)
    return vo.residuals(M, c.kind, p)


def band(c, r):
    """Pairs whose residual lies within BAND of the threshold."""
    return int((np.abs(r - c.thresh) <= BAND * c.thresh).sum())


def refit(c, p, inl, c1, c2, s):
    if c.kind == ESSENTIAL:
        return eo.refit(p, inl, c.K1, c.K2, s)
    return vo.refit(p, c.kind, inl, c1, c2, s)


def spectrum(c, p, inl, c1, c2, s):
    """lambda2 / lambda_max of the refit's normal matrix over the pairs inl (the rows of vo.refit / eo.refit)."""
    q = p[inl]
    if c.kind == ESSENTIAL:
        lam = s * math.sqrt(math.sqrt(c.K1[0, 0] * c.K1[1, 1]) * math.sqrt(c.K2[0, 0] * c.K2[1, 1]))
        x, y, X, Y = (eo.calibrated(q, c.K1, c.K2) * lam).T
    else:
        x, y, X, Y = ((q - np.concatenate([c1, c2])) * s).T
    one, zero = np.ones(len(q)), np.zeros(len(q))
    if c.kind == vo.HOMOGRAPHY:
        A = np.vstack([np.column_stack([x, y, one, zero, zero, zero, -X * x, -X * y, -X]),
                       np.column_stack([zero, zero, zero, x, y, one, -Y * x, -Y * y, -Y])])
    else:
        A = np.column_stack([X * x, X * y, X, Y * x, Y * y, Y, x, y, one])
    w = np.linalg.eigvalsh(A.T @ A)
    return float(w[1] / w[-1]) if w[-1] > 0 else 0.0


def unit(M):
    """Unit Frobenius norm, the largest-magnitude entry positive (F's and E's output scaling; H compared so too)."""
    return eo.unit_sign(M)


def diff(a, b):
    a, b = unit(a), unit(b)
    return float(np.linalg.norm(a - b))


def out_model(c, M):
    """What the call returns for the normalised-space model whose pixel form is M: H / H[2][2], F and E unit-signed;
    E projected to the essential manifold first."""
    if c.kind == ESSENTIAL:
        return unit(eo.project(M)[0])
    return vo.scale_model(M, c.kind)


def pose_margins(E, q):
    """The smallest relative magnitude, over every pose candidate and pair of q, of the two depth numerators and of the
    parallel-ray test of eo.in_front."""
    worst = np.inf
    for R, t in eo.pose_candidates(E):
        a = np.column_stack([q[:, 0], q[:, 1], np.ones(len(q))]) @ R.T
        b = np.column_stack([q[:, 2], q[:, 3], np.ones(len(q))])
        aa, bb, ab = (a * a).sum(1), (b * b).sum(1), (a * b).sum(1)
        at, bt = a @ t, b @ t
        for v, sc in ((aa * bb - ab * ab - eo.PARALLEL * aa * bb, aa * bb),
                      (ab * bt - at * bb, np.abs(ab * bt) + np.abs(at * bb)),
                      (aa * bt - ab * at, np.abs(aa * bt) + np.abs(ab * at))):
            if len(q):
                worst = min(worst, float((np.abs(v) / sc).min()))
    return worst


# ---- the device calls ---------------------------------------------------------------------------------------------------
Result = namedtuple("Result", "valid M C N k model R t inliers stats")


def _records(cs, xy):
    r = np.zeros(len(xy), cs.SIFT_DTYPE)
    r["xpos"], r["ypos"] = xy[:, 0], xy[:, 1]
    return r


def run(cs, c):
    """The models entry point, then the verify entry point with the same arguments."""
    L = cs.lib()
    recs = (_records(cs, c.x1), _records(cs, c.x2))
    bufs = [cs.DeviceBuffer(max(r.nbytes, 576)) for r in recs]
    try:
        bufs[0].upload(recs[0])
        bufs[1].upload(recs[1])
        pb, ob = cs.DeviceBuffer(max(c.pairs.nbytes, 8)), cs.DeviceBuffer(max(c.pairs.nbytes, 8))
        bufs += [pb, ob]
        pb.upload(np.ascontiguousarray(c.pairs))
        a = (bufs[0].ptr, len(c.x1), bufs[1].ptr, len(c.x2), pb.ptr, len(c.pairs))
        per = PER_SAMPLE[c.kind]
        M, C, N = np.zeros((per * c.loops, 9)), np.zeros(per * c.loops, np.int32), np.zeros(5)
        R, t = np.zeros(9), np.zeros(3)
        model = np.zeros(9)
        if c.kind == ESSENTIAL:
            k1, k2 = np.ascontiguousarray(c.K1), np.ascontiguousarray(c.K2)
            v = L.cs_verify_essential_models(*a, k1.ctypes.data, k2.ctypes.data, c.loops, c.thresh, c.seed,
                                             M.ctypes.data, C.ctypes.data, N.ctypes.data)
            assert v >= 0, L.cs_last_error()
            k = L.cs_verify_essential(*a, k1.ctypes.data, k2.ctypes.data, c.loops, c.thresh, c.seed, model.ctypes.data,
                                      R.ctypes.data, t.ctypes.data, ob.ptr, len(c.pairs), None)
            assert k >= 0, L.cs_last_error()
            st = list(cs.essential_stats())
        else:
            v = L.cs_verify_models(*a, c.kind, c.loops, c.thresh, c.seed, M.ctypes.data, C.ctypes.data, N.ctypes.data)
            assert v >= 0, L.cs_last_error()
            k = L.cs_verify_pairs(*a, c.kind, c.loops, c.thresh, c.seed, model.ctypes.data, ob.ptr, len(c.pairs), None)
            assert k >= 0, L.cs_last_error()
            st = list(cs.verify_stats())
        inl = ob.download(np.int32, 2 * k).reshape(-1, 2) if k else np.zeros((0, 2), np.int32)
    finally:
        for b in bufs:
            b.free()
    return Result(v, M, C, N, k, model.reshape(3, 3), R.reshape(3, 3), t, inl, st)


@functools.lru_cache(maxsize=None)
def result(cs, name):
    return run(cs, case(name))


# ---- the checks ---------------------------------------------------------------------------------------------------------
def check(c, g):
    """Every assertion of one case on the device result g; returns what the case showed ({kept, tie, clustered})."""
    st = g.stats
    ok, p = valid(c)
    # validity, the slot statistics and the arg-max rule: exact
    assert g.valid == st[0] == ok.sum() and st[1] == (~ok).sum()
    live = ~np.isnan(g.M[:, 0])
    per = PER_SAMPLE[c.kind]
    assert st[3] == live.sum() and st[2] == live[::per].sum()
    assert (g.C[~live] == 0).all()
    if not live.any():
        assert st[4] == -1 and st[5] == st[6] == st[7] == g.k == 0 and not g.model.any()
        return {"kept": 0, "tie": False, "clustered": False}
    counts = np.where(live, g.C, -1)
    best = int(np.argmax(counts))                                     # the first of the largest
    assert st[4] == best and st[5] == g.C[best]
    # the minimal model's inliers and the refit, from the device's own slot and normalisation
    c1, c2, s = g.N[:2], g.N[2:4], float(g.N[4])
    Mb = g.M[best].reshape(3, 3)
    r0 = residuals(c, Mb, p)
    inl0 = r0 < c.thresh
    assert band(c, r0) == 0, "a pair on the minimal model's threshold"
    assert inl0.sum() == st[5]
    Rr = refit(c, p, inl0, c1, c2, s)
    clustered = Rr is not None and spectrum(c, p, inl0, c1, c2, s) < CLUSTERED
    if Rr is None:
        assert st[6] == 0
    elif not clustered:
        rR = residuals(c, Rr, p)
        assert band(c, rR) == 0, "a pair on the refit's threshold"
        assert st[6] == int((rR < c.thresh).sum() >= inl0.sum())
    kept = st[6]
    # the returned model
    out = g.model
    assert np.isfinite(out).all()
    if c.kind == vo.HOMOGRAPHY:
        assert out[2, 2] == 1.0 or out[2, 2] == 0.0
    else:
        assert abs(np.linalg.norm(out) - 1) < 1e-12 and out.reshape(-1)[np.argmax(np.abs(out))] > 0
    if not kept:
        assert diff(out, out_model(c, Mb)) <= SLOT_TOL, diff(out, out_model(c, Mb))
    elif not clustered:
        assert diff(out, out_model(c, Rr)) <= MODEL_TOL, diff(out, out_model(c, Rr))
    if c.kind == vo.FUNDAMENTAL:
        assert abs(np.linalg.det(unit(out))) <= 1e-12
    # the final inliers: the returned model's, in input order; a kept refit has no fewer than the minimal model
    rO = residuals(c, out, p)
    assert band(c, rO) == 0, "a pair on the returned model's threshold"
    final = rO < c.thresh
    assert np.array_equal(g.inliers, c.pairs[ok][final])
    assert g.k == st[7] == final.sum()
    assert st[7] >= st[5] if kept else st[7] == st[5]
    if c.kind == ESSENTIAL:
        check_pose(c, g, p[final])
    return {"kept": kept, "tie": bool(kept and st[7] == st[5]), "clustered": clustered}


def check_pose(c, g, pf):
    R, t, st = g.R, g.t, g.stats
    assert abs(np.linalg.det(R) - 1) < 1e-9 and np.abs(R.T @ R - np.eye(3)).max() < 1e-9
    assert abs(np.linalg.norm(t) - 1) < 1e-12
    Ex = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ R
    assert abs(abs(np.sum(Ex * g.model)) / np.linalg.norm(Ex) - 1) < 1e-9       # E proportional to [t]x R
    if "rotation" in c.tags:
        return
    q = eo.calibrated(pf, c.K1, c.K2)
    assert pose_margins(g.model, q) > NEAR_ZERO
    Rw, tw, front, runner = eo.choose_pose(g.model, q)
    assert (st[8], st[9]) == (front, runner)
    if front > runner:
        assert np.abs(R - Rw).max() <= POSE_TOL and np.abs(t - tw).max() <= POSE_TOL


def check_tags(c, g, shown):
    st = g.stats
    if "exact" in c.tags:
        assert shown["kept"] == 1 and shown["tie"] and st[5] == st[0]
    if "drop" in c.tags:
        assert shown["kept"] == 0
    if "tiny" in c.tags:
        live = ~np.isnan(g.M[:, 0])
        assert st[4] == int(np.argmax(live)) and st[5] == SAMPLE[c.kind]
        assert st[6] == int(c.kind == vo.HOMOGRAPHY) and st[7] == SAMPLE[c.kind]
    if "clustered" in c.tags:
        assert shown["clustered"]


@pytest.mark.parametrize("name", NAMES)
def test_refit_against_restatement(cs, name):
    c = case(name)
    g = result(cs, name)
    check_tags(c, g, check(c, g))


def test_keep_rule_branches_occur(cs):
    """Across the cases, each model keeps a refit on a tie (cntR == cnt0), keeps one, and drops one."""
    for k, kind in KINDS.items():
        shown = []
        for name in NAMES:
            if case(name).kind == kind:
                g = result(cs, name)
                shown.append((g.stats[6], bool(g.stats[6] and g.stats[7] == g.stats[5])))
        assert (0, False) in shown and (1, True) in shown, (k, shown)
        assert any(kept for kept, _ in shown), k


@pytest.mark.parametrize("name", [n for n in NAMES if "whole" in tags(n)])
def test_whole_call_restated(cs, name):
    """The whole call in float64 from scratch picks the device's slot and count, and returns its model and inliers."""
    c = case(name)
    g = result(cs, name)
    assert c.loops <= 512
    a = (c.x1[:, 0], c.x1[:, 1], c.x2[:, 0], c.x2[:, 1], c.pairs, len(c.x1), len(c.x2))
    if c.kind == ESSENTIAL:
        M, R, t, inl, best, cnt = eo.verify(*a, c.K1, c.K2, c.loops, c.thresh, c.seed)
    else:
        M, inl, best, cnt = vo.verify(*a, c.kind, c.loops, c.thresh, c.seed)
    assert (best, cnt) == (g.stats[4], g.stats[5])
    assert diff(g.model, M) <= (SLOT_TOL if not g.stats[6] else MODEL_TOL), diff(g.model, M)
    assert np.array_equal(inl, g.inliers)
    if c.kind == ESSENTIAL and g.stats[8] > g.stats[9]:
        assert np.abs(R - g.R).max() <= POSE_TOL and np.abs(t - g.t).max() <= POSE_TOL


# ---- the batch ----------------------------------------------------------------------------------------------------------
BATCH_LOOPS, BATCH_THRESH = 256, 2.0


@pytest.mark.parametrize("kind", ["F", "H", "E"])
def test_batch_equals_single_calls(cs, kind):
    """Every case of a model in one jagged batch (common numLoops and threshold): each job equals its single call byte
    for byte."""
    L = cs.lib()
    cases = [case(n) for n in NAMES if case(n).kind == KINDS[kind]]
    bufs = []

    def put(arr):
        b = cs.DeviceBuffer(max(arr.nbytes, 576))
        if arr.nbytes:
            b.upload(np.ascontiguousarray(arr))
        bufs.append(b)
        return b

    try:
        J = len(cases)
        t = (cs.VerifyJob * J)()
        dev = []
        for q, c in enumerate(cases):
            s1, s2, pr = put(_records(cs, c.x1)), put(_records(cs, c.x2)), put(c.pairs)
            ib, isg = put(np.full(2 * len(c.pairs), -7, np.int32)), put(np.full(2 * len(c.pairs), -7, np.int32))
            dev.append((s1, s2, pr, ib, isg))
            t[q] = cs.VerifyJob(s1.ptr, len(c.x1), s2.ptr, len(c.x2), pr.ptr, len(c.pairs), c.seed, ib.ptr,
                                len(c.pairs))
        counts = np.full(J, -1, np.int32)
        if kind == "E":
            k1 = np.ascontiguousarray([c.K1.reshape(9) for c in cases])
            k2 = np.ascontiguousarray([c.K2.reshape(9) for c in cases])
            E, R, tt, stats = np.zeros((J, 9)), np.zeros((J, 9)), np.zeros((J, 3)), np.zeros((J, 10), np.int64)
            r = L.cs_verify_essential_batch(ctypes.addressof(t), J, k1.ctypes.data, k2.ctypes.data, BATCH_LOOPS,
                                            BATCH_THRESH, E.ctypes.data, R.ctypes.data, tt.ctypes.data,
                                            counts.ctypes.data, stats.ctypes.data, None)
        else:
            E, stats = np.zeros((J, 9)), np.zeros((J, 8), np.int64)
            r = L.cs_verify_pairs_batch(ctypes.addressof(t), J, KINDS[kind], BATCH_LOOPS, BATCH_THRESH, E.ctypes.data,
                                        counts.ctypes.data, stats.ctypes.data, None)
        assert r == 0, L.cs_last_error()
        for q, c in enumerate(cases):
            s1, s2, pr, ib, isg = dev[q]
            a = (s1.ptr, len(c.x1), s2.ptr, len(c.x2), pr.ptr, len(c.pairs))
            m = np.zeros(9)
            if kind == "E":
                Rs, ts = np.zeros(9), np.zeros(3)
                k1, k2 = np.ascontiguousarray(c.K1), np.ascontiguousarray(c.K2)
                k = L.cs_verify_essential(*a, k1.ctypes.data, k2.ctypes.data, BATCH_LOOPS, BATCH_THRESH, c.seed,
                                          m.ctypes.data, Rs.ctypes.data, ts.ctypes.data, isg.ptr, len(c.pairs), None)
                st = np.array(cs.essential_stats(), np.int64)
                assert R[q].tobytes() == Rs.tobytes() and tt[q].tobytes() == ts.tobytes(), c.name
            else:
                k = L.cs_verify_pairs(*a, KINDS[kind], BATCH_LOOPS, BATCH_THRESH, c.seed, m.ctypes.data, isg.ptr,
                                      len(c.pairs), None)
                st = np.array(cs.verify_stats(), np.int64)
            assert k >= 0, L.cs_last_error()
            assert E[q].tobytes() == m.tobytes() and counts[q] == k and np.array_equal(stats[q], st), c.name
            got = ib.download(np.int32, 2 * len(c.pairs)).reshape(-1, 2)
            want = isg.download(np.int32, 2 * len(c.pairs)).reshape(-1, 2)
            assert np.array_equal(got, want), c.name
    finally:
        for b in bufs:
            b.free()
