"""Scenes for absolute pose (cs_absolute_pose_batch): a camera with skewed, unequal intrinsics looking at a cloud of
known points (triangulate_cases' cameras and intrinsics), records of its noisy projections with a fraction of
outliers, and the pointOf table that ties them together."""
import numpy as np

import triangulate_cases as tc

W, H = tc.W, tc.H


def job(rng, V, noise=0.5, outlier=0.3, extra=0, numPoints=None):
    """One image of V correspondences: (xy float32 [V + extra, 2], pointOf int32, points [P, 3], K, R, t).  The points
    lie in [-3, 3]^3 in front of the camera; a fraction `outlier` of the records sit at uniform positions; `extra`
    records name no point (pointOf -1)."""
    while True:
        Ks, Rs, ts = tc.cameras(rng, 1)
        K, R, t = Ks[0], Rs[0], ts[0]
        P = numPoints or V
        X = rng.uniform(-3, 3, (P, 3))
        Xc = X @ R.T + t
        if (Xc[:, 2] > 1.0).all():
            break
    pointOf = rng.permutation(P)[:V] if P >= V else rng.integers(0, P, V)
    u = (X[pointOf] @ R.T + t) @ K.T
    xy = u[:, :2] / u[:, 2:] + rng.normal(0, noise, (V, 2))
    out = rng.random(V) < outlier
    xy[out] = rng.uniform([0, 0], [W, H], (int(out.sum()), 2))
    if extra:
        xy = np.concatenate([xy, rng.uniform([0, 0], [W, H], (extra, 2))])
        pointOf = np.concatenate([pointOf, -np.ones(extra, np.int64)])
    order = rng.permutation(len(xy))
    return (np.ascontiguousarray(xy[order], np.float32), pointOf[order].astype(np.int32), X, K, R, t)


def batch(seed, sizes, noise=0.5, outliers=(0.1, 0.5)):
    """Jobs of the given correspondence counts over one shared point array: (xys, pointOfs, points, Ks, Rs, ts)."""
    rng = np.random.default_rng(seed)
    xys, pos, Ks, Rs, ts, pts = [], [], [], [], [], []
    base = 0
    for V in sizes:
        xy, po, X, K, R, t = job(rng, V, noise, rng.uniform(*outliers), extra=int(rng.integers(0, 4)))
        xys.append(xy)
        pos.append(np.where(po >= 0, po + base, -1).astype(np.int32))
        pts.append(X)
        Ks.append(K); Rs.append(R); ts.append(t)
        base += len(X)
    return xys, pos, np.concatenate(pts), np.array(Ks), np.array(Rs), np.array(ts)


def records(xy):
    """SiftPoint records with these positions (every other field zero)."""
    from cudasift_b200 import SIFT_DTYPE
    r = np.zeros(len(xy), SIFT_DTYPE)
    r["xpos"], r["ypos"] = xy[:, 0], xy[:, 1]
    return r
