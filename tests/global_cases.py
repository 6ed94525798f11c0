"""View graphs for rotation averaging (cs_rotation_averaging): cameras on a shell around the scene (triangulate_cases),
each image paired with its nearest cameras, the pair's relative rotation R_j R_i^T perturbed by a small rotation, a
fraction of pairs replaced by random rotations, and inlier-count-like weights."""
import numpy as np

import rotavg_oracle as ro
import triangulate_cases as tc


def random_rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def view_graph(seed, numImages=50, neighbours=6, noiseDeg=0.0, outliers=0.0, components=1, weights=(50, 300),
               outlierWeights=(15, 60)):
    """Cameras on a shell; each image paired with its `neighbours` nearest cameras (by centre), deduplicated, as
    {lower, higher} image.  Relative rotations Q = R_j R_i^T exp(n) with n of sigma noiseDeg per axis; a fraction
    `outliers` of edges replaced by uniform random rotations.  Weights are drawn as inlier counts: uniform integers in
    `weights`, and in `outlierWeights` for a replaced edge (a wrong relative pose keeps few inliers; the ranges overlap,
    so the spanning tree may still take one).  With components > 1 the images are split into that many groups by index
    and only pairs inside a group are kept.  Returns dict(Rs, Cs, edges, Rrel, weights, outlier)."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = tc.cameras(rng, numImages)
    Cs = -np.einsum("aji,aj->ai", Rs, ts)
    group = np.arange(numImages) * components // numImages
    pairs = set()
    for a in range(numImages):
        d = np.linalg.norm(Cs - Cs[a], axis=1)
        d[group != group[a]] = np.inf
        for b in np.argsort(d, kind="stable")[1:neighbours + 1]:
            if np.isfinite(d[b]):
                pairs.add((min(a, int(b)), max(a, int(b))))
    edges = np.array(sorted(pairs), np.int32).reshape(-1, 2)
    E = len(edges)
    Rrel = np.empty((E, 3, 3))
    for e, (i, j) in enumerate(edges):
        Rrel[e] = Rs[j] @ Rs[i].T @ ro.exp_rot(np.radians(noiseDeg) * rng.normal(size=3))
    outlier = rng.random(E) < outliers
    for e in np.flatnonzero(outlier):
        Rrel[e] = random_rotation(rng)
    w = np.where(outlier, rng.integers(*outlierWeights, E), rng.integers(*weights, E)).astype(np.float64)
    return dict(Rs=Rs, Cs=Cs, edges=edges, Rrel=Rrel, weights=w, outlier=outlier)
