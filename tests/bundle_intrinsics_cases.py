"""Scenes for self-calibrating bundle adjustment (cs_bundle_adjust_intrinsics): bundle_cases' cameras on a path around a
point cloud, imaged through radial distortion (k1, k2), and started from a focal length off by a factor, k = 0 and
perturbed poses and points."""
import numpy as np

import bundle_cases as bc
import bundle_intrinsics_oracle as bio
import triangulate_cases as tc

W, H = tc.W, tc.H


def scene(seed, k=(-0.08, 0.01), focal=1.07, numImages=6, numPoints=150, lengths=(3, 12), noise=0.0, outlier=0.0,
          rot=0.005, trans=0.05, point=0.03):
    """A dict as bundle_cases.scene's, plus k (the true (k1, k2) of every image) and K0 (K with K0, K1 and K4 scaled
    by `focal`: the guessed start, the ratios of the truth held).  Outliers are uniform positions with use False."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = bc.path_cameras(rng, numImages)
    kk = np.tile(np.asarray(k, np.float64), (numImages, 1))
    b = tc.Builder(numImages)
    Xs, use = [], []
    while len(Xs) < numPoints:
        X = rng.uniform(-2, 2, 3)
        seen = []
        for a in range(numImages):
            Xc = Rs[a] @ X + ts[a]
            if Xc[2] <= 0:
                continue
            px = bio.distort(Ks[a], kk[a], Xc[None])[0]
            if 0 <= px[0] < W and 0 <= px[1] < H:
                seen.append((a, px))
        L = int(rng.integers(lengths[0], lengths[1] + 1))
        if len(seen) < 2:
            continue
        pick = sorted(rng.permutation(len(seen))[:min(L, len(seen))])
        obs = []
        for j in pick:
            a, px = seen[j]
            bad = rng.random() < outlier
            q = rng.uniform([0, 0], [W, H]) if bad else px + rng.normal(0, noise, 2)
            obs.append((a, b.record(a, q[0], q[1])))
            use.append(not bad)
        b.track(obs)
        Xs.append(X)
    xy, offsets, members = b.arrays()
    X = np.array(Xs)
    R0, t0, X0 = bc.perturb(rng, Rs, ts, X, rot, trans, point)
    K0 = Ks.copy()
    K0[:, 0, :2] *= focal
    K0[:, 1, 1] *= focal
    return dict(xy=xy, offsets=offsets, members=members, use=np.array(use), K=Ks, k=kk, K0=K0, R=Rs, t=ts, X=X, R0=R0,
                t0=t0, X0=X0)
