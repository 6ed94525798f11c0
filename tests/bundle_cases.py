"""Scenes for bundle adjustment (cs_bundle_adjust): cameras with skewed, unequal intrinsics (triangulate_cases') on a
path around a point cloud, tracks of 2 to 12 views with pixel noise, outlier observations switched off through use,
and perturbed poses and points to start from.  large() builds BAL-like sizes for the benchmark."""
import numpy as np

import bundle_oracle as bo
import triangulate_cases as tc

W, H = tc.W, tc.H


def path_cameras(rng, n, radius=10.0, arc=1.4):
    """n cameras on an arc of the given angle around the origin, looking at it with small rolls."""
    Ks, Rs, ts = [], [], []
    for a in range(n):
        th = -arc / 2 + arc * a / max(n - 1, 1)
        C = np.array([radius * np.sin(th), rng.uniform(-1, 1), -radius * np.cos(th)])
        R = tc.look_at(C, rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.2, 0.2))
        Ks.append(tc.intrinsics(rng))
        Rs.append(R)
        ts.append(-R @ C)
    return np.array(Ks), np.array(Rs), np.array(ts)


def perturb(rng, Rs, ts, X, rot, trans, point, first=2):
    """Poses of cameras first.. rotated by about rot radians and moved by about trans; points moved by about point."""
    R1, t1 = Rs.copy(), ts.copy()
    for a in range(first, len(Rs)):
        R1[a] = bo.rodrigues(rng.normal(0, rot, 3)) @ Rs[a]
        t1[a] = ts[a] + rng.normal(0, trans, 3)
    return R1, t1, X + rng.normal(0, point, X.shape)


def scene(seed, numImages=6, numPoints=150, lengths=(2, 12), noise=0.5, outlier=0.05, rot=0.01, trans=0.1,
          point=0.05):
    """A dict: xy (per image float32 [n, 2]), offsets, members, use (False for the outliers), K, R, t (truth),
    R0, t0, X0 (the start) and X (truth)."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = path_cameras(rng, numImages)
    b = tc.Builder(numImages)
    Xs, use = [], []
    while len(Xs) < numPoints:
        X = rng.uniform(-2, 2, 3)
        seen = []
        for a in range(numImages):
            u = Ks[a] @ (Rs[a] @ X + ts[a])
            if u[2] > 0 and 0 <= u[0] / u[2] < W and 0 <= u[1] / u[2] < H:
                seen.append((a, u[:2] / u[2]))
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
    R0, t0, X0 = perturb(rng, Rs, ts, X, rot, trans, point)
    return dict(xy=xy, offsets=offsets, members=members, use=np.array(use), K=Ks, R=Rs, t=ts, X=X, R0=R0, t0=t0,
                X0=X0)


def large(seed, numImages, numPoints, perPoint=4, noise=0.5, rot=0.002, trans=0.02, point=0.02):
    """BAL-like sizes, vectorised: cameras on a circle of radius 20 looking at a cloud of radius 5, each point seen by
    perPoint consecutive cameras of the path.  The same dict as scene() (use all True)."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = [], [], []
    for a in range(numImages):
        th = 2 * np.pi * a / numImages
        C = np.array([20 * np.sin(th), rng.uniform(-1, 1), -20 * np.cos(th)])
        R = tc.look_at(C, np.zeros(3), rng.uniform(-0.1, 0.1))
        Ks.append(tc.intrinsics(rng)); Rs.append(R); ts.append(-R @ C)
    Ks, Rs, ts = np.array(Ks), np.array(Rs), np.array(ts)
    X = rng.uniform(-3, 3, (numPoints, 3))
    c0 = rng.integers(0, numImages, numPoints)
    cams = (c0[:, None] + np.arange(perPoint)[None]) % numImages          # [P, L]
    a = cams.reshape(-1)
    k = np.repeat(np.arange(numPoints), perPoint)
    u = np.einsum("nij,nj->ni", Ks[a], np.einsum("nij,nj->ni", Rs[a], X[k]) + ts[a])
    px = u[:, :2] / u[:, 2:] + rng.normal(0, noise, (len(a), 2))
    order = np.argsort(a, kind="stable")
    feat = np.empty(len(a), np.int64)
    counts = np.bincount(a, minlength=numImages)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    feat[order] = np.arange(len(a)) - starts[a[order]]
    xy = [np.ascontiguousarray(px[order[starts[i]:starts[i] + counts[i]]], np.float32) for i in range(numImages)]
    members = np.stack([a, feat], 1).astype(np.int32)
    offsets = (np.arange(numPoints + 1) * perPoint).astype(np.int32)
    R0, t0, X0 = perturb(rng, Rs, ts, X, rot, trans, point)
    return dict(xy=xy, offsets=offsets, members=members, use=np.ones(len(a), bool), K=Ks, R=Rs, t=ts, X=X, R0=R0,
                t0=t0, X0=X0)


def gauge(t):
    """The default gauge of BundleAdjust: image 0 held, image 1 holds its largest |t| component."""
    f = np.zeros(len(t), np.uint8)
    f[0] = 1
    if len(t) > 1:
        f[1] = 2 + int(np.argmax(np.abs(t[1])))
    return f


def chain(cs, seed=3):
    """The six shifted views of the incremental chain (a plane Z = Z0 = 10 seen by cameras R = I, f = 200, translated
    by the shifts) through the device chain: extraction, the ratio, verify and guided batches, BuildTracks.  Views 2 to
    5 get about two pixels of pose error (R, t0); views 0 and 1 keep the truth.  Returns a dict with the SiftData of
    every view (the caller frees them), their record positions, the tracks, K, the true t and the perturbed poses."""
    import itertools
    from cudasift_b200.synth import synth_image
    w, h = 960, 540
    img = synth_image(w, h, seed=9)
    shifts = [(0, 0), (3, 5), (-4, 6), (8, -2), (-6, -7), (10, 9)]
    views = [np.ascontiguousarray(np.roll(img, s, axis=(0, 1))) for s in shifts]
    pitch = cs.iAlignUp(w, 128)
    cis = [cs.CudaImage().Allocate(w, h, pitch, False, None, v) for v in views]
    for ci in cis:
        ci.Download()
    ex = cs.Extractor(w, h, 5, 1000, False, batch=6, maxCandidates=16384)
    datas = []
    try:
        ex.submit_device_batch([ci.d_data for ci in cis], pitch, 1.0, 3.0, 0.0)
        counts = ex.wait_batch(6)
        for i in range(6):
            d = cs.SiftData()
            cs.InitSiftData(d, int(counts[i]))
            d._buf.upload(ex.device_points_at(i, int(counts[i])))
            d.numPts = int(counts[i])
            datas.append(d)
    finally:
        ex.close()
    try:
        pairs_idx = list(itertools.combinations(range(6), 2))
        ratio, _, _ = cs.MatchSiftDataRatioBatch(datas, pairs_idx)
        Mv, inl, _, _ = cs.VerifyPairsBatch([(datas[a], datas[b], ratio[k], k) for k, (a, b) in enumerate(pairs_idx)],
                                            "fundamental", 1024, 4.0)
        keep = [k for k in range(len(pairs_idx)) if len(inl[k]) >= 30]
        jobs = [pairs_idx[k] for k in keep]
        guided, _, _ = cs.MatchSiftDataGuidedBatch(datas, jobs, "fundamental", Mv[keep], 4.0)
        sizes = [d.numPts for d in datas]
        offsets, members, _, _, _ = cs.BuildTracks(sizes, [(a, b, g) for (a, b), g in zip(jobs, guided)])
        recs = [d._buf.download(cs.SIFT_DTYPE, d.numPts) for d in datas]
    except BaseException:
        for d in datas:
            cs.FreeSiftData(d)
        raise
    xy = [np.stack([r["xpos"], r["ypos"]], 1).astype(np.float32) for r in recs]
    f, Z0 = 200.0, 10.0
    K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]])
    ts = np.array([[dx * Z0 / f, dy * Z0 / f, 0.0] for dy, dx in shifts])
    rng = np.random.default_rng(seed)
    Rs, ts0 = np.stack([np.eye(3)] * 6), ts.copy()
    for a in range(2, 6):
        Rs[a] = bo.rodrigues(rng.normal(0, 1.0 / f, 3)) @ Rs[a]
        ts0[a] = ts[a] + np.append(rng.normal(0, Z0 / f, 2), 0.0)
    return dict(datas=datas, xy=xy, offsets=offsets, members=members, K=K, ts=ts, Rs=Rs, ts0=ts0, f=f, Z0=Z0, w=w,
                h=h)
