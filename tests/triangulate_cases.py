"""Scenes for triangulation (cs_triangulate_tracks): pinhole cameras with skewed, unequal intrinsics and arbitrary
rolls around a point cloud, tracks of noisy observations with outliers, and the record positions of every image."""
import numpy as np

W, H = 1280, 960


def look_at(C, target, roll):
    """The rotation of a camera at C whose optical axis points at target, rolled about that axis."""
    z = target - C
    z = z / np.linalg.norm(z)
    up = np.array([0.0, 1.0, 0.0]) if abs(z[1]) < 0.9 else np.array([1.0, 0.0, 0.0])
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    c, s = np.cos(roll), np.sin(roll)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]) @ np.stack([x, y, z])


def intrinsics(rng):
    fx = rng.uniform(600, 1400)
    return np.array([[fx, rng.uniform(-4, 4), W / 2 + rng.uniform(-30, 30)],
                     [0, fx * rng.uniform(0.85, 1.15), H / 2 + rng.uniform(-30, 30)], [0, 0, 1.0]])


def cameras(rng, n, radius=(8.0, 15.0), away=0):
    """n cameras on a shell around the origin looking at it; the last `away` of them look away (every point behind)."""
    Ks, Rs, ts = [], [], []
    for a in range(n):
        d = rng.normal(size=3)
        C = d / np.linalg.norm(d) * rng.uniform(*radius)
        target = rng.uniform(-0.5, 0.5, 3)
        R = look_at(C, target if a < n - away else 2 * C - target, rng.uniform(0, 2 * np.pi))
        Ks.append(intrinsics(rng))
        Rs.append(R)
        ts.append(-R @ C)
    return np.array(Ks), np.array(Rs), np.array(ts)


def project(K, R, t, X):
    u = K @ (R @ X + t)
    return u[:2] / u[2]


class Builder:
    """Records per image (positions only) and tracks as BuildTracks returns them."""

    def __init__(self, numImages):
        self.xy = [[] for _ in range(numImages)]
        self.offsets, self.members = [0], []

    def record(self, a, x, y):
        self.xy[a].append((x, y))
        return len(self.xy[a]) - 1

    def track(self, obs):
        """obs: [(image, feature)] as members."""
        self.members += [list(o) for o in obs]
        self.offsets.append(len(self.members))

    def arrays(self):
        xy = [np.array(p, np.float32).reshape(-1, 2) for p in self.xy]
        return xy, np.array(self.offsets, np.int32), np.array(self.members, np.int32).reshape(-1, 2)


def scene(seed, numImages=80, numTracks=300, lengths=(2, 64), noise=0.5, outliers=(0.1, 0.3), away=2, repeat=0.0):
    """Random tracks over numImages cameras (the last `away` looking away): each of a length in lengths, over distinct
    images (one image twice with probability repeat), its points in [-3, 3]^3, pixel noise of sigma `noise` and a
    fraction of outliers drawn per track from `outliers` (uniform positions).  Returns (xy, Ks, Rs, ts, offsets,
    members, points)."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = cameras(rng, numImages, away=away)
    b = Builder(numImages)
    pts = rng.uniform(-3, 3, (numTracks, 3))
    for k in range(numTracks):
        L = int(rng.integers(lengths[0], lengths[1] + 1))
        imgs = list(rng.choice(numImages, min(L, numImages), replace=False))
        if rng.random() < repeat:
            imgs.append(imgs[0])
        rate = rng.uniform(*outliers)
        obs = []
        for a in imgs:
            a = int(a)
            if a >= numImages - away or rng.random() < rate:
                x, y = rng.uniform(0, W), rng.uniform(0, H)
            else:
                x, y = project(Ks[a], Rs[a], ts[a], pts[k]) + rng.normal(0, noise, 2)
            obs.append((a, b.record(a, x, y)))
        b.track(obs)
    xy, offsets, members = b.arrays()
    return xy, Ks, Rs, ts, offsets, members, pts


def scale(Ks, Rs, ts):
    """The scene scale: the largest distance of a camera centre from the origin."""
    return float(np.max(np.linalg.norm(np.einsum("aji,aj->ai", Rs, ts), axis=1)))


def collection(seed, numTracks, numImages=1000, lengths=(2, 12), outlier=0.1, noise=0.5):
    """A large collection, built vectorised: numTracks points in [-3, 3]^3, each seen by a length in lengths of images
    drawn with replacement (so some tracks hold two members of one image), pixel noise of sigma `noise`, a fraction
    `outlier` of uniform observations.  Returns (xy, Ks, Rs, ts, offsets, members, points)."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = cameras(rng, numImages)
    pts = rng.uniform(-3, 3, (numTracks, 3))
    L = rng.integers(lengths[0], lengths[1] + 1, numTracks)
    offsets = np.concatenate([[0], np.cumsum(L)]).astype(np.int64)
    M = int(offsets[-1])
    track = np.repeat(np.arange(numTracks), L)
    a = rng.integers(0, numImages, M)
    Xc = np.einsum("mij,mj->mi", Rs[a], pts[track]) + ts[a]
    u = np.einsum("mij,mj->mi", Ks[a], Xc)
    px = u[:, :2] / u[:, 2:] + rng.normal(0, noise, (M, 2))
    out = rng.random(M) < outlier
    px[out] = rng.uniform([0, 0], [W, H], (int(out.sum()), 2))
    order = np.argsort(a, kind="stable")
    counts = np.bincount(a, minlength=numImages)
    starts = np.concatenate([[0], np.cumsum(counts)])
    f = np.empty(M, np.int64)
    f[order] = np.arange(M) - starts[a[order]]
    xy = [np.ascontiguousarray(px[order[starts[i]:starts[i + 1]]], np.float32) for i in range(numImages)]
    members = np.stack([a, f], 1).astype(np.int32)
    return xy, Ks, Rs, ts, offsets.astype(np.int32), members, pts
