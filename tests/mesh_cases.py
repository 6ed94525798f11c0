"""Point clouds for the Poisson mesher's tests: sphere, torus, two nested spheres (a hollow shell), an upper hemisphere
(an open surface), and the piecewise-planar scene of stereo_cases through the library; plus analytic fields."""
import numpy as np

CENTRE = np.array([0.3, -0.2, 1.5])


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def sphere(n, radius=1.0, seed=0, centre=CENTRE):
    """Uniform samples with exact outward normals: (xyz float32 [n, 3], normal float32 [n, 3])."""
    u = _unit(np.random.default_rng(seed), n)
    return (centre + radius * u).astype(np.float32), u.astype(np.float32)


def torus(n, R=1.0, r=0.4, seed=0, centre=CENTRE):
    """Samples of a torus around z (area-uniform), exact outward normals."""
    rng = np.random.default_rng(seed)
    u = rng.uniform(0, 2 * np.pi, 4 * n)
    v = rng.uniform(0, 2 * np.pi, 4 * n)
    keep = rng.uniform(0, 1, 4 * n) < (R + r * np.cos(v)) / (R + r)
    u, v = u[keep][:n], v[keep][:n]
    nrm = np.stack([np.cos(v) * np.cos(u), np.cos(v) * np.sin(u), np.sin(v)], 1)
    ctr = np.stack([R * np.cos(u), R * np.sin(u), np.zeros_like(u)], 1)
    return (centre + ctr + r * nrm).astype(np.float32), nrm.astype(np.float32)


def shell(n, outer=1.0, inner=0.5, seed=0):
    """Two nested spheres, the inner one with inward normals: a hollow shell."""
    x1, n1 = sphere(n, outer, seed)
    x2, n2 = sphere(max(n // 4, 1), inner, seed + 1)
    return np.concatenate([x1, x2]), np.concatenate([n1, -n2])


def hemisphere(n, radius=1.0, seed=0):
    """The upper half (z >= centre z) of a sphere: an open surface."""
    x, nr = sphere(2 * n, radius, seed)
    up = x[:, 2] >= CENTRE[2]
    return x[up][:n], nr[up][:n]


def sphere_field(N, radius):
    """R - |x - c| on an (N + 1)^3 grid (z, y, x) around the centre: the inside is a ball."""
    c = N / 2 + 0.137
    k, j, i = np.meshgrid(*(np.arange(N + 1, dtype=float),) * 3, indexing="ij")
    return (radius - np.sqrt((i - c) ** 2 + (j - c) ** 2 + (k - c) ** 2)).astype(np.float32)


def torus_field(N, R, r):
    c = N / 2 + 0.137
    k, j, i = np.meshgrid(*(np.arange(N + 1, dtype=float),) * 3, indexing="ij")
    x, y, z = i - c, j - c, k - c
    return (r - np.sqrt((np.sqrt(x * x + y * y) - R) ** 2 + z * z)).astype(np.float32)


def rect_distance(P, rects):
    """Distance of points P [n, 3] to the nearest rectangle of stereo_cases.scene()."""
    best = np.full(len(P), np.inf)
    for r in rects:
        d = P - r["c"]
        a = np.clip(d @ r["u"], -r["hu"], r["hu"])
        b = np.clip(d @ r["v"], -r["hv"], r["hv"])
        best = np.minimum(best, np.linalg.norm(d - a[:, None] * r["u"] - b[:, None] * r["v"], axis=1))
    return best
