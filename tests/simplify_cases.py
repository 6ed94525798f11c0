"""Meshes for the simplifier's tests: small hand-made ones (a bowtie, a tetrahedron, an edge with three faces, a flipped
face, a flat grid with a boundary) and the marching-tetrahedra meshes of mesh_cases' sphere and torus fields and of the
screened sheet, with jittered copies."""
import numpy as np

import mesh_cases as mc
import mesh_oracle as mo


def grid(n=8, jitter=0.0, seed=0):
    """A flat n x n grid of unit squares in z = 0, two triangles each, counter-clockwise seen from +z."""
    i, j = np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing="xy")
    v = np.stack([i.ravel(), j.ravel(), np.zeros(i.size)], 1).astype(np.float64)
    if jitter:
        v[:, :2] += np.random.default_rng(seed).uniform(-jitter, jitter, (len(v), 2))
    t = []
    for y in range(n):
        for x in range(n):
            a = y * (n + 1) + x
            t += [(a, a + 1, a + n + 2), (a, a + n + 2, a + n + 1)]
    return v.astype(np.float32), np.array(t, np.int32)


def bowtie():
    """Two fans that share one vertex (0): vertex 0 is frozen."""
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0.1], [-1, 0, 0], [-1, -1, 0], [0, -1, 0.1]], np.float32)
    t = np.array([[0, 1, 2], [0, 2, 3], [0, 4, 5], [0, 5, 6]], np.int32)
    return v, t


def tetrahedron():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    t = np.array([[0, 2, 1], [0, 1, 3], [1, 2, 3], [0, 3, 2]], np.int32)
    return v, t


def three_faces():
    """A grid with one more face on its interior edge (a, a + n + 2): both ends are frozen."""
    v, t = grid(4)
    a = 1 * 5 + 1
    v = np.concatenate([v, [[1.5, 1.5, 1.0]]]).astype(np.float32)
    return v, np.concatenate([t, [[a, a + 6, len(v) - 1]]]).astype(np.int32), (a, a + 6)


def flipped():
    """A grid with one face reversed: its edges are traversed twice in the same direction, its corners are frozen."""
    v, t = grid(4)
    t = t.copy()
    k = 2 * (1 * 4 + 1)
    t[k] = t[k][::-1]
    return v, t, t[k].copy()


def _jitter(v, amount, seed):
    rng = np.random.default_rng(seed)
    return (v.astype(np.float64) + rng.uniform(-amount, amount, v.shape)).astype(np.float32)


def sphere_mesh(N=24, radius=8.3, jitter=0.0, seed=0):
    """Marching tetrahedra of mesh_cases.sphere_field (grid units), and the analytic centre and radius."""
    m = mo.extract(mc.sphere_field(N, radius), 0.0)
    v = _jitter(m["vertices"], jitter, seed) if jitter else m["vertices"]
    return v, m["triangles"].astype(np.int32), np.full(3, N / 2 + 0.137), radius


def torus_mesh(N=24, R=7.0, r=2.6, jitter=0.0, seed=0):
    m = mo.extract(mc.torus_field(N, R, r), 0.0)
    v = _jitter(m["vertices"], jitter, seed) if jitter else m["vertices"]
    return v, m["triangles"].astype(np.int32), np.full(3, N / 2 + 0.137), (R, r)


def torus_distance(P, c, R, r):
    p = np.asarray(P, np.float64) - c
    return np.abs(np.sqrt((np.sqrt(p[:, 0] ** 2 + p[:, 1] ** 2) - R) ** 2 + p[:, 2] ** 2) - r)


def sheet_mesh(depth=5, jitter=0.0, seed=0, n=40000):
    """The screened oracle's mesh of the wavy sheet, trimmed at 0.5 (world units), and its grid spacing h."""
    import mesh_screened_cases as msc
    import mesh_screened_oracle as so
    x, nr = msc.sheet(n, seed=1)
    m = so.mesh(x, nr, depth=depth, alpha=4.0, trim=0.5)
    v = _jitter(m["vertices"], jitter * m["h"], seed) if jitter else m["vertices"]
    return v, m["triangles"].astype(np.int32), m["h"]
