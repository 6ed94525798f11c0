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


# ---- meshes for the rule-by-rule GPU checks (tests/test_simplify_rules_gpu.py) ----------------------------------------
def _mesh(v, t):
    return np.asarray(v, np.float64).astype(np.float32), np.asarray(t, np.int32).reshape(-1, 3)


def two_chains():
    """Vertex 0 holds two open chains of faces (three and two faces) that leave it in different directions, not in one
    plane: 0 is frozen."""
    v = [[0, 0, 0], [1, 0, 0.2], [1, 1, 0], [0, 1, 0.3], [-1, 1, 0.1], [-1, -1, 0.4], [0, -1, 0], [1, -1, 0.5]]
    t = [[0, 1, 2], [0, 2, 3], [0, 3, 4], [0, 5, 6], [0, 6, 7]]
    return _mesh(v, t)


def cycle_and_chain():
    """Vertex 0 is the centre of a closed hexagonal fan and also of an open chain of two faces above it: 0 is frozen,
    the rim of the hexagon is a boundary."""
    a = np.arange(6) * np.pi / 3
    v = [[0, 0, 0]] + [[np.cos(x), np.sin(x), 0.1 * (k % 2)] for k, x in enumerate(a)]
    v += [[0.2, 0.1, 1.0], [0.5, -0.4, 1.2], [-0.3, 0.2, 1.1]]
    t = [[0, 1 + k, 1 + (k + 1) % 6] for k in range(6)] + [[0, 7, 8], [0, 8, 9]]
    return _mesh(v, t)


def four_faces():
    """grid(4) with two more faces on its interior edge (a, a + 6), one in each direction: four faces on one edge."""
    v, t = grid(4)
    a = 1 * 5 + 1
    v = np.concatenate([v, [[1.5, 1.5, 1.0], [1.5, 1.5, -1.0]]]).astype(np.float32)
    return v, np.concatenate([t, [[a, a + 6, len(v) - 2], [a + 6, a, len(v) - 1]]]).astype(np.int32)


def mobius(n=12, w=0.3):
    """A Moebius strip of n quads (2n faces): along the seam that closes it two faces traverse edges in the same
    direction, so the seam's vertices are frozen and the rest is an open manifold band."""
    v = []
    for i in range(n):
        a = 2 * np.pi * i / n
        for s in (-w, w):
            r = 1 + s * np.cos(a / 2)
            v.append([r * np.cos(a), r * np.sin(a), s * np.sin(a / 2)])
    t = []
    for i in range(n):
        a0, a1 = 2 * i, 2 * i + 1
        if i + 1 < n:
            b0, b1 = 2 * i + 2, 2 * i + 3
        else:
            b0, b1 = 1, 0       # the half twist: the inner rail joins the outer one
        t += [(a0, b0, b1), (a0, b1, a1)]
    return _mesh(v, t)


def repeated_face():
    """grid(4) with face 9 listed twice in the same order: its corners are frozen."""
    v, t = grid(4)
    return v, np.concatenate([t, t[9:10]]).astype(np.int32)


def pillow():
    """Two faces on the same three vertices, (a, b, c) and (a, c, b): closed, every edge refused (the apexes of each
    edge are the same vertex)."""
    return _mesh([[0, 0, 0], [1, 0, 0], [0, 1, 0.5]], [[0, 1, 2], [0, 2, 1]])


def collapsed_rows(n=5, coincident=False):
    """grid(n) with row 1 moved onto row 0's line (y = 0): the faces between them are collinear (zero area), so the
    vertices of row 0 have only zero-area faces (A = 0, quadric 0).  With coincident the rows also share x, so each
    vertex of row 1 coincides with the one below it."""
    v, t = grid(n)
    v = v.copy()
    row = slice(n + 1, 2 * (n + 1))
    v[row, 1] = 0
    if not coincident:
        v[row, 0] += 0.5
    return v, t


def folded_grid(n=8, slope=0.7):
    """A flat grid folded along x = n / 2 (a roof): the vertices on the fold have rank-2 quadrics."""
    v, t = grid(n)
    v = v.astype(np.float64)
    v[:, 2] = slope * np.abs(v[:, 0] - n / 2)
    return v.astype(np.float32), t


def box(n=4):
    """The closed surface of the cube [0, n]^3 with n x n unit squares per side, outward: rank-3 quadrics at the
    corners, rank 2 on the edges, rank 1 elsewhere."""
    index, v, t = {}, [], []

    def vid(p):
        k = tuple(int(c) for c in p)
        if k not in index:
            index[k] = len(v)
            v.append(k)
        return index[k]

    for axis in range(3):
        for side in (0, n):
            u_ax, w_ax = [a for a in range(3) if a != axis]
            for i in range(n):
                for j in range(n):
                    q = []
                    for di, dj in ((0, 0), (1, 0), (1, 1), (0, 1)):
                        p = [0, 0, 0]
                        p[axis], p[u_ax], p[w_ax] = side, i + di, j + dj
                        q.append(vid(p))
                    # (u, w, axis) is right-handed for axis 0 and 2 and left-handed for 1
                    out = (side == n) == (axis != 1)
                    f = [(q[0], q[1], q[2]), (q[0], q[2], q[3])]
                    t += f if out else [tuple(reversed(x)) for x in f]
    return _mesh(v, t)


def tilted_grid(n=8, jitter=0.0, seed=0):
    """grid(n) rotated off every axis (and shifted), so each coordinate is rounded to float32: every error of the flat
    mesh is rounding noise rather than an exact 0."""
    v, t = grid(n, jitter, seed)
    c, s = np.cos, np.sin
    a, b, g = 0.37, 0.61, 0.23
    R = (np.array([[c(a), -s(a), 0], [s(a), c(a), 0], [0, 0, 1]]) @
         np.array([[c(b), 0, s(b)], [0, 1, 0], [-s(b), 0, c(b)]]) @
         np.array([[1, 0, 0], [0, c(g), -s(g)], [0, s(g), c(g)]]))
    return (v.astype(np.float64) @ R.T + [0.3, -1.7, 2.9]).astype(np.float32), t


def bumpy_grid(n=7, seed=0, amount=0.3):
    """grid(n) with every vertex jittered in z and in the plane: a small open mesh where every error differs."""
    v, t = grid(n, 0.2, seed)
    v = v.astype(np.float64)
    v[:, 2] = np.random.default_rng(seed + 1).uniform(-amount, amount, len(v))
    return v.astype(np.float32), t


def fan(k, closed=False, seed=0):
    """Centre 0 and k rim vertices on a wavy arc: k - 1 faces (an open fan, k faces closed), every face holding the
    centre, so every closed 1-ring holds it too."""
    a = 2 * np.pi * np.arange(k) / k if closed else np.linspace(0, 1.7 * np.pi, k)
    rng = np.random.default_rng(seed)
    r = 1 + 0.05 * rng.uniform(-1, 1, k)
    v = [[0, 0, 0.2]] + [[r[i] * np.cos(x), r[i] * np.sin(x), 0.1 * np.sin(5 * x)] for i, x in enumerate(a)]
    m = k if closed else k - 1
    return _mesh(v, [[0, 1 + i, 1 + (i + 1) % k] for i in range(m)])


def strip(T, seed=0):
    """A band of T triangles on T + 2 vertices (two rails, z jittered): face i is (i, i + 1, i + 2), every other one
    reversed so the band is oriented."""
    rng = np.random.default_rng(seed)
    i = np.arange(T + 2)
    v = np.stack([i // 2, i % 2, 0.2 * rng.uniform(-1, 1, T + 2)], 1)
    t = [(k, k + 1, k + 2) if k % 2 == 0 else (k + 1, k, k + 2) for k in range(T)]
    return _mesh(v, t)


def permuted(v, t, seed, inten=None):
    """The same mesh with vertex ids permuted, triangles shuffled and each triangle's corners rotated."""
    rng = np.random.default_rng(seed)
    V = len(v)
    perm = rng.permutation(V)                 # new id of old vertex x is perm[x]
    inv = np.argsort(perm)
    nt = perm[np.asarray(t)][rng.permutation(len(t))]
    rot = rng.integers(0, 3, len(nt))
    nt = np.stack([np.roll(f, -r) for f, r in zip(nt, rot)]).astype(np.int32)
    return v[inv], nt, None if inten is None else inten[inv]


def with_unused(v, t, factor=10, nan_every=7, seed=0, inten=None):
    """The mesh's vertices spread among factor x V unused ones (random positions, every nan_every-th one NaN)."""
    rng = np.random.default_rng(seed)
    V = len(v)
    N = V * (factor + 1)
    slots = np.sort(rng.choice(N, V, replace=False))
    out = rng.uniform(-5, 5, (N, 3)).astype(np.float32)
    unused = np.setdiff1d(np.arange(N), slots)
    out[unused[::nan_every]] = np.nan
    out[slots] = v
    oi = None
    if inten is not None:
        oi = rng.uniform(0, 1, N).astype(np.float32)
        oi[slots] = inten
    return out, slots[np.asarray(t)].astype(np.int32), oi


def components(*meshes):
    """Several meshes in one vertex and triangle list, each shifted apart."""
    vs, ts, base = [], [], 0
    for k, (v, t) in enumerate(meshes):
        vs.append(np.asarray(v, np.float64) + [40.0 * k, 0, 0])
        ts.append(np.asarray(t, np.int64) + base)
        base += len(v)
    return np.concatenate(vs).astype(np.float32), np.concatenate(ts).astype(np.int32)
