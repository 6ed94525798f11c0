"""Hand-made meshes for cs_clean_mesh: a grid with holes of 3, 4, 8 and 40 edges, a fin, duplicate faces (one
reversed), zero-area faces, a bowtie vertex on a hole rim, and a sphere with holes, islands and a long-edge sliver
fan.  Each returns (vertices float32 [V, 3], triangles int32 [T, 3], intensity float32 [V])."""
import numpy as np


def _inten(V):
    return np.linspace(0.0, 1.0, V).astype(np.float32)


def grid(n=30, h=1.0, drop=()):
    """An n x n grid of cells, two faces per cell (counter-clockwise seen from +z); cells in drop are left out."""
    ij = np.stack(np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing="ij"), -1).reshape(-1, 2)
    v = np.c_[ij * h, np.zeros(len(ij))].astype(np.float32)
    vid = lambda i, j: i * (n + 1) + j
    drop = set(drop)
    t = []
    for i in range(n):
        for j in range(n):
            if (i, j) in drop:
                continue
            a, b, c, d = vid(i, j), vid(i + 1, j), vid(i + 1, j + 1), vid(i, j + 1)
            t += [(a, b, c), (a, c, d)]
    return v, np.array(t, np.int32)


def _cells(i0, j0, w):
    return [(i, j) for i in range(i0, i0 + w) for j in range(j0, j0 + w)]


def holes():
    """Holes of 4 (one cell), 8 (2 x 2 cells), 40 (10 x 10 cells) and 3 edges (one face) in a 30 x 30 grid."""
    v, t = grid(30, drop=_cells(3, 3, 1) + _cells(8, 3, 2) + _cells(15, 15, 10))
    a = 20 * 31 + 4                                             # one face of cell (20, 4), away from the others
    t = np.delete(t, np.flatnonzero((t == [a, a + 31, a + 32]).all(1)), axis=0)
    return v, t, _inten(len(v))


def fin():
    """A third face (to a vertex above the grid) on one interior edge of a 10 x 10 grid."""
    v, t = grid(10)
    top = len(v)
    v = np.r_[v, [[2.5, 2.5, 1.0]]].astype(np.float32)
    a, b = t[20, 0], t[20, 2]                                   # the diagonal of a cell
    t = np.r_[t, [[a, b, top]]].astype(np.int32)
    return v, t, _inten(len(v))


def duplicates():
    """A reversed copy of face 10 in front of a 10 x 10 grid, and a plain copy of face 20 and a rotated one of face 5 at its end."""
    v, t = grid(10)
    t = np.r_[t[10:11, ::-1], t, t[20:21], t[[5]][:, [1, 2, 0]]].astype(np.int32)
    return v, t, _inten(len(v))


def zero_area():
    """A 10 x 10 grid with a collinear face along a row and a face with two coincident vertices."""
    v, t = grid(10)
    extra = len(v)
    v = np.r_[v, v[12:13]].astype(np.float32)                     # a copy of vertex 12's position
    t = np.r_[t[:4], [[0, 11, 22]], t[4:], [[12, 13, extra]]].astype(np.int32)
    return v, t, _inten(len(v))


def bowtie():
    """Two holes of one cell that touch at a corner of a 10 x 10 grid: the rim vertex has two boundary half-edges in
    and two out, so neither hole is a loop."""
    v, t = grid(10, drop=[(3, 3), (4, 4)])
    return v, t, _inten(len(v))


def icosphere(level=3):
    p = (1 + 5 ** 0.5) / 2
    v = [(-1, p, 0), (1, p, 0), (-1, -p, 0), (1, -p, 0), (0, -1, p), (0, 1, p), (0, -1, -p), (0, 1, -p), (p, 0, -1),
         (p, 0, 1), (-p, 0, -1), (-p, 0, 1)]
    v = [np.array(x, np.float64) / np.linalg.norm(x) for x in v]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
         (8, 6, 7), (9, 8, 1)]
    for _ in range(level):
        mid = {}

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                x = v[a] + v[b]
                v.append(x / np.linalg.norm(x))
                mid[k] = len(v) - 1
            return mid[k]
        f = [g for a, b, c in f for g in ((a, m(a, b), m(c, a)), (b, m(b, c), m(a, b)), (c, m(c, a), m(b, c)),
                                          (m(a, b), m(b, c), m(c, a)))]
    return np.array(v, np.float32), np.array(f, np.int32)


def sphere_mess(level=3):
    """An icosphere with a hole of one face and one of a vertex's whole 1-ring (its centre unused), three islands of
    8 faces, and a sliver fan of 6 faces from a far apex to a chain of sphere vertices."""
    v, t = icosphere(level)
    ring = np.flatnonzero((t == 40).any(1))
    t = np.delete(t, np.r_[ring, [len(t) - 7]], axis=0)
    parts = [v]
    tris = [t]
    off = len(v)
    for k in range(3):
        gv, gt = grid(2, h=0.05)
        parts.append(gv + np.float32([3.0 + k, 0.0, 0.0]))
        tris.append(gt + off)
        off += len(gv)
    apex = off
    parts.append(np.float32([[0.0, 0.0, 9.0]]))
    chain = t[:7, 0]
    tris.append(np.array([[chain[i], chain[i + 1], apex] for i in range(6) if chain[i] != chain[i + 1]], np.int32))
    v = np.concatenate(parts).astype(np.float32)
    return v, np.concatenate(tris).astype(np.int32), _inten(len(v))


def enclosed_slivers():
    """A 10 x 10 grid whose cell (4, 4) is split into a zero-area face between its two halves: the cell's diagonal
    vertex is moved onto the diagonal's midpoint, so three faces meet there and one of them has zero area; every edge of
    that face is held by another face."""
    v, t = grid(10)
    mid = len(v)
    a, b, c, d = 4 * 11 + 4, 5 * 11 + 4, 5 * 11 + 5, 4 * 11 + 5
    v = np.r_[v, [(v[a] + v[c]) / 2]].astype(np.float32)
    k = np.flatnonzero((t == [a, b, c]).all(1))[0]
    t = np.r_[t[:k], [[a, b, mid], [mid, b, c], [a, mid, c]], t[k + 1:]].astype(np.int32)
    return v, t, _inten(len(v))


CASES = {"holes": holes, "enclosed_slivers": enclosed_slivers, "fin": fin, "duplicates": duplicates, "zero_area": zero_area, "bowtie": bowtie,
         "sphere_mess": sphere_mess}
# the settings each case is run with (besides the defaults)
SETTINGS = {"holes": dict(maxHoleEdges=40), "sphere_mess": dict(longEdgeFactor=3.0), "bowtie": dict(maxHoleEdges=8)}


def sheet_meshes():
    """mesh_screened_cases.sheet(20000) meshed by the screened oracle at depth 5, trim 0.5 and 1.0."""
    import mesh_screened_cases as msc
    import mesh_screened_oracle as so
    x, n = msc.sheet(20000, seed=0)[:2]
    out = {}
    for trim in (0.5, 1.0):
        r = so.mesh(x, n, depth=5, trim=trim)
        out[trim] = (np.asarray(r["vertices"], np.float32), np.asarray(r["triangles"], np.int32))
    return out


def punch(v, t, seed=0, rings=100, faces=100, islands=5):
    """A closed mesh with holes of several sizes and islands added: the faces of `rings` random vertices' 1-rings and
    `faces` random single faces removed (holes of 3 edges up to a few merged rings), then `islands` 8-face grids far
    outside the mesh's box."""
    rng = np.random.default_rng(seed)
    t = np.asarray(t, np.int32)
    centres = rng.choice(len(v), rings, replace=False)
    gone = np.isin(t, centres).any(1)
    gone[rng.choice(len(t), faces, replace=False)] = True
    t = t[~gone]
    lo, hi = v.min(0), v.max(0)
    parts, tris, off = [v], [t], len(v)
    for k in range(islands):
        gv, gt = grid(2, h=0.01 * float((hi - lo).max()))
        parts.append(gv + (hi + (k + 1) * 0.1 * (hi - lo)).astype(np.float32))
        tris.append(gt + off)
        off += len(gv)
    return np.concatenate(parts).astype(np.float32), np.concatenate(tris).astype(np.int32)
