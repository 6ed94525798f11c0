"""Inputs for seam levelling (cs_level_texture_seams), one generator per rule of the header, each built directly rather
than through TextureMesh so that every chart, corner and seam edge is placed on purpose.  A case is a dict of v, t,
labels, uv, charts, atlas and kw (the call's keyword arguments).  Each face's uv is its own: faces that share a vertex
need not share its uv, so both sides of a seam edge get the lengths and positions a rule needs.  Vertex ids are
permuted, faces shuffled and corners rotated within each face (where corner 0 stays in the same chart), and atlas
values span six orders of magnitude so that a change in any summation order changes the bits; texels outside every
chart hold NaN (with a payload), -0.0 and infinities, which the call must copy bit for bit."""
import numpy as np

import seam_oracle as so

QNAN = np.array([0x7FC0BEEF], np.uint32).view(np.float32)[0]
OUTSIDE = np.array([QNAN, -0.0, np.inf, -np.inf, 0.0], np.float32)


class _Mesh:
    """Faces with their own uv, in chart-local texels of their label's chart (charts[label] -> (ox, oy))."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.v, self.t, self.lab, self.uv = [], [], [], []

    def verts(self, n):
        base = len(self.v)
        self.v += list(self.rng.uniform(-10, 10, (n, 3)))
        return list(range(base, base + n))

    def face(self, ids, label, uvs):
        self.t.append(list(ids))
        self.lab.append(label)
        self.uv.append([list(map(float, p)) for p in uvs])

    def near(self, p, r=2.5):
        return np.asarray(p, np.float64) + self.rng.uniform(-r, r, 2)

    def case(self, charts, rows, width, seed, atlas=None, rotate=True, **kw):
        charts = np.asarray(charts, np.int32).reshape(-1, 8)
        v, t = np.asarray(self.v, np.float32), np.asarray(self.t, np.int64)
        uv, lab = np.asarray(self.uv, np.float32).reshape(-1, 3, 2), np.asarray(self.lab, np.int32)
        if atlas is None:
            atlas = make_atlas(rows, width, charts, seed)
        return shuffle(dict(v=v, t=t, labels=lab, uv=uv, charts=charts, atlas=atlas, kw=kw), seed, rotate)


def make_atlas(rows, width, charts, seed, inside=None):
    """Chart texels 10^u for u uniform in [-2, 4) (or `inside`), every other texel one of OUTSIDE."""
    rng = np.random.default_rng(seed + 1000)
    a = OUTSIDE[rng.integers(0, len(OUTSIDE), (rows, width))]
    for e in charts:
        blk = (10.0 ** rng.uniform(-2, 4, (e[4], e[3]))) if inside is None else np.full((e[4], e[3]), inside)
        a[e[6]:e[6] + e[4], e[5]:e[5] + e[3]] = blk
    return a.astype(np.float32)


def shuffle(c, seed, rotate=True, unused=5):
    """Vertex ids permuted (with unused vertices, every other one NaN), faces in random order, and each face's corners
    rotated by 0, 1 or 2 where its rotated corner 0 lands in the same chart (rule 1 reads corner 0 only)."""
    rng = np.random.default_rng(seed)
    v, t, lab, uv = c["v"], c["t"], c["labels"], c["uv"]
    extra = rng.uniform(-50, 50, (unused, 3)).astype(np.float32)
    extra[::2] = np.nan
    allv = np.concatenate([v, extra])
    perm = rng.permutation(len(allv))
    nv = np.empty_like(allv)
    nv[perm] = allv
    fo = rng.permutation(len(t))
    t, lab, uv = perm[t][fo], lab[fo], uv[fo]
    if rotate:
        rows, width = c["atlas"].shape
        t, uv = t.copy(), uv.copy()
        for f in range(len(t)):
            r = int(rng.integers(0, 3))
            if not r:
                continue
            ru = np.roll(uv[f], -r, axis=0)
            if lab[f] < 0 or not np.isfinite(uv[f]).all() or \
                    so.chart_of(ru, lab[f], c["charts"], rows, width) == so.chart_of(uv[f], lab[f], c["charts"],
                                                                                   rows, width) >= 0:
                t[f], uv[f] = np.roll(t[f], -r), ru
    return dict(c, v=nv, t=t.astype(np.int32), labels=lab, uv=uv)


def _at(charts, label):
    e = charts[[i for i, x in enumerate(charts) if x[0] == label][0]]
    return np.array([e[5], e[6]], np.float64)


# ---- rule 1: the chart lookup ---------------------------------------------------------------------------------------
LOOKUP_W, LOOKUP_ROWS = 128, 16
ROW0 = [3, 10, 10, 41, 17, 96, 5, 10, 63, 2, 88, 11, 47, 31, 74, 6, 59, 20, 8, 90, 27, 14, 35, 52]
ROW1 = [10, 5, 72, 3, 63, 66, 14, 90, 81, 17]
ROW1_OX = [0, 12, 24, 36, 48, 62, 74, 86, 98, 110]          # a 2-texel gap at x = 60, 61


def lookup_charts():
    """Shelf 0: 24 touching 5 x 6 charts from x = 0 to 120 (x 120..127 in no chart); shelf 1: 10 charts 12 x 7 at
    y = 6 with a gap at x = 60..61; rows 13..15 in no chart.  Labels repeat across charts and are not contiguous."""
    c = [[l, 0, 0, 5, 6, 5 * i, 0, 0] for i, l in enumerate(ROW0)]
    c += [[l, 0, 0, 12, 7, ox, 6, 0] for l, ox in zip(ROW1, ROW1_OX)]
    return np.array(c, np.int32)


def lookup(variant="valid", seed=11):
    """Rule 1.  Seam pairs across every pair of touching charts in shelf 0: the left face's corner 0 in its chart's last
    column (x = ox + 4.75), the right face's exactly on the left chart's exclusive right edge (x = ox + 5.0, which is
    the right chart's first column); pairs across the shelves with corner 0 in shelf 0's last row (y = 5.75) and exactly
    on its exclusive bottom edge (y = 6.0); a corner 0 exactly on a chart's top-left corner; the other corners anywhere
    near, inside or outside the chart.  An unseen face with NaN uv.  Each invalid variant breaks one face or vertex."""
    charts = lookup_charts()
    m = _Mesh(seed)
    for i in range(len(ROW0) - 1):
        P, Q, R, S = m.verts(4)
        a = np.array([5 * i + 4.75, 2.5])
        b = np.array([5 * i + 5.0, 3.0 if i % 2 else 0.0])
        m.face((P, Q, R), ROW0[i], [a, m.near(a), m.near(a)])
        m.face((Q, P, S), ROW0[i + 1], [b, m.near(b), m.near(b)])
    for j, ox in enumerate(ROW1_OX):
        P, Q, R, S = m.verts(4)
        i = (ox + 3) // 5
        a = np.array([ox + 3.5, 5.75])
        b = np.array([ox + 3.0 + 0.5 * (j % 2), 6.0])
        m.face((P, Q, R), ROW0[i], [a, m.near(a), m.near(a)])
        m.face((Q, P, S), ROW1[j], [b, m.near(b), m.near(b)])
    P, Q, R = m.verts(3)
    m.face((P, Q, R), ROW1[9], [(110.0, 6.0), (109.0, 5.0), (111.0, 4.0)])   # the top-left texel, the others outside
    m.face((Q, P, m.verts(1)[0]), -1, [(np.nan, np.nan)] * 3)
    c = m.case(charts, LOOKUP_ROWS, LOOKUP_W, seed, rotate=False)
    return _break(c, variant)


# the invalid variants: the uv of corner 0 of face 0 (before the shuffle, the first seam pair's left face) moved, or
# one index, vertex, uv coordinate or label of a seen face broken
INVALID = ["gap", "gap_between", "right_edge", "bottom_edge", "past_width", "past_rows", "negative_x",
           "negative_index", "repeated_vertex", "nan_vertex", "inf_uv", "nan_uv", "label_plus_1000", "overlap"]


def _break(c, variant):
    if variant == "valid":
        return c
    c = dict(c, v=c["v"].copy(), t=c["t"].copy(), uv=c["uv"].copy(), labels=c["labels"].copy(),
             charts=c["charts"].copy())
    seen = np.flatnonzero(c["labels"] >= 0)
    # the face of label ROW0[0] = 3 whose corner 0 is in chart 0 (x in [0, 5), y in [0, 6))
    f = int([g for g in seen if c["labels"][g] == 3 and c["uv"][g, 0, 0] < 5][0])
    u = c["uv"][f]
    moves = {"gap": (121.5, 2.0), "gap_between": (60.5, 8.0), "right_edge": (5.0, 2.0), "bottom_edge": (2.0, 6.0),
             "past_width": (128.0, 2.0), "past_rows": (2.0, 16.0), "negative_x": (-0.25, 2.0)}
    if variant in moves:
        u[0] = moves[variant]
    elif variant == "overlap":
        # chart 0 (label 3) widened over charts 1..7 and face f's corner 0 moved to x = 22.5: the first chart of label
        # 3 that holds it is chart 0, the last chart of the row index with ox <= 22 is chart 4 (label 17)
        c["charts"][0] = [3, 0, 0, 40, 6, 0, 0, 0]
        u[0] = (22.5, 2.0)
    elif variant == "negative_index":
        c["t"][f, 1] = -1
    elif variant == "repeated_vertex":
        c["t"][f, 2] = c["t"][f, 0]
    elif variant == "nan_vertex":
        c["v"][c["t"][f, 2]] = [0.0, np.nan, 0.0]
    elif variant == "inf_uv":
        u[2, 1] = np.inf
    elif variant == "nan_uv":
        u[1, 0] = np.nan
    elif variant == "label_plus_1000":
        c["labels"][f] += 1000
    else:
        raise ValueError(variant)
    return c


# ---- rule 3: the seam samples ---------------------------------------------------------------------------------------
SAMPLE_LABELS = [5, 12, 300, 77777, 2 ** 31 - 2, 9, 1 << 20, 46]
SAMPLE_W = 2608


def sample_charts():
    """One chart per label, 10 rows each: the first two 2600 wide (room for an edge 2500 texels long), the rest 200;
    the last 3 atlas rows and every column right of a chart in no chart."""
    return np.array([[l, 0, 0, 2600 if k < 2 else 200, 10, 0, 10 * k, 0] for k, l in enumerate(SAMPLE_LABELS)],
                    np.int32)


def samples(seed=21):
    """Rule 3.  Seam edges (labels L0 = 5 and L1 = 12 unless noted), each side's uv placed on purpose:
    a uv length of 0 on one side and on both (S = 1); lengths of exactly 5 (3-4-5) against 2 (S = 5 by ceil of an
    integer) and 5 + 2^-16 (S = 6); 2500.5 texels (S = 2501); samples at integer texel positions on both sides
    (fx = fy = 0); a side along its chart's last column and row, and one whose far end leaves its chart and the atlas
    (taps clamped to the chart); an edge held by 3 faces and one by 4 (no seam); a seam with one side unseen (no seam);
    a fan of 6 faces of alternating labels around one vertex (6 seam edges between the same labels meet there: one row
    sums 6 ends in edge-key order); a fan of 8 faces with 8 labels around one vertex (28 label pairs, 7 seam rows);
    labels up to 2^31 - 2."""
    charts = sample_charts()
    L = SAMPLE_LABELS
    m = _Mesh(seed)
    col = {l: 2.0 for l in L}

    def spot(l, w=6.0):
        x = col[l]
        col[l] += w
        return x

    def pair(la, lb, pa, qa, pb, qb, ra=None, rb=None):
        """Two faces on edge (P, Q): side la with P, Q at pa, qa (local to la's chart), side lb at pb, qb."""
        P, Q, R, S = m.verts(4)
        oa, ob = _at(charts, la), _at(charts, lb)
        ra = m.near(pa, 2.0) if ra is None else ra
        rb = m.near(pb, 2.0) if rb is None else rb
        m.face((P, Q, R), la, [oa + pa, oa + qa, oa + np.asarray(ra)])
        m.face((P, S, Q), lb, [ob + pb, ob + np.asarray(rb), ob + qb])
        return P, Q

    x = spot(L[0]), spot(L[1])
    pair(L[0], L[1], (x[0], 3.0), (x[0], 3.0), (x[1] + 0.5, 2.5), (x[1] + 3.8, 2.9))        # 0 on one side
    x = spot(L[0]), spot(L[1])
    pair(L[0], L[1], (x[0] + 1.5, 4.5), (x[0] + 1.5, 4.5), (x[1] + 2.25, 6.0), (x[1] + 2.25, 6.0))   # 0 on both
    x = spot(L[0]), spot(L[1])
    pair(L[0], L[1], (x[0], 1.0), (x[0] + 3.0, 5.0), (x[1], 2.0), (x[1] + 2.0, 2.0))        # exactly 5 against 2
    x = spot(L[0]), spot(L[1])
    pair(L[0], L[1], (x[0], 2.0), (x[0] + 5.0 + 2.0 ** -16, 2.0), (x[1], 7.0), (x[1] + 1.0, 7.5))   # 5 + 2^-16
    x = spot(L[0], 2508.0), spot(L[1])
    pair(L[0], L[1], (x[0], 4.25), (x[0] + 2500.5, 4.25), (x[1], 5.0), (x[1] + 1.5, 6.0))   # S = 2501
    x = spot(L[0]), spot(L[1])
    pair(L[0], L[1], (x[0] + 0.5, 4.0), (x[0] + 6.5, 4.0), (x[1] + 0.5, 1.0), (x[1] + 6.5, 1.0))    # fx = fy = 0
    # clamped taps: along the last column and row of L2's 200 x 10 chart, and a far end outside chart and atlas
    pair(L[2], L[3], (199.25, 9.5), (199.75, 5.5), (1.0, 9.8), (-3.5, 12.25), ra=(198.0, 8.0), rb=(3.0, 8.0))
    pair(L[2], L[3], (196.5, 9.75), (190.0, 9.75), (10.0, 3.0), (204.5, -7.5), ra=(193.0, 8.5), rb=(12.0, 2.0))
    # 3 and 4 faces on one edge, and a seam with one side unseen
    for labels in ((L[0], L[1], L[2]), (L[0], L[1], L[0], L[3])):
        P, Q = m.verts(2)
        for l in labels:
            o = _at(charts, l) + (spot(l), 5.0)
            m.face((P, Q, m.verts(1)[0]), l, [o, m.near(o), m.near(o)])
    P, Q, R, S = m.verts(4)
    o = _at(charts, L[0]) + (spot(L[0]), 5.0)
    m.face((P, Q, R), L[0], [o, m.near(o), m.near(o)])
    m.face((Q, P, S), -1, [(np.nan, 0.0)] * 3)
    # fans: 6 faces of alternating labels, 8 faces of 8 labels
    for labels in ([L[0], L[1]] * 3, L):
        C = m.verts(1)[0]
        ring = m.verts(len(labels))
        for k, l in enumerate(labels):
            o = _at(charts, l) + (spot(l), 5.0)
            m.face((C, ring[k], ring[(k + 1) % len(labels)]), l, [o, m.near(o, 3.5), m.near(o, 3.5)])
    return m.case(charts, 83, SAMPLE_W, seed)


# ---- rules 4-6: the rows and the solve ------------------------------------------------------------------------------
def grid(n=10, labels=(4, 19, 7), seed=31, inside=None, **kw):
    """An n x n grid of cells (two faces each) whose labels come in blocks of 3 x 3 cells, each face's uv a small
    triangle anywhere in its label's 64 x 64 chart."""
    m = _Mesh(seed)
    ids = np.array(m.verts((n + 1) * (n + 1))).reshape(n + 1, n + 1)
    charts = np.array([[l, 0, 0, 64, 64, 64 * k, 0, 0] for k, l in enumerate(labels)], np.int32)
    for i in range(n):
        for j in range(n):
            l = labels[(i // 3 + 2 * (j // 3)) % len(labels)]
            for tri in ((ids[i, j], ids[i, j + 1], ids[i + 1, j + 1]), (ids[i, j], ids[i + 1, j + 1], ids[i + 1, j])):
                o = _at(charts, l) + m.rng.uniform(3, 60, 2)
                m.face(tri, l, [o, m.near(o, 3.0), m.near(o, 3.0)])
    atlas = None if inside is None else make_atlas(64, 64 * len(labels), charts, seed, inside)
    return m.case(charts, 64, 64 * len(labels), seed, atlas, **kw)


SOLVE = {
    "smoothness_0": dict(smoothness=0.0),
    "smoothness_50": dict(smoothness=50.0),
    "regularization_1e-6": dict(regularization=1e-6),
    "regularization_1": dict(regularization=1.0),
    "tol_0": dict(tol=0.0, maxIterations=40),
    "max_iterations_0": dict(maxIterations=0),
}


def solve(name):
    """Rules 4-6 on grid() with one argument far from its default."""
    return grid(**SOLVE[name])


def constant():
    """b = 0: every chart texel 64 (a power of two, so every target is exactly 64): status 0 after 0 iterations."""
    return grid(inside=64.0)


def valence(n=3000, seed=41):
    """A closed fan of n faces of alternating labels around one vertex: its two unknowns have n smoothness rows and one
    seam row each (more than 11 pieces of 256 incidences), and its seam row sums n edge ends."""
    m = _Mesh(seed)
    charts = np.array([[6, 0, 0, 256, 256, 0, 0, 0], [13, 0, 0, 256, 256, 256, 0, 0]], np.int32)
    C = m.verts(1)[0]
    ring = m.verts(n)
    for k in range(n):
        l = (6, 13)[k % 2]
        o = _at(charts, l) + m.rng.uniform(3, 252, 2)
        m.face((C, ring[k], ring[(k + 1) % n]), l, [o, m.near(o, 2.0), m.near(o, 2.0)])
    return m.case(charts, 256, 512, seed)


def counts(rows, unknowns=None, seed=51):
    """Exactly `rows` seam rows (seam pairs: 2 rows and 6 unknowns; a 3-face strip a, b, a: 3 rows and 8 unknowns) and,
    when given, exactly `unknowns` unknowns (isolated faces: 3; isolated same-label pairs: 4)."""
    m = _Mesh(seed)
    charts = np.array([[1, 0, 0, 128, 128, 0, 0, 0], [2, 0, 0, 128, 128, 128, 0, 0]], np.int32)
    put = lambda l: _at(charts, l) + m.rng.uniform(3, 124, 2)

    def tri(ids, l):
        o = put(l)
        m.face(ids, l, [o, m.near(o, 2.0), m.near(o, 2.0)])

    triples, N = rows % 2, 0
    for _ in range(triples):
        C, r0, r1, r2, r3 = m.verts(5)
        tri((C, r0, r1), 1), tri((C, r1, r2), 2), tri((C, r2, r3), 1)
        N += 8
    for _ in range((rows - 3 * triples) // 2):
        P, Q, R, S = m.verts(4)
        tri((P, Q, R), 1), tri((Q, P, S), 2)
        N += 6
    if unknowns is not None:
        extra = unknowns - N
        assert extra >= 0 and extra not in (1, 2, 5), (rows, unknowns)
        fours = next(k for k in range(4) if (extra - 4 * k) % 3 == 0)
        for _ in range(fours):
            P, Q, R, S = m.verts(4)
            tri((P, Q, R), 2), tri((Q, P, S), 2)
        for _ in range((extra - 4 * fours) // 3):
            tri(m.verts(3), 1)
    return m.case(charts, 128, 256, seed)


COUNTS = {"rows_255_unknowns_2047": (255, 2047), "rows_256_unknowns_2048": (256, 2048),
          "rows_257_unknowns_2049": (257, 2049), "rows_2047": (2047, None), "rows_2048": (2048, None),
          "rows_2049_unknowns_6400": (2049, 6400)}


# ---- rule 7: the texels ---------------------------------------------------------------------------------------------
def texel_charts():
    """Label 4 at the atlas's top-left corner (20 x 16), label 9 touching it (18 x 16), label 1 away from every border
    (15 x 10 at (40, 3)); columns 38, 39 and 55..59, rows 16..19 and the rows above label 1 in no chart."""
    return np.array([[4, 0, 0, 20, 16, 0, 0, 0], [9, 0, 0, 18, 16, 20, 0, 0], [1, 0, 0, 15, 10, 40, 3, 0]], np.int32)


def texels(padding=2, seed=61):
    """Rule 7 at uv corners on integer texel centres: two faces of label 4 sharing a diagonal edge whose texels lie on
    it (the lower-vertex edge rule), seamed to label 9 and 1; a mirrored face (A < 0); a collinear face and one with three
    equal corners (A = 0); two faces exactly 1 texel either side of a texel between them (a key tie); two faces whose
    distances from a texel round to the same float but whose squares do not; faces in the corners of the atlas and of
    the charts (boxes clamped at chart and atlas borders)."""
    charts = texel_charts()
    m = _Mesh(seed)
    a, b, c, d = m.verts(4)
    m.face((a, b, c), 4, [(2, 2), (8, 2), (2, 8)])
    m.face((b, d, c), 4, [(8, 2), (8, 8), (2, 8)])
    e, f_ = m.verts(2)
    m.face((b, a, e), 9, [(27, 9), (21, 9), (24, 14)])                    # seam on (a, b)
    m.face((d, b, f_), 1, [(46, 10), (46, 4), (52, 7)])                   # seam on (b, d)
    g, h = m.verts(2)
    m.face((c, d, g), 9, [(22, 3), (30, 3), (26, 1)])                     # mirrored: A < 0; seam on (c, d)
    m.face((g, d, h), 4, [(11, 3), (13, 4), (15, 5)])                     # collinear
    m.face((h, g, m.verts(1)[0]), 9, [(33.5, 12.5)] * 3)                  # three equal corners
    i, j, k, l = m.verts(4)
    m.face((i, j, k), 4, [(13, 11), (14, 11), (13.5, 13)])                # texel (12, 11) is 1 from both
    m.face((j, i, l), 1, [(52, 11), (51, 11), (51.5, 9)])                 # texel (53, 11) ties with the next face
    p, q = m.verts(2)
    m.face((i, p, q), 1, [(54, 11), (54, 12.5), (54.5, 12)])
    r, s, u = m.verts(3)
    m.face((r, s, u), 4, [(11, 11), (10, 11), (10.5, 13)])
    m.face((s, r, m.verts(1)[0]), 9, [(37.5, 15.5), (36.25, 14.0), (37.75, 13.5)])   # chart corner
    m.face((p, q, m.verts(1)[0]), 4, [(0.25, 0.25), (1.5, 0.5), (0.5, 1.75)])        # atlas corner
    m.face((q, p, m.verts(1)[0]), 1, [(40.25, 3.5), (41.0, 3.0), (40.5, 4.5)])       # label 1's top-left
    # texels (17, 10) and (17, 5): the nearest corners of two faces at distances sqrt(2.0014651417...) and
    # sqrt(2.0014653801...), equal as floats but not as float squares
    for X, Y, first in ((17, 10, 0), (17, 5, 1)):
        near, far = np.array([X + 1.00048828125, Y + 1.000244140625]), np.array([X - 1.0, Y - 1.000732421875])
        faces = [[near, near + (1, 0), near + (0, 1)], [far, far - (1, 0), far - (0, 1)]]
        for k in (first, 1 - first):
            ids = m.verts(3)
            m.face(ids, 4, faces[k])
            o = np.array([31.0 + 3 * first + 1.5 * k, 6.0])            # a seam to label 9: an offset of its own
            m.face((ids[1], ids[0], m.verts(1)[0]), 9, [o, o + (1, 0.5), o + (0.5, 1.5)])
    return m.case(charts, 20, 60, seed, padding=padding)


# ---- an end order that reaches the seam energy -----------------------------------------------------------------------
def ends(n=8, seed=72):
    """Rule 3's end order where info[0] shows it: a fan of n faces of alternating labels 2 and 5 around one vertex
    (its row sums n edge ends), each seam edge 40 texels long, the centre's uv 3 texels apart on each face of label 2.
    Label 2's chart is 10^3..10^8 at the texels around those places and 10^-2..10^2 elsewhere, label 5's chart
    10^-2..10^2: the ends at the centre span orders of magnitude, so their order changes the row's F_a, and that row
    dominates the seam energy, so the change reaches the total's bits."""
    m = _Mesh(seed)
    charts = np.array([[2, 0, 0, 96, 96, 0, 0, 0], [5, 0, 0, 96, 96, 96, 0, 0]], np.int32)
    C = m.verts(1)[0]
    ring = m.verts(n)
    for k in range(n):
        l = (2, 5)[k % 2]
        o = _at(charts, l) + (40.25 + 3.0 * (k // 2), 48.5)
        ang = 2 * np.pi * np.array([k, k + 1]) / n
        r = [o + 40.0 * np.array([np.cos(x), np.sin(x)]) for x in ang]
        m.face((C, ring[k], ring[(k + 1) % n]), l, [o, r[0], r[1]])
    rng = np.random.default_rng(seed)
    atlas = make_atlas(96, 192, charts, seed)
    atlas[:, :192] = (10.0 ** rng.uniform(-2, 2, (96, 192))).astype(np.float32)
    atlas[46:52, 38:54] = (10.0 ** rng.uniform(3, 8, (6, 16))).astype(np.float32)
    return m.case(charts, 96, 192, seed, atlas)


# ---- scale: all three levels of the totals --------------------------------------------------------------------------
def scale(n=400, seed=81):
    """An n x n grid of cells (two faces each) whose labels 0..3 follow (i mod 2) + 2 (j mod 2): every inside vertex
    has 4 unknowns and 4 seam rows, so at n = 400 (320 000 faces) both counts pass 2048 x 256 = 524 288 and every
    total of the solve runs all three levels.  Each face's uv is a small triangle at its cell's place in its label's
    chart."""
    rng = np.random.default_rng(seed)
    ids = np.arange((n + 1) * (n + 1)).reshape(n + 1, n + 1)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    i, j = i.reshape(-1), j.reshape(-1)
    t = np.concatenate([np.stack([ids[i, j], ids[i, j + 1], ids[i + 1, j + 1]], 1),
                        np.stack([ids[i, j], ids[i + 1, j + 1], ids[i + 1, j]], 1)])
    lab = np.tile((i % 2) + 2 * (j % 2), 2).astype(np.int32)
    W = (n // 2) * 5 // 2 + 8
    charts = np.array([[l, 0, 0, W, W, W * (l % 2), W * (l // 2), 0] for l in range(4)], np.int32)
    cell = np.stack([np.tile(j // 2, 2), np.tile(i // 2, 2)], 1) * 2.5 + 2.0
    base = charts[lab][:, 5:7] + cell + np.r_[np.zeros((n * n, 2)), np.full((n * n, 2), 0.75)]
    uv = base[:, None, :] + rng.uniform(0, 1.5, (len(t), 3, 2))
    uv[:, 0] = base
    v = np.concatenate([rng.uniform(-1, 1, ((n + 1) * (n + 1), 2)), np.zeros(((n + 1) * (n + 1), 1))], 1)
    atlas = make_atlas(2 * W, 2 * W, charts, seed)
    return dict(v=v.astype(np.float32), t=t.astype(np.int32), labels=lab, uv=uv.astype(np.float32), charts=charts,
                atlas=atlas, kw={})


# ---- the small cases by name ----------------------------------------------------------------------------------------
CASES = {"lookup": lookup, "samples": samples, "ends": ends, "constant": constant, "valence": valence,
         "texels_pad0": lambda: texels(0), "texels_pad2": texels, "texels_pad5": lambda: texels(5),
         "texels_pad16": lambda: texels(16)}
CASES.update({"solve_" + k: (lambda k=k: solve(k)) for k in SOLVE})
CASES.update({"counts_" + k: (lambda a=a: counts(*a)) for k, a in COUNTS.items()})
CASES.update({"invalid_" + k: (lambda k=k: lookup(k)) for k in INVALID})
