"""cs_clean_mesh restated in float64 (numpy and Python floats, every operation rounded once, in the header's order):
the input check, degenerate and duplicate faces, the long-edge statistics in coop.cuh's three-level order, the
non-manifold edges, the components and the non-manifold vertices, the boundary loops and their ear cutting, Taubin
smoothing and the output order.  mutation names a deliberate change of one rule, for the tests that must see it."""
import math

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from simplify_oracle import validate
from texture_oracle import tree_total

MAX_HOLE = 256
DEFAULTS = dict(removeDegenerate=True, longEdgeFactor=20.0, removeNonManifold=True, minComponentFaces=50,
                minComponentFraction=0.0, maxHoleEdges=30, smoothIterations=0, smoothLambda=0.5, smoothMu=-0.53)
OFF = dict(removeDegenerate=False, longEdgeFactor=0.0, removeNonManifold=False, minComponentFaces=0,
           minComponentFraction=0.0, maxHoleEdges=0, smoothIterations=0)


# ---- float64 vectors in the header's order ----------------------------------------------------------------------------
def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _normal(p0, p1, p2):
    return _cross(p1 - p0, p2 - p0)


def _sub(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def _dot3(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _normal3(p0, p1, p2):
    a, b = _sub(p1, p0), _sub(p2, p0)
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _edge_keys(t, faces):
    """(key (min << 32) | max, corner) of every corner edge of the given faces, corner 3f + k from k to k + 1."""
    c = (3 * faces[:, None] + np.arange(3)).reshape(-1)
    a = t.reshape(-1)[c]
    b = t.reshape(-1)[3 * (c // 3) + (c % 3 + 1) % 3]
    return (np.minimum(a, b) << 32) | np.maximum(a, b), c


def _runs(keys, corners):
    """corners sorted by (key, corner), and each one's run start and run length."""
    o = np.lexsort((corners, keys))
    k, c = keys[o], corners[o]
    head = np.r_[True, k[1:] != k[:-1]]
    start = np.maximum.accumulate(np.where(head, np.arange(len(k)), 0))
    ends = np.r_[np.flatnonzero(head)[1:], len(k)]
    length = (ends - np.flatnonzero(head))[np.cumsum(head) - 1]
    return k, c, start, length


def ear_cut(P, ring, edges=frozenset(), mutation=None):
    """Rule 6's ear cutting of the loop ring (vertex ids in loop order, lowest first) among the kept faces' edges
    (keys (min << 32) | max): the faces, or None."""
    p0 = P[ring[0]]
    N = (0.0, 0.0, 0.0)
    for i in range(1, len(ring) - 1):
        n = _normal3(p0, P[ring[i]], P[ring[i + 1]])
        N = (N[0] + n[0], N[1] + n[1], N[2] + n[2])
    r = list(ring)
    faces = []
    while len(r) > 3:
        n = len(r)
        best, bc = -1, 0.0
        for i in range(n):
            pa, pb, pc = P[r[i - 1]], P[r[i]], P[r[(i + 1) % n]]
            if not _dot3(_normal3(pa, pb, pc), N) > 0.0:
                continue
            a, c = r[i - 1], r[(i + 1) % n]
            if (min(a, c) << 32) | max(a, c) in edges:
                continue
            if any(_dot3(_normal3(pa, pb, P[q]), N) > 0.0 and _dot3(_normal3(pb, pc, P[q]), N) > 0.0 and
                   _dot3(_normal3(pc, pa, P[q]), N) > 0.0 for q in r if q not in (a, r[i], c)):
                continue
            u, w = _sub(pa, pb), _sub(pc, pb)
            cs = _dot3(u, w) / math.sqrt(_dot3(u, u) * _dot3(w, w))
            if best < 0 or cs > bc or (mutation == "ear_tie_last" and cs == bc):
                best, bc = i, cs
        if best < 0:
            return None
        faces.append((r[best - 1], r[best], r[(best + 1) % n]))
        del r[best]
    if not _dot3(_normal3(P[r[0]], P[r[1]], P[r[2]]), N) > 0.0:
        return None
    faces.append((r[0], r[1], r[2]))
    if mutation == "fill_reversed":
        faces = [(a, c, b) for a, b, c in faces]
    return faces


def boundary_loops(t, alive):
    """Rule 6's boundary half-edges of the alive faces: (loops as lists of half-edges (from, to) in loop order from
    the lowest vertex, the number of half-edges on no loop)."""
    faces = np.flatnonzero(alive)
    keys, corners = _edge_keys(t, faces)
    k, c, start, length = _runs(keys, corners)
    bc = np.sort(c[length == 1])
    flat = t.reshape(-1)
    frm = flat[3 * (bc // 3) + (bc % 3 + 1) % 3]
    to = flat[bc]
    hin, hout = {}, {}
    for a, b in zip(frm.tolist(), to.tolist()):
        hout[a] = hout.get(a, 0) + 1
        hin[b] = hin.get(b, 0) + 1
    out_of = {a: h for h, a in enumerate(frm.tolist()) if hout[a] == 1}
    succ = [out_of[b] if hin.get(b) == 1 and hout.get(b) == 1 else -1 for b in to.tolist()]
    state = [0] * len(bc)       # 0 unseen, 1 on a loop, 2 on no loop
    loops, chain = [], 0
    for h in range(len(bc)):
        if state[h]:
            continue
        walk, g = [h], succ[h]
        while g >= 0 and g != h and not state[g]:
            walk.append(g)
            g = succ[g]
        if g == h:
            for x in walk:
                state[x] = 1
            s = min(range(len(walk)), key=lambda i: frm[walk[i]])
            walk = walk[s:] + walk[:s]
            loops.append([(int(frm[x]), int(to[x])) for x in walk])
        else:
            for x in walk:
                state[x] = 2
            chain += len(walk)
    # the walk from h may start inside a path whose earlier part is unseen: those are marked when reached
    loops.sort(key=lambda lp: lp[0][0])
    return loops, chain


def clean(verts, tris, intensity=None, mutation=None, **kw):
    """The outputs of cs_clean_mesh: dict(vertices, triangles, intensity, info [3], stats [19])."""
    prm = dict(DEFAULTS, **kw)
    X = np.asarray(verts, np.float32).reshape(-1, 3)
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    V, T = len(X), len(t)
    stats = [0] * 19
    stats[0] = T
    empty = dict(vertices=np.zeros((0, 3), np.float32), triangles=np.zeros((0, 3), np.int32),
                 intensity=None if intensity is None else np.zeros(0, np.float32), info=[0.0, 0.0, 0.0])
    if T == 0:
        return dict(empty, stats=stats)
    if not validate(X, t):
        stats[18] = 2
        return dict(empty, stats=stats)
    P = X.astype(np.float64)
    alive = np.ones(T, bool)
    # rule 2
    if prm["removeDegenerate"]:
        n = _normal(P[t[:, 0]], P[t[:, 1]], P[t[:, 2]])
        keys, corners = _edge_keys(t, np.arange(T))
        _, inv, cnt = np.unique(keys, return_inverse=True, return_counts=True)
        enclosed = (cnt[inv].reshape(T, 3) >= 2).all(1) & (mutation != "drop_enclosed")
        deg = (_dot(n, n) == 0.0) & ~enclosed
        alive &= ~deg
        stats[1] = int(deg.sum())
        idx = np.flatnonzero(alive)
        s = np.sort(t[idx], axis=1)
        if mutation == "keep_highest":
            _, first = np.unique(s[::-1], axis=0, return_index=True)
            keep = idx[::-1][first]
        else:
            _, first = np.unique(s, axis=0, return_index=True)
            keep = idx[first]
        dup = alive.copy()
        dup[keep] = False
        alive &= ~dup
        stats[2] = int(dup.sum())
    info = [0.0, 0.0, 0.0]
    # rule 3
    if prm["longEdgeFactor"] > 0:
        keys, corners = _edge_keys(t, np.arange(T))
        o = np.argsort(keys, kind="stable")
        ks = keys[o]
        head = np.r_[True, ks[1:] != ks[:-1]]
        run = np.cumsum(head) - 1
        kept = np.zeros(run[-1] + 1, bool)
        kept[run[alive[corners[o] // 3]]] = True
        head &= kept[run]
        a, b = ks >> 32, ks & 0xffffffff
        d = P[b] - P[a]
        ln = np.sqrt(_dot(d, d))
        e = lambda v: np.where(head, v, 0.0)
        N, S1, S2 = tree_total(e(np.ones(len(ks)))), tree_total(e(ln)), tree_total(e(ln * ln))
        m = s = 0.0
        if N > 0:
            m = S1 / N
            var = S2 / N - m * m
            s = math.sqrt(var) if var > 0 else 0.0
        thr = m + prm["longEdgeFactor"] * s
        info = [m, s, thr]
        long_ = np.zeros(T, bool)
        for j in range(3):
            u, w = t[:, j], t[:, (j + 1) % 3]
            dd = P[np.maximum(u, w)] - P[np.minimum(u, w)]
            long_ |= np.sqrt(_dot(dd, dd)) > thr
        long_ &= alive
        alive &= ~long_
        stats[3] = int(long_.sum())
    # rule 4
    if prm["removeNonManifold"]:
        keys, corners = _edge_keys(t, np.flatnonzero(alive))
        k, c, start, length = _runs(keys, corners)
        rank = np.arange(len(k)) - start
        fin = np.zeros(T, bool)
        fin[c[rank >= 2] // 3] = True
        alive &= ~fin
        stats[4] = int(fin.sum())
    # rule 5 and the non-manifold vertices
    faces = np.flatnonzero(alive)
    keys, corners = _edge_keys(t, faces)
    k, c, start, length = _runs(keys, corners)
    two = np.flatnonzero((length == 2) & (np.arange(len(k)) == start))
    c1, c2 = c[two], c[two + 1]
    A = coo_matrix((np.ones(len(two)), (c1 // 3, c2 // 3)), shape=(T, T))
    _, lab = connected_components(A, directed=False)
    flat = t.reshape(-1)
    nx = lambda cc: 3 * (cc // 3) + (cc % 3 + 1) % 3
    same = flat[c1] == flat[c2]
    ca = np.r_[c1, nx(c1)]
    cb = np.r_[np.where(same, c2, nx(c2)), np.where(same, nx(c2), c2)]
    Cg = coo_matrix((np.ones(len(ca)), (ca, cb)), shape=(3 * T, 3 * T))
    _, clab = connected_components(Cg, directed=False)
    ac = (3 * faces[:, None] + np.arange(3)).reshape(-1)
    fans = np.zeros(V, np.int64)
    pairs = np.unique(np.stack([flat[ac], clab[ac]], 1), axis=0)
    np.add.at(fans, pairs[:, 0], 1)
    stats[8] = int((fans > 1).sum())
    comp, size = np.unique(lab[faces], return_counts=True)
    stats[6] = len(comp)
    largest = int(size.max()) if len(size) else 0
    if prm["minComponentFaces"] > 1 or prm["minComponentFraction"] > 0:
        small = (size < prm["minComponentFaces"]) | (size.astype(np.float64) < prm["minComponentFraction"] * float(largest))
        drop = np.zeros(T, bool)
        drop[faces] = np.isin(lab[faces], comp[small])
        alive &= ~drop
        stats[5] = int(drop.sum())
        stats[7] = int(small.sum())
    # rule 6
    fills = []
    if prm["maxHoleEdges"] > 0:
        loops, chain = boundary_loops(t, alive)
        Pt = [tuple(float(x) for x in row) for row in P]
        keys, _ = _edge_keys(t, np.flatnonzero(alive))
        edges = frozenset(keys.tolist())
        filled = 0
        for lp in loops:
            if 3 <= len(lp) <= prm["maxHoleEdges"]:
                f = ear_cut(Pt, [h[0] for h in lp], edges, mutation)
                if f is not None:
                    fills += f
                    filled += 1
        stats[9], stats[10], stats[11], stats[12], stats[13] = len(loops), filled, len(loops) - filled, chain, len(fills)
    out = np.concatenate([t[alive], np.asarray(fills, np.int64).reshape(-1, 3)])
    # rule 7
    pos = P.copy()
    if prm["smoothIterations"] > 0 and len(out):
        a = out.reshape(-1)
        b = out[:, [1, 2, 0]].reshape(-1)
        dk = np.sort(np.r_[(a << 32) | b, (b << 32) | a])
        u, cnt = np.unique(dk, return_counts=True)
        src, dst = u >> 32, u & 0xffffffff
        fixed = np.zeros(V, bool)
        fixed[src[cnt != 2]] = True
        nb = [[] for _ in range(V)]
        for s_, d_ in zip(src.tolist(), dst.tolist()):
            nb[s_].append(d_)
        has = np.array([len(x) > 0 for x in nb]) & ~fixed
        vs = np.flatnonzero(has)
        kmax = max((len(nb[v]) for v in vs), default=0)
        idx = np.full((len(vs), kmax), -1, np.int64)
        for r_, v in enumerate(vs):
            idx[r_, :len(nb[v])] = nb[v]
        kk = (idx >= 0).sum(1).astype(np.float64)[:, None]
        for _ in range(prm["smoothIterations"]):
            for f in (prm["smoothLambda"], prm["smoothMu"]):
                s = np.zeros((len(vs), 3))
                for j in range(kmax):
                    s = s + np.where(idx[:, j:j + 1] >= 0, pos[np.maximum(idx[:, j], 0)], 0.0)
                x = pos[vs]
                new = pos.copy()
                new[vs] = x + f * (s / kk - x)
                pos = new
    # rule 8
    used = np.zeros(V, bool)
    used[out.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    ov = pos[used].astype(np.float32)
    ot = remap[out].astype(np.int32).reshape(-1, 3)
    stats[14], stats[15], stats[16], stats[17] = len(ov), len(ot), len(ov), len(ot)
    oi = None if intensity is None else np.asarray(intensity, np.float32)[used]
    return dict(vertices=ov, triangles=ot, intensity=oi, info=info, stats=stats)


# ---- topology checks -------------------------------------------------------------------------------------------------
def topology(tris, V=None):
    """(boundary edges, edges held by three or more faces, Euler characteristic V - E + F over used vertices,
    consistently oriented: every edge held by two faces is traversed once in each direction)."""
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    a, b = t.reshape(-1), t[:, [1, 2, 0]].reshape(-1)
    und = (np.minimum(a, b) << 32) | np.maximum(a, b)
    u, cnt = np.unique(und, return_counts=True)
    d = np.unique((a << 32) | b)
    Vu = len(np.unique(t))
    oriented = len(d) == len(a)
    return int((cnt == 1).sum()), int((cnt > 2).sum()), Vu - len(u) + len(t), oriented


def components(tris):
    """Face counts of the components joined across edges held by exactly two faces."""
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    T = len(t)
    keys, corners = _edge_keys(t, np.arange(T))
    k, c, start, length = _runs(keys, corners)
    two = np.flatnonzero((length == 2) & (np.arange(len(k)) == start))
    A = coo_matrix((np.ones(len(two)), (c[two] // 3, c[two + 1] // 3)), shape=(T, T))
    _, lab = connected_components(A, directed=False)
    return np.bincount(lab)
