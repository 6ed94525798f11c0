"""cs_simplify_mesh restated in float64 (Python floats, every operation rounded once, in the header's order): input
checks, frozen vertices, quadrics, edge evaluation, the gated parallel pass, the collapse and the output order; plus a
sequential greedy decimator (Garland & Heckbert 1997, one collapse at a time from a heap) under the same validity rules,
which serves as the quality reference."""
import heapq
import math

import numpy as np

F_SHIFT = 1                     # f = 1 / 2^F_SHIFT: the cheapest ceil(C f) candidates compete in a pass
BOUNDARY_WEIGHT = 1.0           # the default boundaryWeight
DET_EPS = 1e-6                  # the minimiser is used when det(A) > DET_EPS a11 a22 a33
MAX_PASSES = 1000
NO_KEY = (1 << 64) - 1


def validate(verts, tris):
    """False when a triangle index lies outside [0, V), a triangle repeats a vertex or a used vertex is not finite."""
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    if len(t) == 0:
        return True
    if t.min() < 0 or t.max() >= len(verts):
        return False
    if ((t[:, 0] == t[:, 1]) | (t[:, 1] == t[:, 2]) | (t[:, 0] == t[:, 2])).any():
        return False
    return bool(np.isfinite(np.asarray(verts, np.float32)[np.unique(t)]).all())


# ---- float64 arithmetic in the header's order ------------------------------------------------------------------------
def sub(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def normal(p0, p1, p2):
    return cross(sub(p1, p0), sub(p2, p0))


def plane_add(q, n, d, w):
    """q += w p p^T for the plane p = (n, d), upper triangle row-major, each entry w (p_i p_j)."""
    p = (n[0], n[1], n[2], d)
    k = 0
    for i in range(4):
        for j in range(i, 4):
            q[k] = q[k] + w * (p[i] * p[j])
            k += 1


def face_plane(p0, p1, p2):
    """(unit normal, offset, area) of a face, or None when its area is 0."""
    n = normal(p0, p1, p2)
    ln = math.sqrt(dot(n, n))
    if not ln > 0:
        return None
    u = (n[0] / ln, n[1] / ln, n[2] / ln)
    return u, -dot(u, p0), 0.5 * ln


def edge_plane(u, pa, pb, bw):
    """The plane through a boundary edge a -> b perpendicular to its face (unit normal u), with its weight."""
    e = sub(pb, pa)
    m = cross(e, u)
    lm = math.sqrt(dot(m, m))
    if not lm > 0:
        return None
    mu = (m[0] / lm, m[1] / lm, m[2] / lm)
    return mu, -dot(mu, pa), bw * dot(e, e)


def cost(q, x):
    a11, a12, a13, b1, a22, a23, b2, a33, b3, c = q
    x0, x1, x2 = x
    r = (a11 * x0 * x0 + a22 * x1 * x1) + a33 * x2 * x2
    r = r + 2.0 * ((a12 * x0 * x1 + a13 * x0 * x2) + a23 * x1 * x2)
    r = r + 2.0 * ((b1 * x0 + b2 * x1) + b3 * x2)
    return r + c


def optimum(q, pu, pv):
    """(position, cost >= 0): the minimiser of q when det(A) > DET_EPS a11 a22 a33, else the best of u, v and the
    midpoint (ties to u, then v)."""
    a11, a12, a13, b1, a22, a23, b2, a33, b3, c = q
    c11 = a22 * a33 - a23 * a23
    c12 = a12 * a33 - a23 * a13
    c13 = a12 * a23 - a22 * a13
    det = (a11 * c11 - a12 * c12) + a13 * c13
    if det > DET_EPS * (a11 * a22 * a33):
        x = (-(((b1 * c11 - a12 * (b2 * a33 - a23 * b3)) + a13 * (b2 * a23 - a22 * b3)) / det),
             -(((a11 * (b2 * a33 - a23 * b3) - b1 * c12) + a13 * (a12 * b3 - b2 * a13)) / det),
             -(((a11 * (a22 * b3 - b2 * a23) - a12 * (a12 * b3 - b2 * a13)) + b1 * c13) / det))
        best = cost(q, x)
    else:
        x, best = pu, cost(q, pu)
        cv = cost(q, pv)
        if cv < best:
            x, best = pv, cv
        mid = ((pu[0] + pv[0]) * 0.5, (pu[1] + pv[1]) * 0.5, (pu[2] + pv[2]) * 0.5)
        cm = cost(q, mid)
        if cm < best:
            x, best = mid, cm
    return x, (best if best > 0 else 0.0)


def error_of(cst, area):
    if area > 0:
        return cst / area
    return 0.0 if cst == 0 else math.inf


def f32(x):
    return float(np.float32(x))


def tie_of(eid):
    """s(id): the bijection of the 32-bit ids that orders equal errors (m = id 0x9E3779B1 mod 2^32, m ^ (m >> 16))."""
    m = (eid * 0x9E3779B1) & 0xFFFFFFFF
    return m ^ (m >> 16)


def key_of(err, eid):
    with np.errstate(over="ignore"):        # an error above FLT_MAX rounds to an infinite key, as on the GPU
        f = np.float32(err)
    return (int(f.view(np.uint32)) << 32) | tie_of(eid)


# ---- the mesh state ---------------------------------------------------------------------------------------------------
def adjacency(tris, nv):
    """vf[x]: the faces holding x, ascending (the stable sort of corner keys)."""
    vf = [[] for _ in range(nv)]
    for t, f in enumerate(tris):
        if f is not None:
            for x in f:
                vf[x].append(t)
    return vf


def has_directed(tris, faces, a, b):
    """Some face among faces traverses a -> b."""
    for t in faces:
        f = tris[t]
        for j in range(3):
            if f[j] == a and f[(j + 1) % 3] == b:
                return True
    return False


def frozen_vertex(tris, faces, x):
    """x's faces are not one fan (one cycle or one open chain), or an edge at x has more than two faces or two faces
    that traverse it in the same direction."""
    nxt, prv = [], []
    for t in faces:
        f = tris[t]
        j = f.index(x)
        nxt.append(f[(j + 1) % 3])
        prv.append(f[(j + 2) % 3])
    k = len(faces)
    for i in range(k):
        if nxt.count(nxt[i]) > 1 or prv.count(prv[i]) > 1:
            return True
    # the link: face i is the link edge nxt[i] -> prv[i]; a chain starts at a face whose nxt no face ends at
    starts = [i for i in range(k) if nxt[i] not in prv]
    if len(starts) > 1:
        return True
    first = starts[0] if starts else 0
    i, count = first, 1
    while True:
        j = next((m for m in range(k) if nxt[m] == prv[i]), None)
        if j is None or j == first:
            break
        i, count = j, count + 1
    return count < k


def boundary_edge(tris, faces_x, x, y):
    """The edge x-y (x not frozen) has one face: no face of x traverses it both ways."""
    return not (has_directed(tris, faces_x, x, y) and has_directed(tris, faces_x, y, x))


def on_boundary(tris, faces, x):
    for t in faces:
        f = tris[t]
        j = f.index(x)
        if not has_directed(tris, faces, f[(j + 1) % 3], x):
            return True
    return False


def vertex_quadric(tris, vf, pos, x, bw):
    """Faces in ascending index, then the boundary edges of those faces in (face, corner) order."""
    q = [0.0] * 10
    area = 0.0
    for t in vf[x]:
        f = tris[t]
        fp = face_plane(pos[f[0]], pos[f[1]], pos[f[2]])
        if fp is not None:
            plane_add(q, fp[0], fp[1], fp[2])
            area = area + fp[2]
    for t in vf[x]:
        f = tris[t]
        fp = face_plane(pos[f[0]], pos[f[1]], pos[f[2]])
        for k in range(3):
            a, b = f[k], f[(k + 1) % 3]
            if fp is None or x not in (a, b) or has_directed(tris, vf[x], b, a):
                continue
            ep = edge_plane(fp[0], pos[a], pos[b], bw)
            if ep is not None:
                plane_add(q, ep[0], ep[1], ep[2])
    return q, area


def neighbours(tris, faces):
    s = set()
    for t in faces:
        s.update(tris[t])
    return s


def evaluate(st, vf, t, k, canonical=True):
    """The edge at corner k of face t: None when it is not the canonical corner or the collapse is not valid, else
    (err, x, u, v, drops)."""
    tris, pos, frozen = st["tris"], st["pos"], st["frozen"]
    f = tris[t]
    a, b = f[k], f[(k + 1) % 3]
    if frozen[a] or frozen[b]:
        return None
    interior = has_directed(tris, vf[b], b, a)
    if canonical and interior and not a < b:
        return None
    u, v = (a, b) if a < b else (b, a)
    apex = [f[(k + 2) % 3]]
    if interior:
        for s in vf[b]:
            g = tris[s]
            for j in range(3):
                if g[j] == b and g[(j + 1) % 3] == a:
                    apex.append(g[(j + 2) % 3])
    # link condition
    nv = neighbours(tris, vf[v])
    for w in neighbours(tris, vf[u]):
        if w != u and w != v and w in nv and w not in apex:
            return None
    if interior:
        if on_boundary(tris, vf[u], u) and on_boundary(tris, vf[v], v):
            return None
        w1, w2 = apex
        if any(w1 in tris[s] and w2 in tris[s] for s in vf[u]) and any(w1 in tris[s] and w2 in tris[s] for s in vf[v]):
            return None
    else:
        w = apex[0]
        if boundary_edge(tris, vf[u], u, w) and boundary_edge(tris, vf[v], v, w):
            return None
    qu, qv = st["Q"][u], st["Q"][v]
    q = [qu[i] + qv[i] for i in range(10)]
    area = st["A"][u] + st["A"][v]
    x, cst = optimum(q, pos[u], pos[v])
    err = error_of(cst, area)
    if not (err < math.inf and math.sqrt(err) <= st["maxError"]):
        return None
    # flips
    for s in vf[u] + vf[v]:
        g = tris[s]
        if u in g and v in g:
            continue
        p = [pos[w] for w in g]
        n0 = normal(p[0], p[1], p[2])
        if not dot(n0, n0) > 0:
            continue
        p = [x if w in (u, v) else pos[w] for w in g]
        if not dot(n0, normal(p[0], p[1], p[2])) > 0:
            return None
    return err, x, u, v, 2 if interior else 1


def collapse(st, u, v, x):
    pos, inten = st["pos"], st["inten"]
    if inten is not None:
        d = sub(pos[v], pos[u])
        den = dot(d, d)
        t = dot(sub(x, pos[u]), d) / den if den > 0 else 0.0
        t = 0.0 if not t > 0 else (1.0 if t > 1 else t)
        inten[u] = f32(inten[u] + t * (inten[v] - inten[u]))
    pos[u] = x
    st["Q"][u] = [st["Q"][u][i] + st["Q"][v][i] for i in range(10)]
    st["A"][u] = st["A"][u] + st["A"][v]


def setup(verts, tris, inten, maxError, bw):
    V = len(verts)
    tl = [tuple(int(i) for i in f) for f in np.asarray(tris, np.int64).reshape(-1, 3)]
    pos = [tuple(float(c) for c in p) for p in np.asarray(verts, np.float32)]
    vf = adjacency(tl, V)
    frozen = [frozen_vertex(tl, vf[x], x) if vf[x] else False for x in range(V)]
    Q, A = [], []
    for x in range(V):
        q, a = vertex_quadric(tl, vf, pos, x, bw) if vf[x] and not frozen[x] else ([0.0] * 10, 0.0)
        Q.append(q)
        A.append(a)
    return dict(tris=tl, tid=list(range(len(tl))), pos=pos, frozen=frozen, Q=Q, A=A, maxError=maxError,
                inten=None if inten is None else [float(c) for c in np.asarray(inten, np.float32)])


def output(st, status, passes, collapses, maxerr, T0):
    tris = st["tris"]
    used = sorted(set(w for f in tris for w in f))
    ren = {w: i for i, w in enumerate(used)}
    verts = np.array([st["pos"][w] for w in used], np.float64).reshape(-1, 3).astype(np.float32)
    tr = np.array([[ren[w] for w in f] for f in tris], np.int64).reshape(-1, 3)
    inten = None if st["inten"] is None else np.array([st["inten"][w] for w in used], np.float32)
    stats = [T0, sum(st["frozen"]), passes, collapses, len(used), len(tris), len(used), len(tris), status]
    return dict(vertices=verts, triangles=tr, intensity=inten, info=math.sqrt(maxerr), stats=stats,
                tid=np.array(st["tid"], np.int64), frozen=np.array(st["frozen"]))


def simplify(verts, tris, inten=None, target=0, maxError=math.inf, boundaryWeight=BOUNDARY_WEIGHT, f_shift=F_SHIFT,
             max_passes=MAX_PASSES):
    """The whole call.  Returns a dict: vertices, triangles, intensity, info (largest applied sqrt(cost / A)), stats
    (the header's 9 entries), tid (input index of every surviving triangle), frozen."""
    V, T0 = len(verts), len(tris)
    if not validate(verts, tris):
        return dict(vertices=np.zeros((0, 3), np.float32), triangles=np.zeros((0, 3), np.int64), intensity=None,
                    info=0.0, stats=[T0, 0, 0, 0, 0, 0, 0, 0, 2])
    st = setup(verts, tris, inten, maxError, boundaryWeight)
    passes = collapses = 0
    maxerr = 0.0
    ver = [0] * V            # bumped on the closed ring of every applied collapse: an edge's evaluation depends on
    cache = {}               # its ends' faces, the positions of their vertices and its ends' quadrics only
    while True:
        tris, T = st["tris"], len(st["tris"])
        if T <= target:
            status = 0
            break
        if passes == max_passes:
            status = 3
            break
        vf = adjacency(tris, V)
        cands = []
        for t in range(T):
            for k in range(3):
                f = tris[t]
                a, b = f[k], f[(k + 1) % 3]
                ck = (st["tid"][t], k)
                hit = cache.get(ck)
                if hit is None or hit[0] != ver[a] or hit[1] != ver[b]:
                    hit = (ver[a], ver[b], evaluate(st, vf, t, k))
                    cache[ck] = hit
                r = hit[2]
                if r is not None:
                    cands.append((key_of(r[0], 3 * st["tid"][t] + k),) + r)
        if not cands:
            status = 1
            break
        C = len(cands)
        m = (C + (1 << f_shift) - 1) >> f_shift
        thr = sorted(c[0] for c in cands)[m - 1]
        compete = [c for c in cands if c[0] <= thr]
        mark = {}
        rings = []
        for c in compete:
            ring = neighbours(tris, vf[c[3]]) | neighbours(tris, vf[c[4]])
            rings.append(ring)
            for w in ring:
                mark[w] = min(mark.get(w, NO_KEY), c[0])
        sel = [c for c, ring in zip(compete, rings) if all(mark[w] == c[0] for w in ring)]
        drops = sum(c[5] for c in sel)
        if T - drops < target:
            sel.sort()
            need, cum, cut = T - target, 0, 0
            while cum < need:
                cum += sel[cut][5]
                cut += 1
            sel = sel[:cut]
        remap = list(range(V))
        for key, err, x, u, v, _ in sel:
            for w in neighbours(tris, vf[u]) | neighbours(tris, vf[v]):
                ver[w] += 1
            collapse(st, u, v, x)
            remap[v] = u
            maxerr = max(maxerr, err)
        nt, nid = [], []
        for f, i in zip(tris, st["tid"]):
            g = tuple(remap[w] for w in f)
            if g[0] != g[1] and g[1] != g[2] and g[0] != g[2]:
                nt.append(g)
                nid.append(i)
        st["tris"], st["tid"] = nt, nid
        passes += 1
        collapses += len(sel)
    return output(st, status, passes, collapses, maxerr, T0)


def greedy(verts, tris, target=0, maxError=math.inf, boundaryWeight=BOUNDARY_WEIGHT):
    """Sequential Garland-Heckbert decimation under the same rules: always the cheapest valid collapse (a heap with
    re-evaluation on pop).  Returns (vertices, triangles) in the same output order as simplify."""
    V = len(verts)
    st = setup(verts, tris, None, maxError, boundaryWeight)
    tris = list(st["tris"])
    st["tris"] = tris
    vf = adjacency(tris, V)
    T = len(tris)

    def edges_at(x):
        out = []
        for t in vf[x]:
            f = tris[t]
            j = f.index(x)
            out.append((t, j))
            out.append((t, (j + 2) % 3))
        return out

    def push(t, k):
        r = evaluate(st, vf, t, k, canonical=False)
        if r is not None:
            f = tris[t]
            heapq.heappush(heap, (r[0], min(f[k], f[(k + 1) % 3]), max(f[k], f[(k + 1) % 3])))

    heap = []
    for t in range(T):
        for k in range(3):
            push(t, k)
    while T > target and heap:
        err, u, v = heapq.heappop(heap)
        at = [(t, k) for (t, k) in edges_at(u) if v in (tris[t][k], tris[t][(k + 1) % 3])]
        if not at:
            continue
        r = evaluate(st, vf, at[0][0], at[0][1], canonical=False)
        if r is None:
            continue
        if r[0] != err:
            heapq.heappush(heap, (r[0], u, v))
            continue
        collapse(st, u, v, r[1])
        for t in vf[v]:
            f = tris[t]
            if u in f:
                tris[t] = None
                T -= 1
                for w in f:
                    if w != v:
                        vf[w].remove(t)
            else:
                tris[t] = tuple(u if w == v else w for w in f)
                vf[u].append(t)
        vf[u].sort()
        vf[v] = []
        for w in neighbours(tris, vf[u]):
            for t, k in edges_at(w):
                push(t, k)
    alive = [f for f in tris if f is not None]
    used = sorted(set(w for f in alive for w in f))
    ren = {w: i for i, w in enumerate(used)}
    return (np.array([st["pos"][w] for w in used], np.float64).reshape(-1, 3),
            np.array([[ren[w] for w in f] for f in alive], np.int64).reshape(-1, 3))


# ---- checks --------------------------------------------------------------------------------------------------------
def manifold_apart_from(tris, frozen_ids):
    """Every edge without a frozen end has one or two faces, traversed in opposite directions; every vertex that is not
    frozen has one fan."""
    tl = [tuple(int(i) for i in f) for f in np.asarray(tris, np.int64).reshape(-1, 3)]
    nv = 1 + max((max(f) for f in tl), default=-1)
    vf = adjacency(tl, nv)
    fz = set(int(i) for i in frozen_ids)
    return all(not frozen_vertex(tl, vf[x], x) for x in range(nv) if vf[x] and x not in fz)


def boundary_loops(tris):
    """The number of boundary loops (directed boundary edges chained head to tail)."""
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    e = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    s = set(map(tuple, e))
    nxt = {}
    for a, b in e:
        if (b, a) not in s:
            nxt.setdefault(int(a), []).append(int(b))
    seen, loops = set(), 0
    for a in list(nxt):
        for b in nxt[a]:
            if (a, b) in seen:
                continue
            loops += 1
            x, y = a, b
            while (x, y) not in seen:
                seen.add((x, y))
                x, y = y, nxt.get(y, [None])[0]
                if y is None:
                    break
    return loops
