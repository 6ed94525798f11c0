"""cs_level_texture_seams restated in float64 (numpy scalars and element-wise operations, each rounded once, in the
header's order): the input check, the unknowns, the seam and smoothness rows, the system and its exact solution
(scipy.sparse direct solve), a float64 Jacobi-PCG with the same preconditioner, the seam energies in coop.cuh's
three-level order, and the texel stage."""
import math

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

import texture_oracle as to


def holds(e, x, y):
    """Whether chart e's rectangle [ox, ox + width) x [oy, oy + height) holds the texel (x, y)."""
    return e[5] <= x < e[5] + e[3] and e[6] <= y < e[6] + e[4]


def chart_of(uv, label, charts, rows, width):
    """Rule 1: the chart whose rectangle holds floor of corner 0's uv and whose image is the label, or -1."""
    x, y = math.floor(float(uv[0, 0])), math.floor(float(uv[0, 1]))
    if not (0 <= x < width and 0 <= y < rows):
        return -1
    for c, e in enumerate(charts):
        if holds(e, x, y) and e[0] == label:
            return c
    return -1


def tap_box(atlas, e):
    """The box the bilinear taps are clamped to: chart e's rectangle (xl, xh, yl, yh), inclusive."""
    return e[5], e[5] + e[3] - 1, e[6], e[6] + e[4] - 1


def bilinear(atlas, e, x, y):
    x0, y0 = math.floor(x), math.floor(y)
    fx, fy = x - x0, y - y0
    xl, xh, yl, yh = tap_box(atlas, e)
    xa, xb = int(min(max(x0, xl), xh)), int(min(max(x0 + 1.0, xl), xh))
    ya, yb = int(min(max(y0, yl), yh)), int(min(max(y0 + 1.0, yl), yh))
    A = lambda r, c: float(atlas[r, c])
    r0 = (1.0 - fx) * A(ya, xa) + fx * A(ya, xb)
    r1 = (1.0 - fx) * A(yb, xa) + fx * A(yb, xb)
    return (1.0 - fy) * r0 + fy * r1


def build(verts, tris, labels, uv, charts, atlas, smoothness=0.1):
    """Rules 1-4.  Returns None for invalid input, else a dict: faceChart, unknown keys (v, l) and corner unknowns,
    seam edges, seam rows (i, j, F_a, F_b) and smoothness rows (i, j)."""
    X = np.asarray(verts, np.float32)
    tr = np.asarray(tris, np.int64).reshape(-1, 3)
    lab = np.asarray(labels, np.int64).reshape(-1)
    U = np.asarray(uv, np.float32).reshape(-1, 3, 2)
    rows, width = atlas.shape
    T = len(tr)
    if not to.validate(X, tr):
        return None
    fc = np.full(T, -1, np.int64)
    for f in range(T):
        if lab[f] < 0:
            continue
        if not np.isfinite(U[f]).all():
            return None
        fc[f] = chart_of(U[f], lab[f], charts, rows, width)
        if fc[f] < 0:
            return None
    seen = lab >= 0
    keys = sorted({(int(tr[f, k]), int(lab[f])) for f in np.nonzero(seen)[0] for k in range(3)})
    unk = {k: i for i, k in enumerate(keys)}
    cu = np.full((T, 3), -1, np.int64)
    for f in np.nonzero(seen)[0]:
        for k in range(3):
            cu[f, k] = unk[(int(tr[f, k]), int(lab[f]))]
    sm = smooth_rows(cu, seen)
    # seam edges in sorted key order
    nbr = to.adjacency(tr)
    edges = {}
    for f in range(T):
        for k in range(3):
            g = nbr[f, k]
            if g < 0:
                continue
            a, b = int(tr[f, k]), int(tr[f, (k + 1) % 3])
            key = (min(a, b) << 32) | max(a, b)
            if key not in edges and seen[f] and seen[g] and lab[f] != lab[g]:
                edges[key] = (f, int(g))
    ends = {}                                # (g(v, a), g(v, b)) -> list of (edge rank, partials)
    for rank, key in enumerate(sorted(edges)):
        f, g = sides(*edges[key], lab)
        P, Q = key >> 32, key & 0xFFFFFFFF
        side = []
        for h in (f, g):
            kP, kQ = list(tr[h]).index(P), list(tr[h]).index(Q)
            uP, vP = float(U[h, kP, 0]), float(U[h, kP, 1])
            uQ, vQ = float(U[h, kQ, 0]), float(U[h, kQ, 1])
            du, dv = uQ - uP, vQ - vP
            side.append((uP, vP, uQ, vQ, math.sqrt(du * du + dv * dv), charts[fc[h]], (h, kP, kQ)))
        S = sample_count(side[0][4], side[1][4])
        sums = [[0.0, 0.0, 0.0], [0.0, 0.0, 0.0]]
        for k in range(S):
            t = sample_t(k, S)
            I = [bilinear(atlas, s[5], s[0] + t * (s[2] - s[0]), s[1] + t * (s[3] - s[1])) for s in side]
            for end, w in enumerate((1.0 - t, t)):
                sums[end][0] = sums[end][0] + w * I[0]
                sums[end][1] = sums[end][1] + w * I[1]
                sums[end][2] = sums[end][2] + w
        for end in range(2):
            ga = cu[side[0][6][0], side[0][6][1 + end]]
            gb = cu[side[1][6][0], side[1][6][1 + end]]
            ends.setdefault((int(ga), int(gb)), []).append(sums[end])
    seam = []
    for (ga, gb) in sorted(ends):
        s = [0.0, 0.0, 0.0]
        for part in end_order(ends[(ga, gb)]):
            s = [s[c] + part[c] for c in range(3)]
        seam.append((ga, gb) + ratio(s))
    return dict(faceChart=fc, keys=keys, cu=cu, seam=seam, smooth=sm, edges=len(edges), seen=int(seen.sum()),
                smoothness=smoothness)


def ratio(s):
    """(F_a, F_b) = (sum w I_a / sum w, sum w I_b / sum w) in IEEE float64 (0 / 0 is NaN, as on the device)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return float(np.float64(s[0]) / s[2]), float(np.float64(s[1]) / s[2])


def smooth_rows(cu, seen):
    """Rule 4: the distinct unknown pairs (min, max) over the edges of seen faces, sorted."""
    return sorted({(min(cu[f, k], cu[f, (k + 1) % 3]), max(cu[f, k], cu[f, (k + 1) % 3]))
                   for f in np.nonzero(seen)[0] for k in range(3)})


def sides(f, g, lab):
    """Rule 3: the two faces of a seam edge, side 0 the lower label."""
    return (g, f) if lab[f] > lab[g] else (f, g)


def sample_count(La, Lb):
    """Rule 3: S = max(1, ceil(max(L_a, L_b)))."""
    return int(max(1.0, math.ceil(max(La, Lb))))


def sample_t(k, S):
    return (k + 0.5) / S


def end_order(parts):
    """Rule 3: the ends of one (v, a, b) in the order they are added (sorted edge key)."""
    return parts


def system(b, reg):
    """Rule 5: the sparse matrix A = L_w + reg I and the right-hand side."""
    N = len(b["keys"])
    rows = [(i, j, 1.0, Fb - Fa) for i, j, Fa, Fb in b["seam"]] + [(i, j, b["smoothness"], 0.0) for i, j in b["smooth"]]
    I, J, Vv = [], [], []
    rhs = np.zeros(N)
    diag = np.full(N, 0.0)
    for i, j, w, d in rows:
        diag[i] += w
        diag[j] += w
        I += [i, j]
        J += [j, i]
        Vv += [-w, -w]
        rhs[i] += w * d
        rhs[j] -= w * d
    A = sp.csr_matrix((Vv, (I, J)), shape=(N, N)) + sp.diags(diag + reg)
    return A.tocsc(), rhs


def solve_exact(b, reg):
    A, rhs = system(b, reg)
    if A.shape[0] == 0:
        return np.zeros(0)
    return spl.spsolve(A, rhs)


def pcg(b, reg, tol, maxIterations):
    """Jacobi-PCG from 0 in float64 with the stop rule of rule 6 (order of sums not the device's).  Returns (x,
    iterations, converged)."""
    A, rhs = system(b, reg)
    d = A.diagonal()
    x = np.zeros(len(rhs))
    r = rhs.copy()
    z = r / d
    p = np.zeros_like(r)
    rr, rz, bb, beta, it = r @ r, r @ z, r @ r, 0.0, 0
    while it < maxIterations and not (rr <= tol * tol * bb):
        p = z + beta * p
        q = A @ p
        pq = p @ q
        if not pq > 0:
            break
        alpha = rz / pq
        x = x + alpha * p
        r = r - alpha * q
        z = r / d
        it += 1
        rr, rzn = r @ r, r @ z
        beta, rz = rzn / rz, rzn
    return x, it, bool(rr <= tol * tol * bb)


def energy(b, g=None):
    """The seam energy in coop.cuh's three-level order over the seam rows."""
    e = []
    for i, j, Fa, Fb in b["seam"]:
        gi, gj = (0.0, 0.0) if g is None else (float(g[i]), float(g[j]))
        t = (Fa + gi) - (Fb + gj)
        e.append(t * t)
    return to.tree_total(np.array(e, np.float64))


def closest(uvf, ids, X, Y):
    """Rule 7: (squared distance, barycentric weights) of (X, Y) to one face's uv triangle."""
    u = [float(uvf[k, 0]) for k in range(3)]
    v = [float(uvf[k, 1]) for k in range(3)]
    A = (u[1] - u[0]) * (v[2] - v[0]) - (v[1] - v[0]) * (u[2] - u[0])
    if A != 0.0:
        s = 1.0 if A > 0 else -1.0
        w = []
        for k in range(3):
            a, b = k, (k + 1) % 3
            lo = ids[a] < ids[b]
            P, Q = (a, b) if lo else (b, a)
            w.append((s if lo else -s) * ((u[Q] - u[P]) * (Y - v[P]) - (v[Q] - v[P]) * (X - u[P])))
            if w[-1] < 0.0:
                break
        if len(w) == 3 and min(w) >= 0.0:
            S = (w[0] + w[1]) + w[2]
            if S > 0.0:
                return 0.0, (w[1] / S, w[2] / S, w[0] / S)
    best, bw = math.inf, None
    for k in range(3):
        k1 = (k + 1) % 3
        dx, dy = u[k1] - u[k], v[k1] - v[k]
        l2 = dx * dx + dy * dy
        t = min(max(((X - u[k]) * dx + (Y - v[k]) * dy) / l2, 0.0), 1.0) if l2 > 0.0 else 0.0
        ex, ey = X - (u[k] + t * dx), Y - (v[k] + t * dy)
        d2 = ex * ex + ey * ey
        if nearer(d2, best):
            best = d2
            bw = [0.0, 0.0, 0.0]
            bw[k], bw[k1] = 1.0 - t, t
    return best, tuple(bw)


def nearer(d2, best):
    """Rule 7: segment k replaces the best so far only when strictly nearer (ties to the lower k)."""
    return d2 < best


def box_grow(padding):
    """Rule 7: a face's uv box grows by padding + 1 texels."""
    return float(padding + 1)


def texel_key(d2, f):
    """Rule 7: (float(distance) bits << 32) | face; the lower key wins."""
    return (np.uint64(np.float32(math.sqrt(d2)).view(np.uint32)) << np.uint64(32)) | np.uint64(f)


def key_wins(k, old):
    """Rule 7: the 64-bit atomicMin: the nearer face, ties to the lower face."""
    return k < old


def corner_sum(bw, o):
    """Rule 7: (b_0 o_0 + b_1 o_1) + b_2 o_2 in float64."""
    return (bw[0] * float(o[0]) + bw[1] * float(o[1])) + bw[2] * float(o[2])


def texels(tris, labels, uv, charts, faceChart, atlas, corner, padding, copy_all=False):
    """Rule 7 given the float corner offsets [T, 3]: (levelled atlas, texels visited)."""
    tr = np.asarray(tris, np.int64).reshape(-1, 3)
    U = np.asarray(uv, np.float32).reshape(-1, 3, 2)
    rows, width = atlas.shape
    key = np.full(rows * width, to.EMPTY, np.uint64)
    g = box_grow(padding)
    for f in np.nonzero(np.asarray(labels) >= 0)[0]:
        e = charts[faceChart[f]]
        xs, ys = U[f, :, 0].astype(np.float64), U[f, :, 1].astype(np.float64)
        xlo = max(float(e[5]), math.floor(min(min(xs[0], xs[1]), xs[2])) - g)
        xhi = min(float(e[5] + e[3] - 1), math.ceil(max(max(xs[0], xs[1]), xs[2])) + g)
        ylo = max(float(e[6]), math.floor(min(min(ys[0], ys[1]), ys[2])) - g)
        yhi = min(float(e[6] + e[4] - 1), math.ceil(max(max(ys[0], ys[1]), ys[2])) + g)
        for y in range(int(ylo), int(yhi) + 1):
            for x in range(int(xlo), int(xhi) + 1):
                d2, _ = closest(U[f], tr[f], float(x), float(y))
                k = texel_key(d2, f)
                i = y * width + x
                if key_wins(k, key[i]):
                    key[i] = k
    out = atlas.copy()
    hit = np.nonzero(key != to.EMPTY)[0]
    if not copy_all:
        for i in hit:
            f = int(key[i] & np.uint64(0xFFFFFFFF))
            y, x = divmod(int(i), width)
            _, bw = closest(U[f], tr[f], float(x), float(y))
            o = corner[f]
            off = corner_sum(bw, o)
            out.flat[i] = np.float32(atlas.flat[i]) + np.float32(off)
    return out, len(hit)


def level(verts, tris, labels, uv, charts, atlas, padding=2, smoothness=0.1, regularization=1e-3, tol=1e-4,
          maxIterations=1000):
    """The whole call with the exact solve: dict with stats (the integers the device reports, CG iterations from the
    oracle PCG), info [3] (energies from the exact solution, residual 0), offsets g, corner offsets and the atlas."""
    atlas = np.asarray(atlas, np.float32)
    T = len(np.asarray(tris).reshape(-1, 3))
    if T == 0:
        return dict(stats=[0] * 7 + [1], info=[0.0, 0.0, 0.0], atlas=atlas.copy())
    b = build(verts, tris, labels, uv, charts, atlas, smoothness)
    if b is None:
        return dict(stats=[0] * 7 + [2], info=[0.0, 0.0, 0.0])
    g = solve_exact(b, regularization)
    _, its, converged = pcg(b, regularization, tol, maxIterations)
    status = 1 if not b["seam"] else 0 if converged else 3
    lab = np.asarray(labels).reshape(-1)
    corner = np.where(b["cu"] >= 0, g[np.maximum(b["cu"], 0)] if len(g) else 0.0, np.nan).astype(np.float32)
    out, visited = texels(tris, lab, uv, charts, b["faceChart"], atlas, corner, padding, copy_all=not b["seam"])
    stats = [b["seen"], len(b["keys"]), b["edges"], len(b["seam"]), len(b["smooth"]), its, visited, status]
    return dict(stats=stats, info=[energy(b), energy(b, g), 0.0], g=g, corner=corner, atlas=out, build=b)


# ---- the same rules vectorised over numpy arrays, for meshes of 10^5 and more faces --------------------------------
# build_np and texels_np give the bytes build and texels give (a CPU test compares them on every small case); the
# scalar functions above stay the statement of the rules.
def _adjacency_np(tr):
    """to.adjacency without the Python loop: the face across each edge held by exactly two faces."""
    T = len(tr)
    a, b = tr, np.roll(tr, -1, axis=1)
    key = ((np.minimum(a, b) << 32) | np.maximum(a, b)).reshape(-1)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    n = len(ks)
    nbr = np.full(3 * T, -1, np.int64)
    if n < 2:
        return nbr.reshape(T, 3)
    i = np.arange(n - 1)
    start = (ks[1:] == ks[:-1]) & np.r_[True, ks[1:-1] != ks[:-2]] & np.r_[ks[2:] != ks[:-2], True]
    i = i[start]
    c1, c2 = order[i], order[i + 1]
    nbr[c1], nbr[c2] = c2 // 3, c1 // 3
    return nbr.reshape(T, 3)


def _bilinear_np(atlas, e, x, y):
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = x - x0, y - y0
    xl, xh, yl, yh = (e[:, 5].astype(np.float64), (e[:, 5] + e[:, 3] - 1).astype(np.float64),
                      e[:, 6].astype(np.float64), (e[:, 6] + e[:, 4] - 1).astype(np.float64))
    clamp = lambda a, l, h: np.minimum(np.maximum(a, l), h).astype(np.int64)
    xa, xb = clamp(x0, xl, xh), clamp(x0 + 1.0, xl, xh)
    ya, yb = clamp(y0, yl, yh), clamp(y0 + 1.0, yl, yh)
    A = atlas.astype(np.float64)
    r0 = (1.0 - fx) * A[ya, xa] + fx * A[ya, xb]
    r1 = (1.0 - fx) * A[yb, xa] + fx * A[yb, xb]
    return (1.0 - fy) * r0 + fy * r1


def build_np(verts, tris, labels, uv, charts, atlas, smoothness=0.1):
    """build, vectorised; the same dict (keys, smooth and seam as lists of tuples)."""
    X = np.asarray(verts, np.float32)
    tr = np.asarray(tris, np.int64).reshape(-1, 3)
    lab = np.asarray(labels, np.int64).reshape(-1)
    U = np.asarray(uv, np.float32).reshape(-1, 3, 2)
    ch = np.asarray(charts, np.int64).reshape(-1, 8)
    rows, width = atlas.shape
    T = len(tr)
    if not to.validate(X, tr):
        return None
    seen = lab >= 0
    if not np.isfinite(U[seen]).all():
        return None
    fc = np.full(T, -1, np.int64)
    x, y = np.floor(U[:, 0, 0].astype(np.float64)), np.floor(U[:, 0, 1].astype(np.float64))
    inside = seen & (x >= 0) & (x < width) & (y >= 0) & (y < rows)
    for c, e in enumerate(ch):                       # the first chart in table order
        hit = inside & (fc < 0) & (e[5] <= x) & (x < e[5] + e[3]) & (e[6] <= y) & (y < e[6] + e[4]) & (lab == e[0])
        fc[hit] = c
    if (fc[seen] < 0).any():
        return None
    f3 = np.nonzero(seen)[0]
    uk = ((tr[f3] << 32) | lab[f3, None]).reshape(-1)
    ukeys = np.unique(uk)
    keys = [(int(k >> 32), int(k & 0xFFFFFFFF)) for k in ukeys]
    cu = np.full((T, 3), -1, np.int64)
    cu[f3] = np.searchsorted(ukeys, uk).reshape(-1, 3)
    a, b = cu[f3], np.roll(cu[f3], -1, axis=1)
    sk = np.unique(((np.minimum(a, b) << 32) | np.maximum(a, b)).reshape(-1))
    sm = [(int(k >> 32), int(k & 0xFFFFFFFF)) for k in sk]
    # seam edges: the first (f, k) of each edge key, when both faces are seen with different labels
    nbr = _adjacency_np(tr)
    ff, kk = np.nonzero(nbr >= 0)
    g = nbr[ff, kk]
    ok = seen[ff] & seen[g] & (lab[ff] != lab[g])
    ff, kk, g = ff[ok], kk[ok], g[ok]
    pa, pb = tr[ff, kk], tr[ff, (kk + 1) % 3]
    ekey = (np.minimum(pa, pb) << 32) | np.maximum(pa, pb)
    ekeys, first = np.unique(ekey, return_index=True)          # sorted; the first occurrence in (f, k) order
    ff, g = ff[first], g[first]
    swap = lab[ff] > lab[g]
    s0, s1 = np.where(swap, g, ff), np.where(swap, ff, g)
    P, Q = ekeys >> 32, ekeys & 0xFFFFFFFF
    E = len(ekeys)
    side = []
    for h in (s0, s1):
        kP, kQ = np.argmax(tr[h] == P[:, None], axis=1), np.argmax(tr[h] == Q[:, None], axis=1)
        uP, vP = U[h, kP, 0].astype(np.float64), U[h, kP, 1].astype(np.float64)
        uQ, vQ = U[h, kQ, 0].astype(np.float64), U[h, kQ, 1].astype(np.float64)
        du, dv = uQ - uP, vQ - vP
        side.append((uP, vP, uQ, vQ, np.sqrt(du * du + dv * dv), ch[fc[h]], h, kP, kQ))
    S = np.maximum(1.0, np.ceil(np.maximum(side[0][4], side[1][4]))).astype(np.int64) if E else np.zeros(0, np.int64)
    sums = np.zeros((2, 3, E))
    for k in range(int(S.max()) if E else 0):
        on = k < S
        t = (k + 0.5) / S[on]
        I = [_bilinear_np(atlas, s[5][on], s[0][on] + t * (s[2][on] - s[0][on]), s[1][on] + t * (s[3][on] - s[1][on]))
             for s in side]
        for end, w in enumerate((1.0 - t, t)):
            sums[end, 0, on] = sums[end, 0, on] + w * I[0]
            sums[end, 1, on] = sums[end, 1, on] + w * I[1]
            sums[end, 2, on] = sums[end, 2, on] + w
    # the ends: (g_a, g_b) of each edge's end 0 (P) and end 1 (Q), added per (g_a, g_b) in edge rank order
    ga = np.stack([cu[side[0][6], side[0][7]], cu[side[0][6], side[0][8]]], 1).reshape(-1)
    gb = np.stack([cu[side[1][6], side[1][7]], cu[side[1][6], side[1][8]]], 1).reshape(-1)
    parts = sums.transpose(2, 0, 1).reshape(-1, 3)              # [edge rank * 2 + end][3]
    xkey = (ga << 32) | gb
    order = np.argsort(xkey, kind="stable")
    xs = xkey[order]
    head = np.r_[True, xs[1:] != xs[:-1]] if len(xs) else np.zeros(0, bool)
    grp = np.cumsum(head) - 1
    pos = np.arange(len(xs)) - np.nonzero(head)[0][grp] if len(xs) else np.zeros(0, np.int64)
    tot = np.zeros((int(head.sum()), 3))
    for j in range(int(pos.max()) + 1 if len(pos) else 0):
        at = pos == j
        tot[grp[at]] = tot[grp[at]] + parts[order[at]]
    rk = xs[head]
    with np.errstate(invalid="ignore", divide="ignore"):
        Fa, Fb = tot[:, 0] / tot[:, 2], tot[:, 1] / tot[:, 2]
    seam = [(int(k >> 32), int(k & 0xFFFFFFFF), float(p), float(q)) for k, p, q in zip(rk, Fa, Fb)]
    return dict(faceChart=fc, keys=keys, cu=cu, seam=seam, smooth=sm, edges=E, seen=int(seen.sum()),
                smoothness=smoothness)


def _closest_np(U, ids, X, Y):
    """closest for arrays: U [n, 3, 2] float32, ids [n, 3], X, Y [n] float64.  Returns (d2, bw [n, 3])."""
    u = [U[:, k, 0].astype(np.float64) for k in range(3)]
    v = [U[:, k, 1].astype(np.float64) for k in range(3)]
    A = (u[1] - u[0]) * (v[2] - v[0]) - (v[1] - v[0]) * (u[2] - u[0])
    s = np.where(A > 0, 1.0, -1.0)
    w = []
    for k in range(3):
        a, b = k, (k + 1) % 3
        lo = ids[:, a] < ids[:, b]
        uP, vP = np.where(lo, u[a], u[b]), np.where(lo, v[a], v[b])
        uQ, vQ = np.where(lo, u[b], u[a]), np.where(lo, v[b], v[a])
        w.append(np.where(lo, s, -s) * ((uQ - uP) * (Y - vP) - (vQ - vP) * (X - uP)))
    S = (w[0] + w[1]) + w[2]
    inside = (A != 0.0) & (w[0] >= 0.0) & (w[1] >= 0.0) & (w[2] >= 0.0) & (S > 0.0)
    best = np.full(len(X), np.inf)
    bw = np.zeros((len(X), 3))
    for k in range(3):
        k1 = (k + 1) % 3
        dx, dy = u[k1] - u[k], v[k1] - v[k]
        l2 = dx * dx + dy * dy
        with np.errstate(invalid="ignore", divide="ignore"):
            m = ((X - u[k]) * dx + (Y - v[k]) * dy) / l2
        m = np.where(0.0 > m, 0.0, m)                           # Python's max(m, 0.0) and min(., 1.0)
        t = np.where(l2 > 0.0, np.where(1.0 < m, 1.0, m), 0.0)
        ex, ey = X - (u[k] + t * dx), Y - (v[k] + t * dy)
        d2 = ex * ex + ey * ey
        nb = d2 < best
        best = np.where(nb, d2, best)
        new = np.zeros((len(X), 3))
        new[:, k], new[:, k1] = 1.0 - t, t
        bw = np.where(nb[:, None], new, bw)
    with np.errstate(invalid="ignore", divide="ignore"):
        bin_ = np.stack([w[1] / S, w[2] / S, w[0] / S], 1)
    return np.where(inside, 0.0, best), np.where(inside[:, None], bin_, bw)


def texels_np(tris, labels, uv, charts, faceChart, atlas, corner, padding, copy_all=False, chunk=1 << 22):
    """texels, vectorised over (face, texel) pairs in chunks of about `chunk` pairs."""
    tr = np.asarray(tris, np.int64).reshape(-1, 3)
    U = np.asarray(uv, np.float32).reshape(-1, 3, 2)
    ch = np.asarray(charts, np.int64).reshape(-1, 8)
    rows, width = atlas.shape
    key = np.full(rows * width, to.EMPTY, np.uint64)
    g = float(padding + 1)
    F = np.nonzero(np.asarray(labels).reshape(-1) >= 0)[0]
    e = ch[faceChart[F]]
    xs, ys = U[F, :, 0].astype(np.float64), U[F, :, 1].astype(np.float64)
    xlo = np.maximum(e[:, 5].astype(np.float64), np.floor(np.minimum(np.minimum(xs[:, 0], xs[:, 1]), xs[:, 2])) - g)
    xhi = np.minimum((e[:, 5] + e[:, 3] - 1).astype(np.float64),
                     np.ceil(np.maximum(np.maximum(xs[:, 0], xs[:, 1]), xs[:, 2])) + g)
    ylo = np.maximum(e[:, 6].astype(np.float64), np.floor(np.minimum(np.minimum(ys[:, 0], ys[:, 1]), ys[:, 2])) - g)
    yhi = np.minimum((e[:, 6] + e[:, 4] - 1).astype(np.float64),
                     np.ceil(np.maximum(np.maximum(ys[:, 0], ys[:, 1]), ys[:, 2])) + g)
    xlo, xhi, ylo, yhi = (a.astype(np.int64) for a in (xlo, xhi, ylo, yhi))
    nw, nh = np.maximum(xhi - xlo + 1, 0), np.maximum(yhi - ylo + 1, 0)
    n = nw * nh
    ends = np.cumsum(n)
    lo = 0
    while lo < len(F):
        hi = int(np.searchsorted(ends, (ends[lo - 1] if lo else 0) + chunk, side="right"))
        hi = max(hi, lo + 1)
        sel = np.arange(lo, hi)
        cnt = n[sel]
        fi = np.repeat(sel, cnt)
        j = np.arange(int(cnt.sum())) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        X, Y = xlo[fi] + j % nw[fi], ylo[fi] + j // nw[fi]
        f = F[fi]
        d2, _ = _closest_np(U[f], tr[f], X.astype(np.float64), Y.astype(np.float64))
        k = (np.sqrt(d2).astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | f.astype(np.uint64)
        np.minimum.at(key, Y * width + X, k)
        lo = hi
    out = atlas.copy()
    hit = np.nonzero(key != to.EMPTY)[0]
    if not copy_all and len(hit):
        f = (key[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        Y, X = np.divmod(hit, width)
        _, bw = _closest_np(U[f], tr[f], X.astype(np.float64), Y.astype(np.float64))
        o = np.asarray(corner, np.float32)[f].astype(np.float64)
        off = (bw[:, 0] * o[:, 0] + bw[:, 1] * o[:, 1]) + bw[:, 2] * o[:, 2]
        out.reshape(-1)[hit] = atlas.reshape(-1)[hit].astype(np.float32) + off.astype(np.float32)
    return out, len(hit)
