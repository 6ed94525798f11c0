"""cs_level_texture_seams restated in float64 (numpy scalars and element-wise operations, each rounded once, in the
header's order): the input check, the unknowns, the seam and smoothness rows, the system and its exact solution
(scipy.sparse direct solve), a float64 Jacobi-PCG with the same preconditioner, the seam energies in coop.cuh's
three-level order, and the texel stage."""
import math

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

import texture_oracle as to


def chart_of(uv, label, charts, rows, width):
    """Rule 1: the chart whose rectangle holds floor of corner 0's uv and whose image is the label, or -1."""
    x, y = math.floor(float(uv[0, 0])), math.floor(float(uv[0, 1]))
    if not (0 <= x < width and 0 <= y < rows):
        return -1
    for c, e in enumerate(charts):
        if e[5] <= x < e[5] + e[3] and e[6] <= y < e[6] + e[4] and e[0] == label:
            return c
    return -1


def bilinear(atlas, e, x, y):
    x0, y0 = math.floor(x), math.floor(y)
    fx, fy = x - x0, y - y0
    xl, xh, yl, yh = e[5], e[5] + e[3] - 1, e[6], e[6] + e[4] - 1
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
    # smoothness rows: distinct unknown pairs over the edges of seen faces
    sm = sorted({(min(cu[f, k], cu[f, (k + 1) % 3]), max(cu[f, k], cu[f, (k + 1) % 3]))
                 for f in np.nonzero(seen)[0] for k in range(3)})
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
        f, g = edges[key]
        if lab[f] > lab[g]:
            f, g = g, f
        P, Q = key >> 32, key & 0xFFFFFFFF
        side = []
        for h in (f, g):
            kP, kQ = list(tr[h]).index(P), list(tr[h]).index(Q)
            uP, vP = float(U[h, kP, 0]), float(U[h, kP, 1])
            uQ, vQ = float(U[h, kQ, 0]), float(U[h, kQ, 1])
            du, dv = uQ - uP, vQ - vP
            side.append((uP, vP, uQ, vQ, math.sqrt(du * du + dv * dv), charts[fc[h]], (h, kP, kQ)))
        S = int(max(1.0, math.ceil(max(side[0][4], side[1][4]))))
        sums = [[0.0, 0.0, 0.0], [0.0, 0.0, 0.0]]
        for k in range(S):
            t = (k + 0.5) / S
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
        for part in ends[(ga, gb)]:
            s = [s[c] + part[c] for c in range(3)]
        seam.append((ga, gb, s[0] / s[2], s[1] / s[2]))
    return dict(faceChart=fc, keys=keys, cu=cu, seam=seam, smooth=sm, edges=len(edges), seen=int(seen.sum()),
                smoothness=smoothness)


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
        if d2 < best:
            best = d2
            bw = [0.0, 0.0, 0.0]
            bw[k], bw[k1] = 1.0 - t, t
    return best, tuple(bw)


def texels(tris, labels, uv, charts, faceChart, atlas, corner, padding, copy_all=False):
    """Rule 7 given the float corner offsets [T, 3]: (levelled atlas, texels visited)."""
    tr = np.asarray(tris, np.int64).reshape(-1, 3)
    U = np.asarray(uv, np.float32).reshape(-1, 3, 2)
    rows, width = atlas.shape
    key = np.full(rows * width, to.EMPTY, np.uint64)
    g = float(padding + 1)
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
                k = (np.uint64(np.float32(math.sqrt(d2)).view(np.uint32)) << np.uint64(32)) | np.uint64(f)
                i = y * width + x
                if k < key[i]:
                    key[i] = k
    out = atlas.copy()
    hit = np.nonzero(key != to.EMPTY)[0]
    if not copy_all:
        for i in hit:
            f = int(key[i] & np.uint64(0xFFFFFFFF))
            y, x = divmod(int(i), width)
            _, bw = closest(U[f], tr[f], float(x), float(y))
            o = corner[f]
            off = (bw[0] * float(o[0]) + bw[1] * float(o[1])) + bw[2] * float(o[2])
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
