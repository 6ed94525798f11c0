"""cs_mesh_refine restated in float64 (numpy element-wise operations, each rounded once, in the header's order): the
fixed and free vertices and l0 from the sorted directed edge keys, cs_texture_mesh's depth buffers
(texture_oracle.depth_buffer), the mapping, the windowed NCC and its image gradient, the face gather in the device's lane
and butterfly order (texture_photo_oracle's lane sums, vectorised), the thin plate, the three-level totals
(texture_oracle.tree_total) and the halving line search.  evaluate() also takes float64 vertices and fixed depth
buffers, for the gradient checks."""
import math

import numpy as np

import texture_oracle as to

EMPTY = to.EMPTY
LANES = 32
M32 = np.uint64(0xFFFFFFFF)
FLOOR = 1.0                      # rule 4: the variance floor, grey levels^2
CAP = 2.0                        # rule 8: the longest step, in units of alpha l0


def topology(V, tris, X):
    """Rule 1: dict with free [V] bool, the neighbour lists (nb, nstart, nend), the corners sorted by vertex (corner,
    cstart, cend), l0 and F.  X: the input vertices as float64."""
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    T = len(t)
    a, b = t.reshape(-1), np.roll(t, -1, axis=1).reshape(-1)
    keys = np.empty(6 * T, np.uint64)
    keys[0::2] = (a.astype(np.uint64) << np.uint64(32)) | b.astype(np.uint64)
    keys[1::2] = (b.astype(np.uint64) << np.uint64(32)) | a.astype(np.uint64)
    ks = np.sort(keys)
    head = np.ones(len(ks), bool)
    head[1:] = ks[1:] != ks[:-1]
    starts = np.nonzero(head)[0]
    lens = np.diff(np.append(starts, len(ks)))
    ua = (ks[starts] >> np.uint64(32)).astype(np.int64)
    ub = (ks[starts] & M32).astype(np.int64)
    used = np.zeros(V, bool)
    used[ua] = True
    bad = np.zeros(V, bool)
    bad[ua[lens != 2]] = True
    free = used & ~bad
    ids = np.arange(V)
    nstart, nend = np.searchsorted(ua, ids, "left"), np.searchsorted(ua, ids, "right")
    # the distinct undirected edges' lengths at their sorted positions, totalled in coop.cuh's order
    length = np.zeros(len(ks))
    up = ua < ub
    d = X[ub[up]] - X[ua[up]]
    length[starts[up]] = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    l0 = to.tree_total(length) / float(len(starts) // 2) if T else 0.0
    corner = np.argsort(t.reshape(-1), kind="stable")
    cv = t.reshape(-1)[corner]
    cstart, cend = np.searchsorted(cv, ids, "left"), np.searchsorted(cv, ids, "right")
    return dict(free=free, nb=ub, nstart=nstart, nend=nend, corner=corner, cstart=cstart, cend=cend, l0=l0,
                F=int(free.sum()))


def _ranked(start, end, sel=None):
    """Rank loops over per-vertex ranges: yields (vertices, list positions) for rank 0, 1, ..."""
    n = end - start
    top = int(n.max()) if len(n) else 0
    for r in range(top):
        v = np.nonzero((n > r) if sel is None else ((n > r) & sel))[0]
        yield v, start[v] + r


def face_corners(X, tr, f, cam):
    """The corners P [n, 3, 3] of faces f and their projections u, v, z [n, 3] in cam (K, R, t, W, H)."""
    K, R, t = cam[:3]
    P = X[tr[f]]
    u, v, z = to.project(K, R, t, P)
    return P, u, v, z


def weights(tr, f, u, v, z, x, y):
    """Rule 3's phi [n, 3] at pixels (x, y) of faces f (rule 2's edge values, screen and perspective-correct
    weights)."""
    A = to.area2(u, v)
    s = np.where(A > 0, 1.0, -1.0)
    n = np.arange(len(f))
    w = []
    for k in range(3):
        a, b = k, (k + 1) % 3
        lo = tr[f, a] < tr[f, b]
        P, Q = np.where(lo, a, b), np.where(lo, b, a)
        du, dv = u[n, Q] - u[n, P], v[n, Q] - v[n, P]
        w.append(np.where(lo, s, -s) * (du * (y - v[n, P]) - dv * (x - u[n, P])))
    S = (w[0] + w[1]) + w[2]
    t0, t1, t2 = (w[1] / S) / z[:, 0], (w[2] / S) / z[:, 1], (w[0] / S) / z[:, 2]
    sm = (t0 + t1) + t2
    return np.stack([t0 / sm, t1 / sm, t2 / sm], 1)


def normals(P):
    e1, e2 = P[..., 1, :] - P[..., 0, :], P[..., 2, :] - P[..., 0, :]
    return np.stack([e1[..., 1] * e2[..., 2] - e1[..., 2] * e2[..., 1], e1[..., 2] * e2[..., 0] - e1[..., 0] * e2[..., 2],
                     e1[..., 0] * e2[..., 1] - e1[..., 1] * e2[..., 0]], -1)


def dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def pair_pass(imgs, cams, bufs, X, tr, i, j, rho, depthTol):
    """Rules 3 to 6 for pair (i, j): dict with the pair's total of e, the scored count, S [T, 3] (the face gather),
    and the mapped and scored masks."""
    K, R, t, W, H = cams[i]
    Ki, Ri, ti = K, R, t
    Kj, Rj, tj, Wj, Hj = cams[j]
    Ii = np.asarray(imgs[i], np.float32).astype(np.float64)
    Ij = np.asarray(imgs[j], np.float32).astype(np.float64)
    T = len(tr)
    keys = bufs[i].reshape(-1)
    q = np.nonzero(keys != EMPTY)[0]
    f = (keys[q] & M32).astype(np.int64)
    y, x = (q // W).astype(np.float64), (q % W).astype(np.float64)
    P, u, v, z = face_corners(X, tr, f, cams[i])
    phi = weights(tr, f, u, v, z, x, y)
    Xp = (phi[:, 0:1] * P[:, 0] + phi[:, 1:2] * P[:, 1]) + phi[:, 2:3] * P[:, 2]
    r = Xp - to.centre(Ri, ti)[None, :]
    nr = dot(normals(P), r)
    uj, vj, zj = to.project(Kj, Rj, tj, Xp)
    with np.errstate(invalid="ignore"):
        ok = (zj > 0) & (uj >= 0) & (uj <= Wj - 1.0) & (vj >= 0) & (vj <= Hj - 1.0) & (nr != 0)
    px = np.where(ok, np.floor(uj + 0.5), 0).astype(np.int64)
    py = np.where(ok, np.floor(vj + 0.5), 0).astype(np.int64)
    kj = bufs[j][py, px]
    dep = (kj >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        ok &= (kj == EMPTY) | ((kj & M32) == f.astype(np.uint64)) | (zj <= dep * (1.0 + depthTol))
    m = np.nonzero(ok)[0]
    uj, vj, zj, r, nr = uj[m], vj[m], zj[m], r[m], nr[m]
    x0 = np.minimum(np.floor(uj), Wj - 2).astype(np.int64)
    y0 = np.minimum(np.floor(vj), Hj - 2).astype(np.int64)
    fx, fy = uj - x0, vj - y0
    I00, I10, I01, I11 = Ij[y0, x0], Ij[y0, x0 + 1], Ij[y0 + 1, x0], Ij[y0 + 1, x0 + 1]
    a = I00 + fx * (I10 - I00)
    b = I01 + fx * (I11 - I01)
    gu = (I10 - I00) + fy * ((I11 - I01) - (I10 - I00))
    gv = b - a
    d = [(Rj[k, 0] * r[:, 0] + Rj[k, 1] * r[:, 1]) + Rj[k, 2] * r[:, 2] for k in range(3)]
    au = (((Kj[0, 0] * d[0] + Kj[0, 1] * d[1]) + Kj[0, 2] * d[2]) - uj * d[2]) / zj
    av = (((Kj[1, 0] * d[0] + Kj[1, 1] * d[1]) + Kj[1, 2] * d[2]) - vj * d[2]) / zj
    n = H * W
    mapped = np.zeros(n, bool)
    J = np.zeros(n)
    c = np.zeros(n)
    mapped[q[m]] = True
    J[q[m]] = a + fy * (b - a)
    c[q[m]] = (gu * au + gv * av) / nr

    # rule 4 over the interior (H - 2 rho) x (W - 2 rho), windows in row-major order
    M2, J2 = mapped.reshape(H, W), J.reshape(H, W)
    scored = np.zeros((H, W), bool)
    A_ = np.zeros((H, W))
    B_, C_, D_, e_ = A_.copy(), A_.copy(), A_.copy(), A_.copy()
    if H > 2 * rho and W > 2 * rho:
        win = lambda a2, dy, dx: a2[rho + dy:H - rho + dy, rho + dx:W - rho + dx]
        allm = np.ones((H - 2 * rho, W - 2 * rho), bool)
        sI = sJ = sII = sJJ = sIJ = np.zeros((H - 2 * rho, W - 2 * rho))
        for dy in range(-rho, rho + 1):
            for dx in range(-rho, rho + 1):
                allm = allm & win(M2, dy, dx)
                ia, jb = win(Ii, dy, dx), win(J2, dy, dx)
                sI, sJ = sI + ia, sJ + jb
                sII, sJJ, sIJ = sII + ia * ia, sJJ + jb * jb, sIJ + ia * jb
        nn = float((2 * rho + 1) ** 2)
        mI, mJ = sI / nn, sJ / nn
        rI, rJ = sII / nn - mI * mI, sJJ / nn - mJ * mJ
        vI, vJ = np.where(rI < FLOOR, FLOOR, rI), np.where(rJ < FLOOR, FLOOR, rJ)
        qq = np.sqrt(vI * vJ)
        ncc = (sIJ / nn - mI * mJ) / qq
        A = 1.0 / qq
        Cc = np.where(rJ < FLOOR, 0.0, ncc / vJ)
        inner = (slice(rho, H - rho), slice(rho, W - rho))
        scored[inner] = allm
        A_[inner] = np.where(allm, A, 0.0)
        B_[inner] = np.where(allm, mI * A, 0.0)
        C_[inner] = np.where(allm, Cc, 0.0)
        D_[inner] = np.where(allm, Cc * mJ, 0.0)
        e_[inner] = np.where(allm, 1.0 - ncc, 0.0)
    total = to.tree_total(e_.reshape(-1))

    # rule 5 at the mapped pixels: the scored x whose window holds y, in row-major order of x
    pad = lambda a2: np.pad(a2, rho)
    Ap, Bp, Cp, Dp, Sp = pad(A_), pad(B_), pad(C_), pad(D_), pad(scored)
    SA = SB = SC = SD = np.zeros((H, W))
    for dy in range(-rho, rho + 1):
        for dx in range(-rho, rho + 1):
            sl = (slice(rho + dy, rho + dy + H), slice(rho + dx, rho + dx + W))
            sel = Sp[sl]
            SA = np.where(sel, SA + Ap[sl], SA)
            SB = np.where(sel, SB + Bp[sl], SB)
            SC = np.where(sel, SC + Cp[sl], SC)
            SD = np.where(sel, SD + Dp[sl], SD)
    g = ((Ii * SA - SB) - J2 * SC) + SD
    s = ((-g / float((2 * rho + 1) ** 2)) * c.reshape(H, W)).reshape(-1)

    # rule 6: the mapped pixels of each face by box index, lane sums in ascending row, then the butterfly
    mq = q[m]
    fm = f[m]
    um, vm = u[m], v[m]
    xlo = np.maximum(0.0, np.ceil(np.minimum(np.minimum(um[:, 0], um[:, 1]), um[:, 2]))).astype(np.int64)
    ylo = np.maximum(0.0, np.ceil(np.minimum(np.minimum(vm[:, 0], vm[:, 1]), vm[:, 2]))).astype(np.int64)
    xhi = np.minimum(W - 1.0, np.floor(np.maximum(np.maximum(um[:, 0], um[:, 1]), um[:, 2]))).astype(np.int64)
    bw = xhi - xlo + 1
    bi = (mq // W - ylo) * bw + (mq % W - xlo)
    lane, row = bi % LANES, bi // LANES
    val = s[mq][:, None] * phi[m]
    acc = np.zeros((T, LANES, 3))
    for rr in np.unique(row):
        sel = row == rr
        acc[fm[sel], lane[sel]] = acc[fm[sel], lane[sel]] + val[sel]
    S = to._butterfly(acc.transpose(0, 2, 1).reshape(-1, LANES)).reshape(T, 3) if T else np.zeros((0, 3))
    return dict(total=total, scored=int(scored.sum()), S=S, mapped=mapped, scoredMask=scored.reshape(-1), s=s)


def evaluate(imgs, cams, X, tr, pairs, topo, rho, depthTol, smoothness, P0=None, bufs=None):
    """One evaluation at the vertices X (float64 [V, 3], normally float32 values): dict with ep, es, G [V, 3], g2,
    the scored count, and per pair its masks; bufs: the depth buffers (None: rule 2 from X rounded to float)."""
    tr = np.asarray(tr, np.int64)
    V, T = len(X), len(tr)
    names = sorted({a for p in pairs for a in p})
    if bufs is None:
        Xf = X.astype(np.float32)
        bufs = {a: to.depth_buffer(*cams[a][:3], cams[a][3], cams[a][4], Xf, tr) for a in names}
    acc = np.zeros((T, 3))
    tot = 0.0
    scored = 0
    per = []
    for i, j in pairs:
        r = pair_pass(imgs, cams, bufs, X, tr, i, j, rho, depthTol)
        acc = acc + r["S"]
        tot = tot + r["total"]
        scored += r["scored"]
        per.append(r)
    P0 = scored if P0 is None else P0
    free = topo["free"]
    # rule 7: U and E_s
    U = np.zeros((V, 3))
    a = np.zeros((V, 3))
    for v, pos in _ranked(topo["nstart"], topo["nend"], free):
        a[v] = a[v] + X[topo["nb"][pos]]
    deg = (topo["nend"] - topo["nstart"]).astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        U[free] = a[free] / deg[free, None] - X[free]
    u2 = np.where(free, (U[:, 0] * U[:, 0] + U[:, 1] * U[:, 1]) + U[:, 2] * U[:, 2], 0.0)
    Ds = float(topo["F"]) * (topo["l0"] * topo["l0"])
    es = to.tree_total(u2) / Ds if Ds > 0 else 0.0
    ks = 2.0 / Ds if Ds > 0 else 0.0
    # rule 6's vertex sums and rule 7's gradient
    nf = normals(X[tr]) if T else np.zeros((0, 3))
    accf = acc.reshape(-1)
    gp = np.zeros((V, 3))
    for v, pos in _ranked(topo["cstart"], topo["cend"], free):
        c = topo["corner"][pos]
        gp[v] = gp[v] + accf[c][:, None] * nf[c // 3]
    gs = -U
    for v, pos in _ranked(topo["nstart"], topo["nend"], free):
        w = topo["nb"][pos]
        fw = free[w]
        v, w = v[fw], w[fw]
        gs[v] = gs[v] + U[w] / deg[w, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        G = np.where(free[:, None], gp / float(P0) + smoothness * (ks * gs), 0.0)
    g2 = to.tree_total(np.where(free, (G[:, 0] * G[:, 0] + G[:, 1] * G[:, 1]) + G[:, 2] * G[:, 2], 0.0))
    ep = tot / float(P0) if P0 else 0.0
    return dict(ep=ep, es=es, G=G, g2=g2, scored=scored, P0=P0, pairs=per, bufs=bufs, acc=acc)


def step_from(X32, G, free, alpha, l0, grms):
    """Rule 8's candidate (float32 [V, 3]) from the accepted vertices X32."""
    al = alpha * l0
    scale, cap = al / grms, CAP * al
    P = X32.astype(np.float64)
    d = -(scale * G)
    ln = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    big = ln > cap
    with np.errstate(invalid="ignore", divide="ignore"):
        d = np.where(big[:, None], d * (cap / ln)[:, None], d)
    return np.where(free[:, None], (P + d).astype(np.float32), X32)


def refine(images, Ks, Rs, ts, verts, tris, pairs, windowRadius=4, smoothness=0.2, step=0.1, maxIterations=8,
           depthTol=0.01, trace=None):
    """The whole call: dict with vertices (float32 [V, 3]), info [4], stats [8] and the energies of the evaluations
    (trace, when a list is given, receives (E, accepted) per candidate)."""
    X32 = np.asarray(verts, np.float32).reshape(-1, 3)
    tr = np.asarray(tris, np.int64).reshape(-1, 3)
    V, T = len(X32), len(tr)
    pairs = [(int(a), int(b)) for a, b in np.asarray(pairs, np.int64).reshape(-1, 2)]
    cams = [(np.asarray(Ks[a], np.float64), np.asarray(Rs[a], np.float64), np.asarray(ts[a], np.float64),
             images[a].shape[1], images[a].shape[0]) for a in range(len(images))]
    if T == 0:
        return dict(vertices=X32.copy(), info=[0.0] * 4, stats=[len(pairs), 0, V, 0, 0, 0, 0, 1])
    if not to.validate(X32, tr):
        return dict(vertices=None, info=[0.0] * 4, stats=[len(pairs), 0, 0, 0, 0, 0, 0, 2])
    X = X32.astype(np.float64)
    topo = topology(V, tr, X)
    F, l0 = topo["F"], topo["l0"]
    ev = evaluate(images, cams, X, tr, pairs, topo, windowRadius, depthTol, smoothness)
    P0 = ev["P0"]
    e0 = (ev["ep"], ev["es"])
    evals, accepted, halvings = 1, 0, 0
    acc, eacc, G, g2 = X32.copy(), e0, ev["G"], ev["g2"]
    E = lambda e: e[0] + smoothness * e[1]
    if P0 == 0:
        status = 1
    else:
        alpha = step
        while True:
            grms = math.sqrt(g2 / float(F)) if F else 0.0
            if grms == 0.0 or alpha < step / 1024.0:
                status = 0
                break
            if evals - 1 == maxIterations:
                status = 3
                break
            cand = step_from(acc, G, topo["free"], alpha, l0, grms)
            ec = evaluate(images, cams, cand.astype(np.float64), tr, pairs, topo, windowRadius, depthTol, smoothness,
                          P0=P0)
            evals += 1
            e = (ec["ep"], ec["es"])
            ok = E(e) < E(eacc)
            if trace is not None:
                trace.append((E(e), ok))
            if ok:
                acc, eacc, G, g2 = cand, e, ec["G"], ec["g2"]
                accepted += 1
                alpha, halvings = step, 0
            else:
                alpha, halvings = alpha * 0.5, halvings + 1
    return dict(vertices=acc, info=[e0[0], e0[1], eacc[0], eacc[1]],
                stats=[len(pairs), F, V - F, P0, evals, accepted, halvings, status], topo=topo)
