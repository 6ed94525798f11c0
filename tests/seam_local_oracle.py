"""cs_level_texture_seams_local restated in float64 with numpy (element-wise operations, each rounded once, in the
header's order): rule 1 by seam_oracle.build_np, rule 7's texel keys by seam_oracle's closest-point and box helpers,
rule 3's sides, positions and bilinear reads by seam_oracle's, then the seam texels, the strip, the 5-point system,
its exact solution (scipy.sparse direct solve), a Jacobi-PCG for the iteration count and the output."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

import seam_oracle as so
import texture_oracle as to


def texel_keys(tris, labels, uv, charts, faceChart, atlas, padding):
    """Rule 2 (cs_level_texture_seams's rule 7): every atlas texel's key face, -1 outside the domain."""
    tr = np.asarray(tris, np.int64).reshape(-1, 3)
    U = np.asarray(uv, np.float32).reshape(-1, 3, 2)
    ch = np.asarray(charts, np.int64).reshape(-1, 8)
    rows, width = atlas.shape
    key = np.full(rows * width, to.EMPTY, np.uint64)
    g = so.box_grow(padding)
    for f in np.nonzero(np.asarray(labels).reshape(-1) >= 0)[0]:
        e = ch[faceChart[f]]
        xs, ys = U[f, :, 0].astype(np.float64), U[f, :, 1].astype(np.float64)
        xlo = int(max(float(e[5]), np.floor(min(min(xs[0], xs[1]), xs[2])) - g))
        xhi = int(min(float(e[5] + e[3] - 1), np.ceil(max(max(xs[0], xs[1]), xs[2])) + g))
        ylo = int(max(float(e[6]), np.floor(min(min(ys[0], ys[1]), ys[2])) - g))
        yhi = int(min(float(e[6] + e[4] - 1), np.ceil(max(max(ys[0], ys[1]), ys[2])) + g))
        if xhi < xlo or yhi < ylo:
            continue
        Y, X = np.mgrid[ylo:yhi + 1, xlo:xhi + 1]
        X, Y = X.reshape(-1), Y.reshape(-1)
        n = len(X)
        d2, _ = so._closest_np(np.repeat(U[f][None], n, 0), np.repeat(tr[f][None], n, 0), X.astype(np.float64),
                               Y.astype(np.float64))
        k = (np.sqrt(d2).astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(f)
        np.minimum.at(key, Y * width + X, k)
    face = np.where(key == to.EMPTY, -1, (key & np.uint64(0xFFFFFFFF)).astype(np.int64))
    return face.reshape(rows, width)


def seam_sides(tris, labels, uv):
    """Rule 3's seam edges in sorted key order: per side s (0: the lower label) the face and the uv of the ends P and
    Q, and the sample count S."""
    tr = np.asarray(tris, np.int64).reshape(-1, 3)
    lab = np.asarray(labels, np.int64).reshape(-1)
    U = np.asarray(uv, np.float32).reshape(-1, 3, 2)
    seen = lab >= 0
    nbr = so._adjacency_np(tr)
    ff, kk = np.nonzero(nbr >= 0)
    g = nbr[ff, kk]
    ok = seen[ff] & seen[g] & (lab[ff] != lab[g])
    ff, kk, g = ff[ok], kk[ok], g[ok]
    pa, pb = tr[ff, kk], tr[ff, (kk + 1) % 3]
    ekeys, first = np.unique((np.minimum(pa, pb) << 32) | np.maximum(pa, pb), return_index=True)
    ff, g = ff[first], g[first]
    swap = lab[ff] > lab[g]
    faces = (np.where(swap, g, ff), np.where(swap, ff, g))
    P, Q = ekeys >> 32, ekeys & 0xFFFFFFFF
    sides, lens = [], []
    for h in faces:
        kP, kQ = np.argmax(tr[h] == P[:, None], axis=1), np.argmax(tr[h] == Q[:, None], axis=1)
        uP, vP = U[h, kP, 0].astype(np.float64), U[h, kP, 1].astype(np.float64)
        uQ, vQ = U[h, kQ, 0].astype(np.float64), U[h, kQ, 1].astype(np.float64)
        du, dv = uQ - uP, vQ - vP
        lens.append(np.sqrt(du * du + dv * dv))
        sides.append((h, uP, vP, uQ, vQ))
    S = np.maximum(1.0, np.ceil(np.maximum(lens[0], lens[1]))).astype(np.int64) if len(ekeys) else np.zeros(0, np.int64)
    return sides, S


def seam_texels(sides, S, charts, faceChart, atlas):
    """Rule 3: (seam texel indices in texel order, f*), from the samples' slots (seam edge, side, k)."""
    ch = np.asarray(charts, np.int64).reshape(-1, 8)
    rows, width = atlas.shape
    E = len(S)
    base = 2 * (np.cumsum(S) - S)
    M = int(S.sum())
    tex = np.zeros(2 * M, np.int64)
    val = np.zeros(2 * M)
    e = [ch[faceChart[s[0]]] for s in sides]
    for k in range(int(S.max()) if E else 0):
        on = k < S
        t = (k + 0.5) / S[on]
        X = [s[1][on] + t * (s[3][on] - s[1][on]) for s in sides]
        Y = [s[2][on] + t * (s[4][on] - s[2][on]) for s in sides]
        m = 0.5 * (so._bilinear_np(atlas, e[0][on], X[0], Y[0]) + so._bilinear_np(atlas, e[1][on], X[1], Y[1]))
        for s in range(2):
            c = e[s][on]
            tx = np.minimum(np.maximum(np.floor(X[s] + 0.5), c[:, 5]), c[:, 5] + c[:, 3] - 1).astype(np.int64)
            ty = np.minimum(np.maximum(np.floor(Y[s] + 0.5), c[:, 6]), c[:, 6] + c[:, 4] - 1).astype(np.int64)
            slot = base[on] + s * S[on] + k
            tex[slot] = ty * width + tx
            val[slot] = m
    order = np.argsort(tex, kind="stable")
    ts = tex[order]
    head = np.r_[True, ts[1:] != ts[:-1]] if len(ts) else np.zeros(0, bool)
    grp = np.cumsum(head) - 1
    pos = np.arange(len(ts)) - np.nonzero(head)[0][grp] if len(ts) else np.zeros(0, np.int64)
    tot = np.zeros(int(head.sum()))
    for j in range(int(pos.max()) + 1 if len(pos) else 0):
        at = pos == j
        tot[grp[at]] = tot[grp[at]] + val[order[at]]
    cnt = np.bincount(grp, minlength=len(tot)).astype(np.float64)
    return ts[head], tot / cnt, M


def neighbours(chart):
    """Rule 2: per direction k in the header's order, (valid [rows, width], index offset) of the neighbour."""
    rows, width = chart.shape
    out = []
    for dx, dy in ((-1, 0), (1, 0), (0, -1), (0, 1)):
        other = np.full((rows, width), -2, np.int64)
        ys, yd = slice(max(0, -dy), rows - max(0, dy)), slice(max(0, dy), rows - max(0, -dy))
        xs, xd = slice(max(0, -dx), width - max(0, dx)), slice(max(0, dx), width - max(0, -dx))
        other[ys, xs] = chart[yd, xd]
        out.append(((chart >= 0) & (other == chart), dy * width + dx))
    return out


def strip(chart, seam, w):
    """Rule 4: the hop distance after w synchronous rounds (-1 outside the domain, a large value unreached)."""
    FAR = np.iinfo(np.int64).max // 2
    d = np.where(chart >= 0, FAR, -1).reshape(-1)
    d[seam] = 0
    nb = neighbours(chart)
    for _ in range(w):
        new = d.copy()
        for ok, off in nb:
            i = np.nonzero(ok.reshape(-1) & (d > 0))[0]
            dj = d[i + off]
            new[i] = np.minimum(new[i], np.where(dj < FAR, dj + 1, FAR))
        d = new
    return d, FAR


def system(chart, d, w, seam, fstar, atlas):
    """Rule 5: (A as scipy CSC, b, free texel indices in row-major order)."""
    g = atlas.reshape(-1).astype(np.float64)
    free = np.nonzero((d >= 1) & (d <= w))[0]
    N = len(free)
    idx = np.full(d.shape, -1, np.int64)
    idx[free] = np.arange(N)
    sval = np.zeros(d.shape)
    sval[seam] = fstar - g[seam]
    diag = np.zeros(N)
    b = np.zeros(N)
    I, J = [], []
    for ok, off in neighbours(chart):
        has = ok.reshape(-1)[free]
        j = free + off
        diag = diag + has
        isfree = has & (idx[np.where(has, j, 0)] >= 0)
        isseam = has & (d[np.where(has, j, 0)] == 0)
        b = np.where(isseam, b + sval[np.where(has, j, 0)], b)
        I.append(np.nonzero(isfree)[0])
        J.append(idx[j[isfree]])
    I, J = np.concatenate(I), np.concatenate(J)
    A = sp.csr_matrix((-np.ones(len(I)), (I, J)), shape=(N, N)) + sp.diags(diag)
    return A.tocsc(), b, free


def pcg(A, b, tol, maxIterations):
    """Jacobi-PCG from 0 with rule 6's stop rule (sums in numpy's order).  Returns (x, iterations, converged)."""
    d = A.diagonal()
    x = np.zeros(len(b))
    r = b.copy()
    z = r / d if len(b) else r
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


def level(verts, tris, labels, uv, charts, atlas, padding=2, stripWidth=20, tol=1e-4, maxIterations=1000):
    """The whole call with the exact solve: dict with stats (CG iterations from the PCG above), info [3] (the residual
    and max |delta| of the exact solution), the atlas, and the pieces the tests look at."""
    atlas = np.asarray(atlas, np.float32)
    T = len(np.asarray(tris).reshape(-1, 3))
    if T == 0:
        return dict(stats=[0] * 7 + [1], info=[0.0, 0.0, 0.0], atlas=atlas.copy())
    bd = so.build_np(verts, tris, labels, uv, charts, atlas, 0.0)
    if bd is None:
        return dict(stats=[0] * 7 + [2], info=[0.0, 0.0, 0.0])
    fc = bd["faceChart"]
    face = texel_keys(tris, labels, uv, charts, fc, atlas, padding)
    chart = np.where(face >= 0, fc[np.maximum(face, 0)], -1)
    sides, S = seam_sides(tris, labels, uv)
    seam, fstar, M = seam_texels(sides, S, charts, fc, atlas)
    assert (chart.reshape(-1)[seam] >= 0).all()
    d, FAR = strip(chart, seam, stripWidth)
    A, b, free = system(chart, d, stripWidth, seam, fstar, atlas)
    delta = spl.spsolve(A, b) if len(b) else np.zeros(0)
    if len(b) == 1:
        delta = np.atleast_1d(delta)
    _, its, conv = pcg(A, b, tol, maxIterations)
    g = atlas.reshape(-1).astype(np.float64)
    out = atlas.copy().reshape(-1)
    out[seam] = fstar.astype(np.float32)
    out[free] = (g[free] + delta).astype(np.float32)
    status = 1 if len(seam) == 0 else 0 if conv else 3
    e = fstar - g[seam]
    stats = [bd["seen"], len(S), M, len(seam), len(free), int((chart >= 0).sum()), its, status]
    info = [to.tree_total(e * e), 0.0, float(np.abs(delta).max()) if len(delta) else 0.0]
    return dict(stats=stats, info=info, atlas=out.reshape(atlas.shape), A=A, b=b, delta=delta, free=free, seam=seam,
                fstar=fstar, d=d, FAR=FAR, chart=chart, faceChart=fc)
