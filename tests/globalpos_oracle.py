"""A float64 statement of cs_global_positioning (include/cudasift_b200.h): the used observations and their rays, the
start draws, the BATA residual v - s (X - c) with the corrector's loss scaling, Levenberg-Marquardt with each scale
eliminated from its own block, the points by Schur, block-Jacobi PCG on the 3 x 3 camera system, the scale's lower
bound, and the final gauge.  Sums are numpy's, so results agree with the device to rounding."""
import numpy as np

SMIN = 1e-6
M64 = (1 << 64) - 1


def splitmix64(z):
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def draw(seed, kind, i, j):
    x = splitmix64((seed + 0x9E3779B97F4A7C15 * ((((kind << 32) | i) * 3 + j) & M64)) & M64)
    return 2.0 * ((x >> 11) * 2.0 ** -53) - 1.0


def loss(kind, c2, s):
    """(c^2 rho(s / c^2), rho') of cs_bundle_adjust_intrinsics' losses, elementwise."""
    if kind == 0:
        return s, np.ones_like(s)
    u = s / c2
    if kind == 1:
        q = np.sqrt(1.0 + u)
        return c2 * (2.0 * u / (q + 1.0)), 1.0 / q
    return c2 * np.log1p(u), 1.0 / (1.0 + u)


def observations(xy, Ks, Rs, offsets, members, use=None):
    """The used observations: (k [O], a [O], v [O, 3]) in track order, then member order, and the participating
    tracks."""
    ks, as_, vs = [], [], []
    has = np.isfinite(Rs).all(axis=(1, 2))
    for k in range(len(offsets) - 1):
        got = []
        for m in range(offsets[k], offsets[k + 1]):
            a, f = members[m]
            if not (0 <= a < len(xy) and 0 <= f < len(xy[a])) or not np.isfinite(xy[a][f]).all():
                continue
            if not has[a] or (use is not None and not use[m]):
                continue
            x, y = float(xy[a][f][0]), float(xy[a][f][1])
            K = Ks[a]
            cy = (y - K[1, 2]) / K[1, 1]
            cx = (x - K[0, 2] - K[0, 1] * cy) / K[0, 0]
            w = Rs[a].T @ np.array([cx, cy, 1.0])
            got.append((k, a, w / np.linalg.norm(w)))
        if len(got) >= 2:
            for k_, a_, v_ in got:
                ks.append(k_)
                as_.append(a_)
                vs.append(v_)
    return np.array(ks, np.int64), np.array(as_, np.int64), np.array(vs).reshape(-1, 3)


def residual(c, X, s, k, a, v):
    d = X[k] - c[a]
    return d, v - s[:, None] * d


def damp(d, lam):
    return d + lam * np.clip(d, 1e-6, 1e32)


def position(xy, Ks, Rs, offsets, members, use=None, ref=0, seed=0, kind=0, lossScale=1.0, maxIterations=100,
             maxLinear=100, tol=1e-6):
    """The call's outputs: dict(t, points, cost, trace, stats (those the statement fixes: [3] [4] [5] [6] [7]))."""
    C, T = len(xy), len(offsets) - 1
    Rs = np.asarray(Rs, np.float64)
    k, a, v = observations(xy, Ks, Rs, offsets, members, use)
    O = len(k)
    c2 = lossScale * lossScale
    c = np.array([[0.0] * 3 if i == ref else [draw(seed, 0, i, j) for j in range(3)] for i in range(C)])
    X = np.array([[draw(seed, 1, i, j) for j in range(3)] for i in range(T)]).reshape(T, 3)
    s = np.ones(O)
    pos = np.zeros(C, bool)
    pos[a] = True
    free = pos.copy()
    free[ref] = False
    part = np.zeros(T, bool)
    part[k] = True

    d, r = residual(c, X, s, k, a, v)
    terms, w2 = loss(kind, c2, np.sum(r * r, 1))
    cost0 = cost = terms.sum()
    lam, trace, cgTotal, accepted = 1e-3, [], 0, 0
    I3 = np.eye(3)
    for it in range(maxIterations if O else 0):
        h = damp(w2 * np.sum(d * d, 1), lam)
        f = w2 / h
        P = (w2 * s * s)[:, None, None] * (I3 - f[:, None, None] * np.einsum("oi,oj->oij", d, d))
        beta = (w2 * s)[:, None] * (r - (f * np.sum(d * r, 1))[:, None] * d)
        dg = w2 * s * s
        V = np.zeros((T, 3, 3))
        np.add.at(V, k, P)
        dgk = np.zeros(T)
        np.add.at(dgk, k, dg)
        V += (lam * np.clip(dgk, 1e-6, 1e32))[:, None, None] * I3
        V[~part] = I3
        bX = np.zeros((T, 3))
        np.add.at(bX, k, beta)
        ok = np.all(np.linalg.eigvalsh(V[part]) > 0)
        cgIt, cand = 0, np.nan
        if ok:
            Vi = np.linalg.inv(V)
            q = np.einsum("kij,kj->ki", Vi, bX)
            U = np.zeros((C, 3, 3))
            np.add.at(U, a, P)
            dga = np.zeros(C)
            np.add.at(dga, a, dg)
            U += (lam * np.clip(dga, 1e-6, 1e32))[:, None, None] * I3
            Wa = {}
            for o in range(O):
                Wa[(k[o], a[o])] = Wa.get((k[o], a[o]), 0.0) + P[o]
            Tm = np.zeros((C, 3, 3))
            for o in range(O):
                Tm[a[o]] += P[o] @ Vi[k[o]] @ Wa[(k[o], a[o])]
            U[~free] = I3
            Mm = U - np.where(free[:, None, None], Tm, 0.0)
            ok = np.all(np.linalg.eigvalsh(0.5 * (Mm + Mm.transpose(0, 2, 1))) > 0)
        if ok:
            Mi = np.linalg.inv(Mm)
            b = np.zeros((C, 3))
            np.add.at(b, a, -beta + np.einsum("oij,oj->oi", P, q[k]))
            b[~free] = 0.0

            def Sp(p):
                hk = np.zeros((T, 3))
                np.add.at(hk, k, np.einsum("oij,oj->oi", P, p[a]))
                y = np.einsum("kij,kj->ki", Vi, hk)
                Wy = np.zeros((C, 3))
                np.add.at(Wy, a, np.einsum("oij,oj->oi", P, y[k]))
                out = np.einsum("aij,aj->ai", U, p) - Wy
                out[~free] = 0.0
                return out

            x, rr_ = np.zeros((C, 3)), b.copy()
            z = np.einsum("aij,aj->ai", Mi, rr_)
            p = np.zeros((C, 3))
            rr, rz, bta = np.sum(rr_ * rr_), np.sum(rr_ * z), 0.0
            thr = tol * tol * rr
            while cgIt < maxLinear and not rr <= thr:
                p = z + bta * p
                qv = Sp(p)
                pq = np.sum(p * qv)
                if not pq > 0.0:
                    break
                al = rz / pq
                x += al * p
                rr_ -= al * qv
                z = np.einsum("aij,aj->ai", Mi, rr_)
                cgIt += 1
                rr, rzn = np.sum(rr_ * rr_), np.sum(rr_ * z)
                bta, rz = rzn / rz, rzn
            dc = np.where(free[:, None], x, 0.0)
            hk = bX.copy()
            np.add.at(hk, k, np.einsum("oij,oj->oi", P, dc[a]))
            dX = np.einsum("kij,kj->ki", Vi, hk)
            Xc = np.where(part[:, None], X + dX, X)
            cc = c + dc
            sc = np.maximum(s + w2 * (np.sum(d * r, 1) - s * np.sum(d * (dX[k] - dc[a]), 1)) / h, SMIN)
            _, rc = residual(cc, Xc, sc, k, a, v)
            cand = loss(kind, c2, np.sum(rc * rc, 1))[0].sum()
        cgTotal += cgIt
        acc = bool(ok) and cand < cost
        trace.append((cand if ok else np.nan, lam, cgIt, 1.0 if acc else 0.0))
        if acc:
            stop = cost - cand <= 1e-10 * cost
            cost, c, X, s = cand, cc, Xc, sc
            lam /= 10.0
            accepted += 1
            d, r = residual(c, X, s, k, a, v)
            w2 = loss(kind, c2, np.sum(r * r, 1))[1]
            if stop:
                break
        else:
            lam *= 10.0
            if lam > 1e16:
                break
    n = pos.sum()
    rms = np.sqrt(np.sum(c[pos] ** 2) / n) if n else 0.0
    scale = rms if rms > 0.0 and np.isfinite(rms) else 1.0
    t = np.full((C, 3), np.nan)
    for i in np.flatnonzero(pos):
        t[i] = -Rs[i] @ c[i] / scale
    points = np.where(part[:, None], X / scale, np.nan)
    stats = dict(used=O, tracks=int(part.sum()), images=int(n), iterations=len(trace), cg=cgTotal)
    return dict(t=t, points=points, cost=(cost0, cost), trace=np.array(trace).reshape(-1, 4), stats=stats,
                accepted=accepted, c=c, X=X, s=s)


def umeyama(A, B):
    """The similarity (scale, R, t) with scale R A + t ~ B (rows), least squares."""
    ma, mb = A.mean(0), B.mean(0)
    Ac, Bc = A - ma, B - mb
    U, S, Vt = np.linalg.svd(Bc.T @ Ac / len(A))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    R = U @ D @ Vt
    sc = np.trace(np.diag(S) @ D) / np.mean(np.sum(Ac * Ac, 1))
    return sc, R, mb - sc * R @ ma
