"""The float64 statement of cs_absolute_pose_batch (include/cudasift_b200.h): the correspondences, the bearings, the
sampler (verify_oracle's, unchanged), Lambda Twist P3P with every choice the header states (the 3x3 Jacobi restated
line for line), the reprojection inlier rule (triangulate_oracle's), the winner, the Levenberg-Marquardt refinement,
the keep rule and the outputs.

The device contracts products into fused multiply-adds and sums the refinement in a per-lane order, so the two agree
to rounding; the tests keep every inlier decision away from its boundary (the band returned with the results)."""
import math

import numpy as np

import triangulate_oracle as to
import verify_oracle as vo

SLOTS = 4
EPS = 1e-10                     # the degeneracy thresholds (collinear world points, near-parallel bearings)
GN_STEPS = 5                    # Gauss-Newton steps on the depths
LM_ITERS = 20
LM_LAMBDA0 = 1e-3
LM_STEP_TOL = 1e-12
LM_COST_TOL = 1e-12


# ---------------------------------------------------------------------------------------------------- correspondences
def correspondences(xy, pointOf, points):
    """xy: float32 [n, 2] record positions; pointOf int [n]; points float64 [P, 3].  Returns (valid [n], rank order
    positions, world points [V, 3], pixels float32 [V, 2], invalid count)."""
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    pointOf = np.asarray(pointOf, np.int64).reshape(-1)
    points = np.asarray(points, np.float64).reshape(-1, 3)
    P = len(points)
    has = pointOf >= 0
    ok = has & (pointOf < P)
    ok[ok] = np.isfinite(points[pointOf[ok]]).all(1)
    ok &= np.isfinite(xy).all(1)
    pos = np.flatnonzero(ok)
    return ok, pos, points[pointOf[pos]], xy[pos], int((has & ~ok).sum())


def bearings(K, px):
    """normalize(K^-1 (x, y, 1)) in double through vp_calibrate's formula: [V, 3]."""
    x, y = px[:, 0].astype(np.float64), px[:, 1].astype(np.float64)
    cy = (y - K[1, 2]) / K[1, 1]
    cx = (x - K[0, 2] - K[0, 1] * cy) / K[0, 0]
    n = np.sqrt(cx * cx + cy * cy + 1.0)
    return np.stack([cx / n, cy / n, 1.0 / n], 1)


# ---------------------------------------------------------------------------------------------------- P3P
def jacobi3(A):
    """vp_jacobi<3> restated line for line: (the rotated a, whose diagonal holds the eigenvalues, and v)."""
    a = [list(map(float, r)) for r in A]
    N = 3
    v = [[1.0 if p == q else 0.0 for q in range(N)] for p in range(N)]
    tot = 0.0
    for p in range(N):
        for q in range(N):
            tot += a[p][q] * a[p][q]
    for sweep in range(30):
        off = 0.0
        for p in range(N):
            for q in range(p + 1, N):
                off += a[p][q] * a[p][q]
        if not off > 1e-32 * tot:
            break
        for p in range(N):
            for q in range(p + 1, N):
                g = 100.0 * abs(a[p][q])
                if sweep > 2 and abs(a[p][p]) + g == abs(a[p][p]) and abs(a[q][q]) + g == abs(a[q][q]):
                    a[p][q] = a[q][p] = 0.0
                    continue
                if a[p][q] == 0.0:
                    continue
                th = (a[q][q] - a[p][p]) / (2.0 * a[p][q])
                t = (1.0 if th >= 0 else -1.0) / (abs(th) + math.sqrt(th * th + 1.0))
                c = 1.0 / math.sqrt(t * t + 1.0)
                s = t * c
                for k in range(N):
                    kp, kq = a[k][p], a[k][q]
                    a[k][p], a[k][q] = c * kp - s * kq, s * kp + c * kq
                for k in range(N):
                    pk, qk = a[p][k], a[q][k]
                    a[p][k], a[q][k] = c * pk - s * qk, s * pk + c * qk
                for k in range(N):
                    kp, kq = v[k][p], v[k][q]
                    v[k][p], v[k][q] = c * kp - s * kq, s * kp + c * kq
    return a, v


def cubic_root(b, c, d):
    """The largest real root of g^3 + b g^2 + c g + d: the closed form (Cardano when the discriminant is >= 0, else
    the trigonometric form), then two Newton steps, each taken when the derivative is nonzero and the result finite."""
    p = c - b * b / 3.0
    q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d
    disc = 0.25 * q * q + p * p * p / 27.0
    if disc >= 0:
        s = math.sqrt(disc)
        z = np.cbrt(-0.5 * q + s) + np.cbrt(-0.5 * q - s)
    else:
        r = math.sqrt(-p / 3.0)
        z = 2.0 * r * math.cos(math.acos(min(1.0, max(-1.0, -0.5 * q / (r * r * r)))) / 3.0)
    g = float(z) - b / 3.0
    for _ in range(2):
        f = ((g + b) * g + c) * g + d
        fp = (3.0 * g + 2.0 * b) * g + c
        if fp == 0.0:
            break
        g1 = g - f / fp
        if math.isfinite(g1):
            g = g1
    return g


def _dot(u, v):
    return u[0] * v[0] + u[1] * v[1] + u[2] * v[2]


def _cross(u, v):
    return [u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]]


def _sub(u, v):
    return [u[0] - v[0], u[1] - v[1], u[2] - v[2]]


def refine_depths(L, a12, a13, a23, b12, b13, b23):
    """Up to GN_STEPS Newton steps on the three distance equations; a step is kept only when it is finite and lowers
    |r1| + |r2| + |r3|, else the refinement stops."""
    def res(l):
        l1, l2, l3 = l
        return (l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12, l1 * l1 + l3 * l3 + b13 * l1 * l3 - a13,
                l2 * l2 + l3 * l3 + b23 * l2 * l3 - a23)
    for _ in range(GN_STEPS):
        l1, l2, l3 = L
        r1, r2, r3 = res(L)
        e = abs(r1) + abs(r2) + abs(r3)
        if e == 0.0:
            break
        v0, v1 = 2.0 * l1 + b12 * l2, 2.0 * l2 + b12 * l1
        v3, v5 = 2.0 * l1 + b13 * l3, 2.0 * l3 + b13 * l1
        v7, v8 = 2.0 * l2 + b23 * l3, 2.0 * l3 + b23 * l2
        det = -v0 * v5 * v7 - v1 * v3 * v8
        if det == 0.0:
            break
        inv = 1.0 / det
        d1 = (-v5 * v7 * r1 - v1 * v8 * r2 + v1 * v5 * r3) * inv
        d2 = (-v3 * v8 * r1 + v0 * v8 * r2 - v0 * v5 * r3) * inv
        d3 = (v3 * v7 * r1 - v0 * v7 * r2 - v1 * v3 * r3) * inv
        N = (l1 - d1, l2 - d2, l3 - d3)
        if not all(math.isfinite(x) for x in N):
            break
        s1, s2, s3 = res(N)
        if not abs(s1) + abs(s2) + abs(s3) < e:
            break
        L = N
    return L


def p3p(y, X):
    """Lambda Twist on bearings y [3][3] and world points X [3][3] in draw order: (degenerate, [(R [3, 3], t [3])] in
    slot order, at most 4)."""
    y = [list(map(float, r)) for r in y]
    X = [list(map(float, r)) for r in X]
    d12, d13, d23 = _sub(X[0], X[1]), _sub(X[0], X[2]), _sub(X[1], X[2])
    a12, a13, a23 = _dot(d12, d12), _dot(d13, d13), _dot(d23, d23)
    n = _cross(d12, d13)
    if not _dot(n, n) > EPS * a12 * a13:
        return True, []
    c12, c13, c23 = _dot(y[0], y[1]), _dot(y[0], y[2]), _dot(y[1], y[2])
    s12, s13, s23 = 1.0 - c12 * c12, 1.0 - c13 * c13, 1.0 - c23 * c23
    if not (s12 > EPS and s13 > EPS and s23 > EPS):
        return True, []
    b12, b13, b23 = -2.0 * c12, -2.0 * c13, -2.0 * c23
    blob = c12 * c23 * c13 - 1.0
    p3 = a13 * (a23 * s13 - a13 * s23)
    p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23 + a23 * (a23 - a12) * s13
    p1 = a23 * (a13 - a23) * s12 - a12 * a12 * s23 - 2.0 * a12 * (blob * a23 + a13 * s23)
    p0 = a12 * (a12 * s23 - a23 * s12)
    if p3 == 0.0:
        return True, []
    g = cubic_root(p2 / p3, p1 / p3, p0 / p3)
    A = [[a23 * (1.0 - g), 0.5 * a23 * b12, -0.5 * a23 * b13 * g],
         [0.0, a23 - a12 + a13 * g, 0.5 * b23 * (a13 * g - a12)],
         [0.0, 0.0, g * (a13 - a23) - a12]]
    A[1][0], A[2][0], A[2][1] = A[0][1], A[0][2], A[1][2]
    if not all(math.isfinite(x) for r in A for x in r):
        return True, []
    a, V = jacobi3(A)
    order = sorted(range(3), key=lambda i: (-abs(a[i][i]), i))
    e0, e1 = a[order[0]][order[0]], a[order[1]][order[1]]
    if e0 == 0.0:
        return True, []
    u0 = [V[i][order[0]] for i in range(3)]
    u1 = [V[i][order[1]] for i in range(3)]
    v = math.sqrt(max(0.0, -e1 / e0))
    Ls = []
    for s in (v, -v):
        w2 = 1.0 / (s * u1[0] - u0[0])
        w0 = (u0[1] - s * u1[1]) * w2
        w1 = (u0[2] - s * u1[2]) * w2
        qa = 1.0 / ((a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12)
        qb = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * qa
        qc = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * qa
        disc = qb * qb - 4.0 * qc
        if not disc >= 0.0:
            continue
        sq = math.sqrt(disc)
        tau1 = 0.5 * (-qb + sq) if qb < 0 else 0.5 * (-qb - sq)
        tau2 = qc / tau1 if tau1 != 0.0 else 0.0
        for tau in (tau1, tau2):
            if not tau > 0.0:
                continue
            dd = a23 / (tau * (b23 + tau) + 1.0)
            if not dd > 0.0:
                continue
            l2 = math.sqrt(dd)
            l3 = tau * l2
            l1 = w0 * l2 + w1 * l3
            if l1 > 0.0:
                Ls.append((l1, l2, l3))
    poses = []
    # the world frame's inverse: rows (c1 x c2, c2 x c0, c0 x c1) / det for the columns c0 = d12, c1 = d13, c2 = n
    det = _dot(d12, _cross(d13, n))
    inv = [[x / det for x in _cross(d13, n)], [x / det for x in _cross(n, d12)], [x / det for x in _cross(d12, d13)]]
    for L in Ls:
        l1, l2, l3 = refine_depths(L, a12, a13, a23, b12, b13, b23)
        if not (l1 > 0 and l2 > 0 and l3 > 0 and math.isfinite(l1) and math.isfinite(l2) and math.isfinite(l3)):
            continue
        r0 = [l1 * c for c in y[0]]
        r1 = [l2 * c for c in y[1]]
        r2 = [l3 * c for c in y[2]]
        yd1, yd2 = _sub(r0, r1), _sub(r0, r2)
        yd3 = _cross(yd1, yd2)
        R = np.array([[yd1[i] * inv[0][j] + yd2[i] * inv[1][j] + yd3[i] * inv[2][j] for j in range(3)]
                      for i in range(3)])
        t = np.array(r0) - R @ np.array(X[0])
        if np.isfinite(R).all() and np.isfinite(t).all():
            poses.append((R, t))
    return False, poses[:SLOTS]


# ---------------------------------------------------------------------------------------------------- scoring
class _Slots:
    """The shape triangulate_oracle.score reads: one projection matrix per 'member'."""

    def __init__(self, P):
        self.P = P


def camera(K, R, t):
    """P = K [R | t]: [..., 3, 4]."""
    return np.einsum("ij,...jk->...ik", K, np.concatenate([R, t[..., None]], -1))


def inliers(P, Xw, px, thr2, chunk=256):
    """The reprojection inlier rule (triangulate_oracle.score) of every pose P [S, 3, 4] on every correspondence:
    (inlier [S, V], depth [S, V], e2 * depth^2 [S, V])."""
    S, V = len(P), len(Xw)
    inl, d, e = np.zeros((S, V), bool), np.zeros((S, V)), np.zeros((S, V))
    if V == 0:
        return inl, d, e
    x, y = px[:, 0].astype(np.float64)[:, None], px[:, 1].astype(np.float64)[:, None]
    for s0 in range(0, S, chunk):
        s1 = min(S, s0 + chunk)
        i, dd, ee = to.score(_Slots(P[s0:s1]), Xw, np.arange(s1 - s0), x, y, thr2)
        inl[s0:s1], d[s0:s1], e[s0:s1] = np.asarray(i).reshape(V, -1).T, dd.T, np.asarray(ee).reshape(V, -1).T
    return inl, d, e


# ---------------------------------------------------------------------------------------------------- refinement
def _rodrigues(w):
    th2 = float(w @ w)
    th = math.sqrt(th2)
    if th2 == 0.0:
        A, B = 1.0, 0.5
    else:
        A, B = math.sin(th) / th, 2.0 * math.sin(0.5 * th) ** 2 / th2
    W = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    return np.eye(3) + A * W + B * (W @ W)


def lm_terms(K, R, t, Xw, px):
    """At pose (R, t) over the correspondences: (H [6, 6], g [6], cost, every depth > 0)."""
    Xc = Xw @ R.T + t
    z = Xc[:, 2]
    a, b = Xc[:, 0] / z, Xc[:, 1] / z
    r = np.stack([K[0, 0] * a + K[0, 1] * b + K[0, 2] - px[:, 0], K[1, 1] * b + K[1, 2] - px[:, 1]], 1)
    gx = np.stack([K[0, 0] / z, K[0, 1] / z, -(K[0, 0] * a + K[0, 1] * b) / z], 1)
    gy = np.stack([np.zeros_like(z), K[1, 1] / z, -K[1, 1] * b / z], 1)
    J = np.stack([np.concatenate([np.cross(Xc, gx), gx], 1), np.concatenate([np.cross(Xc, gy), gy], 1)], 1)
    J = J.reshape(-1, 6)
    rr = r.reshape(-1)
    return J.T @ J, J.T @ rr, float(rr @ rr), bool((z > 0).all())


def cholesky_solve(M, rhs):
    """M x = rhs by Cholesky; None when a pivot is not > 0 or not finite."""
    n = len(M)
    L = np.zeros((n, n))
    for j in range(n):
        d = M[j, j] - sum(L[j, k] * L[j, k] for k in range(j))
        if not (d > 0 and math.isfinite(d)):
            return None
        L[j, j] = math.sqrt(d)
        for i in range(j + 1, n):
            L[i, j] = (M[i, j] - sum(L[i, k] * L[j, k] for k in range(j))) / L[j, j]
    z = np.zeros(n)
    for i in range(n):
        z[i] = (rhs[i] - sum(L[i, k] * z[k] for k in range(i))) / L[i, i]
    x = np.zeros(n)
    for i in reversed(range(n)):
        x[i] = (z[i] - sum(L[k, i] * x[k] for k in range(i + 1, n))) / L[i, i]
    return x


def refine(K, R, t, Xw, px):
    """Levenberg-Marquardt on the squared pixel error over the given correspondences from (R, t): the update
    R <- exp([w]x) R, t <- exp([w]x) t + delta, the damped system (H + lambda diag(H)) step = -g, lambda from 1e-3,
    x10 on a rejected step and /10 on an accepted one; a step is accepted when every depth stays > 0 and the cost
    decreases.  At most 20 iterations; it stops after an accepted step whose largest |component| is <= 1e-12 or whose
    cost decrease is <= 1e-12 of the cost before it.  Returns (R, t, accepted steps)."""
    H, g, cost, _ = lm_terms(K, R, t, Xw, px)
    lam, acc = LM_LAMBDA0, 0
    for _ in range(LM_ITERS):
        step = cholesky_solve(H + lam * np.diag(np.diag(H)), -g)
        if step is None:
            lam *= 10.0
            continue
        Q = _rodrigues(step[:3])
        R1, t1 = Q @ R, Q @ t + step[3:]
        H1, g1, c1, front = lm_terms(K, R1, t1, Xw, px)
        if front and c1 < cost:
            dec = cost - c1
            stop = np.abs(step).max() <= LM_STEP_TOL or dec <= LM_COST_TOL * cost
            R, t, H, g, cost, lam, acc = R1, t1, H1, g1, c1, lam / 10.0, acc + 1
            if stop:
                break
        else:
            lam *= 10.0
    return R, t, acc


# ---------------------------------------------------------------------------------------------------- the call
class Band:
    """The smallest relative distance of an inlier decision from its boundary (e2 d^2 against maxError^2 d^2)."""

    def __init__(self):
        self.e2 = np.inf

    def add(self, d, e, thr2):
        m = d > 0
        if m.any():
            t = thr2 * d[m] ** 2
            self.e2 = min(self.e2, float(np.min(np.abs(e[m] - t) / t)))


def slot_models(K, Xw, by, numLoops, seed):
    """Every slot's pose: (R [4 numLoops, 3, 3], t [4 numLoops, 3], NaN-filled when empty; non-degenerate samples)."""
    V = len(Xw)
    R = np.full((SLOTS * numLoops, 3, 3), np.nan)
    t = np.full((SLOTS * numLoops, 3), np.nan)
    idx = vo.samples(seed, numLoops, V, 3)
    good = 0
    for s in range(numLoops):
        if idx[s, 0] < 0:
            continue
        deg, poses = p3p(by[idx[s]], Xw[idx[s]])
        good += not deg
        for r, (Rr, tr) in enumerate(poses):
            R[SLOTS * s + r], t[SLOTS * s + r] = Rr, tr
    return R, t, good


def pose_job(xy, pointOf, points, K, numLoops=1024, maxError=4.0, seed=0, band=None):
    """One job.  Returns dict(R, t, count, errors float32 [n], inlier bool [n], stats [8], slotR, slotT, slotCounts)."""
    K = np.asarray(K, np.float64).reshape(3, 3)
    thr2 = float(maxError) * float(maxError)
    band = band if band is not None else Band()
    n = len(np.asarray(xy).reshape(-1, 2))
    ok, pos, Xw, px, invalid = correspondences(xy, pointOf, points)
    V = len(pos)
    errors, inlier = np.full(n, np.nan, np.float32), np.zeros(n, bool)
    stats = np.array([V, invalid, 0, 0, -1, 0, 0, 0], np.int64)
    by = bearings(K, px)
    sR, sT, good = slot_models(K, Xw, by, numLoops, seed)
    live = ~np.isnan(sR[:, 0, 0])
    counts = np.zeros(len(sR), np.int64)
    if live.any() and V:
        inl, d, e = inliers(camera(K, sR[live], sT[live]), Xw, px, thr2)
        band.add(d, e, thr2)
        counts[live] = inl.sum(1)
    stats[2], stats[3] = good, int(live.sum())
    out = dict(R=np.zeros((3, 3)), t=np.zeros(3), count=0, errors=errors, inlier=inlier, stats=stats, slotR=sR,
               slotT=sT, slotCounts=np.where(live, counts, 0), band=band)
    if not live.any():
        return out
    w = int(np.flatnonzero(live)[np.argmax(counts[live])])      # the most inliers, then the lowest slot
    c0 = int(counts[w])
    stats[4], stats[5] = w, c0
    if c0 < 3:
        return out
    inl, _, _ = inliers(camera(K, sR[w][None], sT[w][None]), Xw, px, thr2)
    r = np.flatnonzero(inl[0])
    R1, t1, _ = refine(K, sR[w], sT[w], Xw[r], px[r])
    R, t, count = sR[w], sT[w], c0
    if np.isfinite(R1).all() and np.isfinite(t1).all():
        inl1, d1, e1 = inliers(camera(K, R1[None], t1[None]), Xw, px, thr2)
        band.add(d1, e1, thr2)
        if int(inl1.sum()) >= c0:
            R, t, count = R1, t1, int(inl1.sum())
            stats[6] = 1
    stats[7] = count
    inl, d, e = inliers(camera(K, R[None], t[None]), Xw, px, thr2)
    band.add(d, e, thr2)
    with np.errstate(divide="ignore", invalid="ignore"):
        err = np.where(d[0] > 0, np.sqrt(e[0] / (d[0] * d[0])), np.inf)
    errors[pos] = err.astype(np.float32)
    inlier[pos] = inl[0]
    out.update(R=R, t=t, count=count)
    return out
