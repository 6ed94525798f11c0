"""A float64 statement of cs_rotation_averaging (include/cudasift_b200.h): the spanning-tree start, the residual and
its log, the Geman-McClure IRLS weights, the Laplacian system and its Jacobi-preconditioned CG, the world-frame update
and the stop rule.  Sums are numpy's, so results agree with the device to rounding, not bit for bit."""
import numpy as np

STOP = 1e-12


def log_rot(D):
    """(rho, theta) of the header's rule: theta = atan2(s, c); rho = v theta / s for c > 0, else theta a from the
    symmetric part, signed so that a.v >= 0."""
    c = 0.5 * (D[0, 0] + D[1, 1] + D[2, 2] - 1.0)
    v = 0.5 * np.array([D[2, 1] - D[1, 2], D[0, 2] - D[2, 0], D[1, 0] - D[0, 1]])
    s = np.sqrt(v @ v)
    th = np.arctan2(s, c)
    if c > 0.0:
        return v * (th / s if s > 0.0 else 1.0), th
    d = np.diag(D)
    k = (2 if d[2] > d[1] else 1) if d[1] > d[0] else (2 if d[2] > d[0] else 0)
    u = 1.0 - c
    a = np.empty(3)
    a[k] = np.sqrt(max(d[k] - c, 0.0) / u)
    for m in range(3):
        if m != k:
            a[m] = 0.5 * (D[k, m] + D[m, k]) / (u * a[k])
    return (-th if a @ v < 0.0 else th) * a, th


def skew(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def exp_rot(w):
    """The Rodrigues rotation of vp_rodrigues."""
    th2 = float(w @ w)
    A, B = 1.0, 0.5
    if th2 != 0.0:
        th = np.sqrt(th2)
        A, B = np.sin(th) / th, 2.0 * np.sin(0.5 * th) ** 2 / th2
    W = skew(w)
    return np.eye(3) + A * W + B * (W @ W)


def jr_inv(rho):
    """The inverse right Jacobian of SO(3); the inverse left one is jr_inv(-rho)."""
    th = np.linalg.norm(rho)
    W = skew(rho)
    if th < 1e-8:
        return np.eye(3) + 0.5 * W + W @ W / 12.0
    return np.eye(3) + 0.5 * W + (1.0 / th ** 2 - (1.0 + np.cos(th)) / (2.0 * th * np.sin(th))) * (W @ W)


def spanning_tree(numImages, edges, Rrel, weights, ref):
    """Kruskal's maximum spanning tree (weight descending, ties to the lower edge index) and the breadth-first walk from
    ref.  Returns (R [N, 3, 3] with NaN for an image not reached, reached bool [N])."""
    edges = np.asarray(edges).reshape(-1, 2)
    parent = list(range(numImages))

    def root(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    tree = []
    for e in np.argsort(-np.asarray(weights, np.float64), kind="stable"):
        a, b = root(int(edges[e, 0])), root(int(edges[e, 1]))
        if a != b:
            parent[b] = a
            tree.append(int(e))
    adj = [[] for _ in range(numImages)]
    for e in sorted(tree):
        adj[edges[e, 0]].append(e)
        adj[edges[e, 1]].append(e)
    R = np.full((numImages, 3, 3), np.nan)
    reached = np.zeros(numImages, bool)
    R[ref], reached[ref] = np.eye(3), True
    queue = [ref]
    for a in queue:
        for e in adj[a]:
            i, j = int(edges[e, 0]), int(edges[e, 1])
            o = j if i == a else i
            if reached[o]:
                continue
            R[o] = Rrel[e] @ R[a] if o == j else Rrel[e].T @ R[a]
            reached[o] = True
            queue.append(o)
    return R, reached


def residuals(R, edges, Rrel, active):
    """rho [E, 3] and theta [E] (NaN for an inactive edge) of D_e = R_j^T Q_e R_i."""
    E = len(edges)
    rho, th = np.zeros((E, 3)), np.full(E, np.nan)
    for e in np.flatnonzero(active):
        i, j = edges[e]
        rho[e], th[e] = log_rot(R[j].T @ (Rrel[e] @ R[i]))
    return rho, th


def loss(theta, w0, sigma):
    """(cost terms, IRLS weights) of the header's loss; sigma in radians (0: squared)."""
    t2 = theta * theta
    q = sigma * sigma / (t2 + sigma * sigma) if sigma > 0.0 else np.ones_like(t2)
    return w0 * t2 * q, w0 * q * q


def laplacian(numImages, edges, w):
    """The weighted adjacency W (symmetric, dense) and diag(L)."""
    W = np.zeros((numImages, numImages))
    np.add.at(W, (edges[:, 0], edges[:, 1]), w)
    np.add.at(W, (edges[:, 1], edges[:, 0]), w)
    return W, W.sum(1)


def rhs(numImages, edges, w, rho, free):
    b = np.zeros((numImages, 3))
    np.add.at(b, edges[:, 0], -w[:, None] * rho)
    np.add.at(b, edges[:, 1], w[:, None] * rho)
    b[~free] = 0.0
    return b


def cg(W, diag, b, free, maxLinear, tol):
    """Jacobi-preconditioned CG on L x = b from x = 0 (held rows identity, b 0): the header's stop rules.  Returns
    (x [N, 3], iterations)."""
    inv = np.where(free & (diag > 0), 1.0 / np.where(diag > 0, diag, 1.0), 0.0)[:, None]
    x, r = np.zeros_like(b), b.copy()
    z = r * inv
    p = np.zeros_like(b)
    rr, rz, beta = np.sum(r * r), np.sum(r * z), 0.0
    thr = tol * tol * rr
    it = 0
    while it < maxLinear and not rr <= thr:
        p = z + beta * p
        q = np.where(free[:, None], diag[:, None] * p - W @ p, 0.0)
        pq = np.sum(p * q)
        if not pq > 0.0:
            break
        alpha = rz / pq
        x += alpha * p
        r -= alpha * q
        z = r * inv
        it += 1
        rr, rzn = np.sum(r * r), np.sum(r * z)
        beta, rz = rzn / rz, rzn
    return x, it


def average(numImages, edges, Rrel, weights, ref=0, maxIterations=50, maxLinear=200, tol=1e-8, sigmaDeg=5.0,
            maxAngleDeg=5.0):
    """The call's outputs: dict(R, residuals (degrees), inlier, cost (start, final), trace [iterations, 3], stats)."""
    edges = np.asarray(edges, np.int64).reshape(-1, 2)
    Rrel = np.asarray(Rrel, np.float64).reshape(-1, 3, 3)
    w0 = np.asarray(weights, np.float64).reshape(-1)
    sigma = sigmaDeg * np.pi / 180.0
    R, reached = spanning_tree(numImages, edges, Rrel, w0, ref)
    free = reached.copy()
    free[ref] = False
    active = reached[edges[:, 0]] if len(edges) else np.zeros(0, bool)
    rho, th = residuals(R, edges, Rrel, active)
    terms, w = loss(np.where(active, th, 0.0), np.where(active, w0, 0.0), sigma)
    cost0 = cost = terms.sum()
    trace, cgTotal = [], 0
    for it in range(maxIterations):
        W, diag = laplacian(numImages, edges, w)
        x, k = cg(W, diag, rhs(numImages, edges, w, rho, free), free, maxLinear, tol)
        cgTotal += k
        step = max((np.linalg.norm(x[a]) for a in np.flatnonzero(free)), default=0.0)
        for a in np.flatnonzero(free):
            R[a] = exp_rot(R[a] @ x[a]) @ R[a]
        trace.append((cost, k, step))
        rho, th = residuals(R, edges, Rrel, active)
        terms, w = loss(np.where(active, th, 0.0), np.where(active, w0, 0.0), sigma)
        cost = terms.sum()
        if step <= STOP:
            break
    deg = np.degrees(th)
    inlier = np.nan_to_num(deg, nan=np.inf) < maxAngleDeg
    stats = np.array([active.sum(), reached.sum() - 1, reached.sum(), len(trace), cgTotal, inlier.sum()], np.int64)
    return dict(R=R, residuals=deg, inlier=inlier, cost=(cost0, cost), trace=np.array(trace).reshape(-1, 3),
                stats=stats)


def align(R, Rtrue):
    """The world rotation S (R_a ~ Rtrue_a S) that best aligns the finite R to Rtrue (the chordal mean), and every
    image's angle to Rtrue_a S in degrees (NaN where R is NaN)."""
    ok = np.isfinite(R).all(axis=(1, 2))
    M = np.einsum("aji,ajk->ik", Rtrue[ok], R[ok])
    U, _, Vt = np.linalg.svd(M)
    S = U @ np.diag([1.0, 1.0, np.linalg.det(U @ Vt)]) @ Vt
    err = np.full(len(R), np.nan)
    for a in np.flatnonzero(ok):
        err[a] = np.degrees(log_rot(R[a] @ (Rtrue[a] @ S).T)[1])
    return S, err
