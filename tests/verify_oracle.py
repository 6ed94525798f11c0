"""A float64 numpy restatement of cs_verify_pairs (csrc/verify.cu) for the tests: the counter-based sampler (bit-exact,
uint64 arithmetic), the normalisation, the 4-point and 7-point minimal solvers, the pixel residuals, the refit and the
output order.  Scoring here is in float64, so an inlier decision may differ from the device's FP32 one only for pairs
whose residual lies at the threshold."""
import math

import numpy as np

GOLDEN = np.uint64(0x9E3779B97F4A7C15)
EPS = 1e-9
MAX_DRAWS = 64
HOMOGRAPHY, FUNDAMENTAL = 1, 2


def splitmix64(z):
    """One splitmix64 step from state z (uint64 array)."""
    with np.errstate(over="ignore"):
        z = z + GOLDEN
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draw(seed, s, d, n):
    """Index of draw d of sample s among n valid pairs (arrays broadcast)."""
    s, d = np.asarray(s, np.uint64), np.asarray(d, np.uint64)
    with np.errstate(over="ignore"):
        x = splitmix64(np.uint64(seed) + GOLDEN * ((s << np.uint64(8)) | d))
    return (((x >> np.uint64(32)) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def samples(seed, numLoops, n, k):
    """[numLoops, k] distinct indices per sample, in draw order; a row of -1 for a degenerate sample (64 draws)."""
    raw = draw(seed, np.arange(numLoops)[:, None], np.arange(MAX_DRAWS)[None, :], max(n, 0))
    out = np.full((numLoops, k), -1, np.int64)
    if n < k:
        return out
    for s in range(numLoops):
        got = []
        for v in raw[s]:
            if v not in got:
                got.append(int(v))
                if len(got) == k:
                    out[s] = got
                    break
    return out


def valid_mask(x1, y1, x2, y2, pairs, n1, n2):
    """Valid pairs and their four pixel coordinates (float32 records -> float64)."""
    i, j = pairs[:, 0].astype(np.int64), pairs[:, 1].astype(np.int64)
    ok = (i >= 0) & (i < n1) & (j >= 0) & (j < n2)
    ii, jj = np.where(ok, i, 0), np.where(ok, j, 0)
    c = np.stack([x1[ii], y1[ii], x2[jj], y2[jj]], 1).astype(np.float64) if len(pairs) else np.zeros((0, 4))
    ok &= np.isfinite(c).all(1)
    return ok, c


def normalisation(p):
    """Centroids c1, c2 and the common scale s (mean distance sqrt(2) over both images); p is [n, 4] pixels."""
    n = len(p)
    if n == 0:
        return np.zeros(2), np.zeros(2), 0.0
    c1, c2 = p[:, :2].mean(0), p[:, 2:].mean(0)
    mean = (np.hypot(*(p[:, :2] - c1).T).sum() + np.hypot(*(p[:, 2:] - c2).T).sum()) / (2.0 * n)
    return c1, c2, (math.sqrt(2.0) / mean if mean > 0 else 0.0)


def nullspace(A):
    """Gaussian elimination with partial pivoting on columns 0..m-1, back substitution for each free column (x_f = 1).
    None when a pivot falls below EPS."""
    A = [list(map(float, r)) for r in A]
    m = len(A)
    for c in range(m):
        p, best = c, abs(A[c][c])
        for r in range(c + 1, m):
            if abs(A[r][c]) > best:
                p, best = r, abs(A[r][c])
        if not best >= EPS:
            return None
        A[c], A[p] = A[p], A[c]
        for r in range(c + 1, m):
            f = A[r][c] / A[c][c]
            for j in range(c, 9):
                A[r][j] -= f * A[c][j]
    out = []
    for f in range(m, 9):
        x = [0.0] * 9
        x[f] = 1.0
        for r in range(m - 1, -1, -1):
            x[r] = -sum(A[r][j] * x[j] for j in range(r + 1, 9)) / A[r][r]
        out.append(x)
    return np.array(out)


def h_rows(x, y, X, Y):
    return [[x, y, 1, 0, 0, 0, -X * x, -X * y, -X], [0, 0, 0, x, y, 1, -Y * x, -Y * y, -Y]]


def f_row(x, y, X, Y):
    return [X * x, X * y, X, Y * x, Y * y, Y, x, y, 1]


def _cross(a, b, c):
    return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])


def solve_h4(u):
    """u: [4, 4] normalised (x, y, X, Y).  The unit-norm H or None (three collinear points in an image, small pivot)."""
    for t in ((0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3)):
        for im in (0, 2):
            if not abs(_cross(u[t[0], im:im + 2], u[t[1], im:im + 2], u[t[2], im:im + 2])) >= EPS:
                return None
    N = nullspace([r for q in u for r in h_rows(*q)])
    if N is None:
        return None
    return N[0] / np.linalg.norm(N[0])


def det3(m):
    """The cofactor expansion the device uses."""
    return (m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) +
            m[2] * (m[3] * m[7] - m[4] * m[6]))


def cubic_roots(c):
    """Real roots of c0 + c1 a + c2 a^2 + c3 a^3 in closed form (unpolished, in the device's order)."""
    cm = max(abs(v) for v in c)
    if not cm > 0:
        return []
    roots = []
    if abs(c[3]) > 1e-10 * cm:
        a, b, d = c[2] / c[3], c[1] / c[3], c[0] / c[3]
        p = b - a * a / 3.0
        q = 2.0 * a * a * a / 27.0 - a * b / 3.0 + d
        disc = 0.25 * q * q + p * p * p / 27.0
        if disc > 0:
            sq = math.sqrt(disc)
            roots.append(np.cbrt(-0.5 * q + sq) + np.cbrt(-0.5 * q - sq) - a / 3.0)
        elif p == 0:
            roots.append(-a / 3.0)
        else:
            r = math.sqrt(-p / 3.0)
            phi = math.acos(min(1.0, max(-1.0, 1.5 * q / p * math.sqrt(-3.0 / p))))
            roots += [2.0 * r * math.cos(phi / 3.0 - 2.0 * math.pi * k / 3.0) - a / 3.0 for k in range(3)]
    elif abs(c[2]) > 1e-10 * cm:
        disc = c[1] * c[1] - 4.0 * c[2] * c[0]
        if disc >= 0:
            qq = -0.5 * (c[1] + math.copysign(1.0, c[1]) * math.sqrt(disc))
            roots.append(qq / c[2])
            if qq != 0:
                roots.append(c[0] / qq)
    elif abs(c[1]) > 1e-10 * cm:
        roots.append(-c[0] / c[1])
    return [float(r) for r in roots]


def solve_f7(u):
    """u: [7, 4] normalised.  Up to three unit-norm F in ascending order of the pencil parameter, or [] (degenerate).
    det(a F1 + (1 - a) F2) is interpolated as a cubic from a = 0, 1, -1, 2; each closed-form root takes two Newton steps
    on the determinant itself."""
    N = nullspace([f_row(*q) for q in u])
    if N is None:
        return []
    F1, F2 = N
    D = F1 - F2
    p = [det3(F2 + a * D) for a in (0.0, 1.0, -1.0, 2.0)]
    c2 = 0.5 * (p[1] + p[2]) - p[0]
    a, b = 0.5 * (p[1] - p[2]), p[3] - p[0] - 4.0 * c2
    c3 = (b - 2.0 * a) / 6.0
    c = [p[0], a - c3, c2, c3]
    roots = []
    for x in cubic_roots(c):
        for _ in range(2):
            d = (3.0 * c[3] * x + 2.0 * c[2]) * x + c[1]
            if d == 0:
                break
            y = x - det3(F2 + x * D) / d
            if math.isfinite(y):
                x = y
        roots.append(x)
    out = []
    for r in sorted(roots):
        F = r * F1 + (1.0 - r) * F2
        nrm = np.linalg.norm(F)
        if nrm > 0 and np.isfinite(nrm):
            out.append(F / nrm)
    return out


def denormalise(m, model, c1, c2, s):
    """Normalised-coordinate model -> pixels, with the output scaling of cs_verify_pairs."""
    T1 = np.array([[s, 0, -s * c1[0]], [0, s, -s * c1[1]], [0, 0, 1]])
    if model == HOMOGRAPHY:
        L = np.array([[1 / s, 0, c2[0]], [0, 1 / s, c2[1]], [0, 0, 1]])
    else:
        L = np.array([[s, 0, -s * c2[0]], [0, s, -s * c2[1]], [0, 0, 1]]).T
    out = L @ np.asarray(m, np.float64).reshape(3, 3) @ T1
    return scale_model(out, model)


def scale_model(M, model):
    M = np.asarray(M, np.float64).reshape(3, 3).copy()
    if model == HOMOGRAPHY:
        return M / M[2, 2] if M[2, 2] != 0 else M
    flat = M.reshape(-1)
    big = int(np.argmax(np.abs(flat)))
    return M * (math.copysign(1.0, flat[big]) / np.linalg.norm(M))


def residuals(M, model, p):
    """Pixel residuals of [n, 4] pairs: transfer error for H, sqrt of the Sampson error for F."""
    x1 = np.column_stack([p[:, 0], p[:, 1], np.ones(len(p))])
    x2 = np.column_stack([p[:, 2], p[:, 3], np.ones(len(p))])
    M = np.asarray(M, np.float64).reshape(3, 3)
    with np.errstate(all="ignore"):
        if model == HOMOGRAPHY:
            q = x1 @ M.T
            return np.hypot(q[:, 0] / q[:, 2] - p[:, 2], q[:, 1] / q[:, 2] - p[:, 3])
        Fx1, Ftx2 = x1 @ M.T, x2 @ M
        num = (x2 * Fx1).sum(1)
        den = Fx1[:, 0] ** 2 + Fx1[:, 1] ** 2 + Ftx2[:, 0] ** 2 + Ftx2[:, 1] ** 2
        return np.sqrt(num * num / den)


def slot_models(p, model, numLoops, seed):
    """Every slot's pixel model ([3*numLoops, 9], NaN when empty), the samples and the normalisation."""
    k = 4 if model == HOMOGRAPHY else 7
    c1, c2, s = normalisation(p)
    smp = samples(seed, numLoops, len(p), k)
    out = np.full((3 * numLoops, 9), np.nan)
    if not s > 0:
        return out, smp, (c1, c2, s)
    u = np.column_stack([(p[:, 0] - c1[0]) * s, (p[:, 1] - c1[1]) * s, (p[:, 2] - c2[0]) * s, (p[:, 3] - c2[1]) * s])
    for i, row in enumerate(smp):
        if row[0] < 0:
            continue
        ms = [solve_h4(u[row])] if model == HOMOGRAPHY else solve_f7(u[row])
        ms = [m for m in ms if m is not None]
        for r, m in enumerate(ms):
            out[3 * i + r] = denormalise(m, model, c1, c2, s).reshape(-1)
    return out, smp, (c1, c2, s)


def refit(p, model, inl, c1, c2, s):
    """One least-squares refit over the inliers: the smallest eigenvector of the normal matrix (8-point for F with rank
    2 enforced, DLT for H) in normalised coordinates, returned in pixels; None with too few inliers."""
    if inl.sum() < (4 if model == HOMOGRAPHY else 8):
        return None
    q = p[inl]
    u = np.column_stack([(q[:, 0] - c1[0]) * s, (q[:, 1] - c1[1]) * s, (q[:, 2] - c2[0]) * s, (q[:, 3] - c2[1]) * s])
    A = np.array([r for v in u for r in h_rows(*v)]) if model == HOMOGRAPHY else np.array([f_row(*v) for v in u])
    w, V = np.linalg.eigh(A.T @ A)
    f = V[:, 0]
    if model == FUNDAMENTAL:
        U, S, Vt = np.linalg.svd(f.reshape(3, 3))
        f = (U @ np.diag([S[0], S[1], 0.0]) @ Vt).reshape(-1)
    return denormalise(f, model, c1, c2, s)


def verify(x1, y1, x2, y2, pairs, n1, n2, model, numLoops, thresh, seed):
    """The whole call in float64: (model 3x3, inlier pairs in input order, winning slot, minimal inlier count)."""
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    ok, c = valid_mask(x1, y1, x2, y2, pairs, n1, n2)
    p = c[ok]
    models, _, (c1, c2, s) = slot_models(p, model, numLoops, seed)
    counts = np.array([(residuals(m, model, p) < thresh).sum() if np.isfinite(m).all() else -1 for m in models])
    if (counts < 0).all():
        return np.zeros((3, 3)), np.zeros((0, 2), np.int32), -1, 0
    best = int(np.argmax(counts))                 # the first of the largest: the lowest slot wins ties
    M = models[best].reshape(3, 3)
    inl = residuals(M, model, p) < thresh
    R = refit(p, model, inl, c1, c2, s)
    if R is not None and (residuals(R, model, p) < thresh).sum() >= inl.sum():
        M = R
    final = residuals(M, model, p) < thresh
    return M, pairs[ok][final].astype(np.int32), best, int(counts[best])


def same_model(a, b, model):
    """Relative difference of two models after the output scaling (and, for F, the sign)."""
    a, b = scale_model(a, model), scale_model(b, model)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))
