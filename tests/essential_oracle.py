"""A float64 numpy restatement of cs_verify_essential (csrc/verify.cu) for the tests: calibrated coordinates, the
sampler of verify_oracle (5 draws), Nister's 5-point solver with the same polynomial construction but its real roots
from np.roots (companion-matrix eigenvalues, an independent root finder), the essential-manifold projection, the
refit, the pose choice and the output conventions.  Scoring is in float64 on pixel Sampson errors, so an inlier
decision may differ from the device's FP32 one only for pairs whose residual lies at the threshold."""
import math

import numpy as np

import verify_oracle as vo

SLOTS = 10
PIVOT = 1e-12
LEAD = 1e-12
PARALLEL = 1e-12
W = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])

# Nister's monomial order: x^3 y^3 x^2y xy^2 x^2z x^2 y^2z y^2 xyz xy | xz^2 xz x yz^2 yz y z^3 z^2 z 1
MONOS = [(3, 0, 0), (0, 3, 0), (2, 1, 0), (1, 2, 0), (2, 0, 1), (2, 0, 0), (0, 2, 1), (0, 2, 0), (1, 1, 1), (1, 1, 0),
         (1, 0, 2), (1, 0, 1), (1, 0, 0), (0, 1, 2), (0, 1, 1), (0, 1, 0), (0, 0, 3), (0, 0, 2), (0, 0, 1), (0, 0, 0)]
INDEX = {m: k for k, m in enumerate(MONOS)}


def calibrate(K, x, y):
    """x^ = K^-1 (x, y, 1) for an upper-triangular K, in the device's operation order."""
    K = np.asarray(K, np.float64).reshape(-1)
    cy = (np.asarray(y, np.float64) - K[5]) / K[4]
    cx = (np.asarray(x, np.float64) - K[2] - K[1] * cy) / K[0]
    return cx, cy


def calibrated(p, K1, K2):
    """[n, 4] pixel pairs -> [n, 4] calibrated (x, y, X, Y)."""
    x, y = calibrate(K1, p[:, 0], p[:, 1])
    X, Y = calibrate(K2, p[:, 2], p[:, 3])
    return np.column_stack([x, y, X, Y])


def unit_sign(M):
    """Unit Frobenius norm, the largest-magnitude entry (the first of equals) positive; None for zero."""
    M = np.asarray(M, np.float64).reshape(3, 3)
    n = np.linalg.norm(M)
    if not n > 0 or not np.isfinite(n):
        return None
    flat = M.reshape(-1)
    return M * (math.copysign(1.0, flat[int(np.argmax(np.abs(flat)))]) / n)


def e_to_f(E, K1, K2):
    K1, K2 = np.asarray(K1, np.float64).reshape(3, 3), np.asarray(K2, np.float64).reshape(3, 3)
    return np.linalg.inv(K2).T @ np.asarray(E, np.float64).reshape(3, 3) @ np.linalg.inv(K1)


def _pmul(p, q):
    """Product of two polynomials given as {exponents: coefficient}."""
    out = {}
    for a, u in p.items():
        for b, v in q.items():
            m = (a[0] + b[0], a[1] + b[1], a[2] + b[2])
            out[m] = out.get(m, 0.0) + u * v
    return out


def _padd(p, q, s=1.0):
    out = dict(p)
    for m, v in q.items():
        out[m] = out.get(m, 0.0) + s * v
    return out


def constraint_matrix(N):
    """The 10 x 20 cubic constraints of E = x N0 + y N1 + z N2 + N3: row 0 det E, row 1 + 3i + j entry (i, j) of
    2 E E^T E - tr(E E^T) E."""
    P = [{(1, 0, 0): N[0][k], (0, 1, 0): N[1][k], (0, 0, 1): N[2][k], (0, 0, 0): N[3][k]} for k in range(9)]
    e = lambda i, j: P[3 * i + j]                                        # noqa: E731
    rows = []
    det = {}
    for c, (a, b), sg in ((0, (1, 2), 1.0), (1, (0, 2), -1.0), (2, (0, 1), 1.0)):
        cof = _padd(_pmul(e(1, a), e(2, b)), _pmul(e(1, b), e(2, a)), -1.0)
        det = _padd(det, _pmul(cof, e(0, c)), sg)
    rows.append(det)
    EEt = [[{} for _ in range(3)] for _ in range(3)]
    for i in range(3):
        for j in range(3):
            for k in range(3):
                EEt[i][j] = _padd(EEt[i][j], _pmul(e(i, k), e(j, k)))
    tr = _padd(_padd(EEt[0][0], EEt[1][1]), EEt[2][2])
    for i in range(3):
        for j in range(3):
            r = {}
            for l in range(3):
                q = {m: 2.0 * v for m, v in EEt[i][l].items()}
                if i == l:
                    q = _padd(q, tr, -1.0)
                r = _padd(r, _pmul(q, e(l, j)))
            rows.append(r)
    C = np.zeros((10, 20))
    for r, poly in enumerate(rows):
        for m, v in poly.items():
            C[r, INDEX[m]] += v
    return C


def gauss_jordan(C):
    """The first ten columns to the identity (partial pivoting, the first of equal magnitudes); None when a pivot is
    at or below PIVOT of the largest |entry|."""
    C = C.copy()
    amax = np.abs(C).max()
    if not amax > 0 or not np.isfinite(amax):
        return None
    for c in range(10):
        p = c + int(np.argmax(np.abs(C[c:, c])))
        if not abs(C[p, c]) > PIVOT * amax:
            return None
        C[[c, p]] = C[[p, c]]
        C[c] /= C[c, c]
        for r in range(10):
            if r != c:
                C[r] -= C[r, c] * C[c]
    return C


def hidden_matrix(G):
    """Rows 4 - z row 5, 6 - z row 7, 8 - z row 9: [q][x, y, 1] polynomials in z (ascending coefficients)."""
    out = []
    for q in range(3):
        a, b = G[4 + 2 * q, 10:], G[5 + 2 * q, 10:]
        px = np.array([a[2], a[1] - b[2], a[0] - b[1], -b[0]])
        py = np.array([a[5], a[4] - b[5], a[3] - b[4], -b[3]])
        p1 = np.array([a[9], a[8] - b[9], a[7] - b[8], a[6] - b[7], -b[6]])
        out.append((px, py, p1))
    return out


def _mul(a, b):
    return np.convolve(a, b)


def _sub(a, b):
    n = max(len(a), len(b))
    return np.pad(a, (0, n - len(a))) - np.pad(b, (0, n - len(b)))


def det_polynomial(B):
    """det of the 3 x 3 polynomial matrix (cofactors along row 0), ascending coefficients of degree 10."""
    (kx, ky, k1), (lx, ly, l1), (mx, my, m1) = B
    d = _mul(kx, _sub(_mul(ly, m1), _mul(l1, my)))
    d = _sub(d, _mul(ky, _sub(_mul(lx, m1), _mul(l1, mx))))
    return d + _mul(k1, _sub(_mul(lx, my), _mul(ly, mx)))


def real_roots(c):
    """The real roots of the ascending polynomial c, ascending: np.roots after dropping leading coefficients at or
    below LEAD of the largest, |imag| <= 1e-9 (1 + |re|), three Newton steps."""
    c = np.asarray(c, np.float64)
    cm = np.abs(c).max()
    if not cm > 0 or not np.isfinite(cm):
        return []
    n = len(c) - 1
    while n > 0 and not abs(c[n]) > LEAD * cm:
        n -= 1
    if n == 0:
        return []
    c = c[:n + 1]
    r = np.roots(c[::-1])
    out = []
    dc = np.polyder(c[::-1])
    for z in r:
        if abs(z.imag) > 1e-9 * (1 + abs(z.real)):
            continue
        x = float(z.real)
        for _ in range(3):
            d = np.polyval(dc, x)
            if d == 0:
                break
            y = x - np.polyval(c[::-1], x) / d
            if not np.isfinite(y):
                break
            x = float(y)
        out.append(x)
    return sorted(out)


def basis(N):
    """Modified Gram-Schmidt of the four null vectors in order, then the fixed orthogonal mix X, Y, Z, W =
    (q0 - q1 + q2 - q3, q0 + q1 - q2 - q3, q0 - q1 - q2 + q3, q0 + q1 + q2 + q3) / 2; None when a vector vanishes."""
    Q = []
    for v in np.asarray(N, np.float64):
        v = v.copy()
        for u in Q:
            v -= (v @ u) * u
        n = math.sqrt(v @ v)
        if not n > 0:
            return None
        Q.append(v / n)
    q0, q1, q2, q3 = Q
    return np.array([q0 - q1 + q2 - q3, q0 + q1 - q2 - q3, q0 - q1 - q2 + q3, q0 + q1 + q2 + q3]) * 0.5


def solve_e5(q):
    """q: [5, 4] calibrated (x, y, X, Y).  The essential matrices of the sample (unit-scaled as the device builds them:
    x X + y Y + z Z + W), in ascending order of z; [] when degenerate."""
    N = vo.nullspace([vo.f_row(*r) for r in q])
    if N is None:
        return []
    N = basis(N)
    if N is None:
        return []
    G = gauss_jordan(constraint_matrix(N))
    if G is None:
        return []
    B = hidden_matrix(G)
    out = []
    for z in real_roots(det_polynomial(B)):
        M = np.array([[np.polyval(p[::-1], z) for p in row] for row in B])
        v = np.zeros(3)
        for a, b in ((0, 1), (0, 2), (1, 2)):
            w = np.cross(M[a], M[b])
            if abs(w[2]) > abs(v[2]):
                v = w
        if v[2] == 0:
            continue
        x, y = v[0] / v[2], v[1] / v[2]
        out.append(x * N[0] + y * N[1] + z * N[2] + N[3])
    return out


def slot_models(p, K1, K2, numLoops, seed):
    """Every slot's E ([10*numLoops, 9] with the output scaling, NaN when empty), the samples and the normalisation."""
    c1, c2, s = vo.normalisation(p)
    smp = vo.samples(seed, numLoops, len(p), 5)
    out = np.full((SLOTS * numLoops, 9), np.nan)
    if not s > 0:
        return out, smp, (c1, c2, s)
    q = calibrated(p, K1, K2)
    for i, row in enumerate(smp):
        if row[0] < 0:
            continue
        r = 0
        for E in solve_e5(q[row]):
            E = unit_sign(E)
            if E is not None:
                out[SLOTS * i + r] = E.reshape(-1)
                r += 1
    return out, smp, (c1, c2, s)


def project(E):
    """The nearest essential matrix U diag(1, 1, 0) V^T and the right-handed U, V (SVD)."""
    U, S, Vt = np.linalg.svd(np.asarray(E, np.float64).reshape(3, 3))
    if not S[1] > 0:
        return None, None, None
    if np.linalg.det(U) < 0:
        U[:, 2] = -U[:, 2]
    if np.linalg.det(Vt) < 0:
        Vt[2] = -Vt[2]
    return U @ np.diag([1.0, 1.0, 0.0]) @ Vt, U, Vt.T


def refit(p, inl, K1, K2, s):
    """The 8-point refit on calibrated coordinates scaled by lambda (not centred), unscaled and projected; None with
    fewer than 8 inliers."""
    if inl.sum() < 8:
        return None
    K1, K2 = np.asarray(K1, np.float64).reshape(-1), np.asarray(K2, np.float64).reshape(-1)
    lam = s * math.sqrt(math.sqrt(K1[0] * K1[4]) * math.sqrt(K2[0] * K2[4]))
    q = calibrated(p[inl], K1, K2) * lam
    A = np.array([vo.f_row(*r) for r in q])
    _, V = np.linalg.eigh(A.T @ A)
    S = np.diag([lam, lam, 1.0])
    Ep, _, _ = project(S @ V[:, 0].reshape(3, 3) @ S)
    return Ep


def in_front(R, t, q):
    """Per calibrated pair: both least-squares depths of l2 x^2 = l1 R x^1 + t positive, the rays not parallel."""
    a = np.column_stack([q[:, 0], q[:, 1], np.ones(len(q))]) @ R.T
    b = np.column_stack([q[:, 2], q[:, 3], np.ones(len(q))])
    aa, bb, ab = (a * a).sum(1), (b * b).sum(1), (a * b).sum(1)
    at, bt = a @ t, b @ t
    ok = aa * bb - ab * ab > PARALLEL * aa * bb
    return ok & (ab * bt - at * bb > 0) & (aa * bt - ab * at > 0)


def pose_candidates(E):
    """(R, t) for (U W V^T, +u3), (U W V^T, -u3), (U W^T V^T, +u3), (U W^T V^T, -u3)."""
    _, U, V = project(E)
    if U is None:
        return []
    Ra, Rb, u3 = U @ W @ V.T, U @ W.T @ V.T, U[:, 2] / np.linalg.norm(U[:, 2])
    return [(Ra, u3), (Ra, -u3), (Rb, u3), (Rb, -u3)]


def choose_pose(E, q):
    """The candidate with the most pairs in front (the first of equals), its count and the runner-up's count."""
    cands = pose_candidates(E)
    if not cands:
        return np.zeros((3, 3)), np.zeros(3), 0, 0
    counts = [int(in_front(R, t, q).sum()) for R, t in cands]
    k = int(np.argmax(counts))
    return cands[k][0], cands[k][1], counts[k], max(c for j, c in enumerate(counts) if j != k)


def residuals(E, K1, K2, p):
    return vo.residuals(e_to_f(E, K1, K2), vo.FUNDAMENTAL, p)


def verify(x1, y1, x2, y2, pairs, n1, n2, K1, K2, numLoops, thresh, seed):
    """The whole call in float64: (E, R, t, inlier pairs in input order, winning slot, its inlier count)."""
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    ok, c = vo.valid_mask(x1, y1, x2, y2, pairs, n1, n2)
    p = c[ok]
    models, _, (c1, c2, s) = slot_models(p, K1, K2, numLoops, seed)
    counts = np.array([(residuals(m, K1, K2, p) < thresh).sum() if np.isfinite(m).all() else -1 for m in models])
    if len(counts) == 0 or (counts < 0).all():
        return np.zeros((3, 3)), np.zeros((3, 3)), np.zeros(3), np.zeros((0, 2), np.int32), -1, 0
    best = int(np.argmax(counts))
    E = models[best].reshape(3, 3)
    inl = residuals(E, K1, K2, p) < thresh
    Er = refit(p, inl, K1, K2, s)
    if Er is not None and (residuals(Er, K1, K2, p) < thresh).sum() >= inl.sum():
        E = Er
    final = residuals(E, K1, K2, p) < thresh
    Ep, _, _ = project(E)
    R, t, _, _ = choose_pose(Ep, calibrated(p[final], K1, K2))
    return unit_sign(Ep), R, t, pairs[ok][final].astype(np.int32), best, int(counts[best])


def same_e(a, b):
    """Relative difference of two essential matrices after the output scaling."""
    a, b = unit_sign(a), unit_sign(b)
    return float(np.linalg.norm(a - b))
