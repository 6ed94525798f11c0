"""The float64 statement of cs_triangulate_tracks (include/cudasift_b200.h): validity, the hypotheses (enumeration and
the counter-based sampler), the two-view DLT solved by a line-for-line restatement of vp_jacobi<4>, admissibility,
inliers, the winner, the refit and its keep rule, and the outputs.  The Jacobi runs vectorised over all hypotheses of
all tracks at once (every matrix follows its own sweeps through masks); the rest runs per track, vectorised over its
hypotheses and members.

The device contracts products into fused multiply-adds and sums the refit in a per-lane order, so the two agree to
rounding: the case generators keep every decision away from its boundary (Band)."""
import math

import numpy as np

GOLDEN = 0x9E3779B97F4A7C15
DRAWS = 16


def splitmix64(z):
    z = np.asarray(z, np.uint64)
    with np.errstate(over="ignore"):
        z = z + np.uint64(GOLDEN)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draw(seed, k, s, V):
    """The ranks (p, q) of samples s of track k among V valid members, and whether each sample has two distinct ranks
    within 16 draws."""
    s = np.asarray(s, np.uint64)
    p, q, got = np.zeros(len(s), np.int64), np.zeros(len(s), np.int64), np.zeros(len(s), np.int64)
    for d in range(DRAWS):
        with np.errstate(over="ignore"):
            x = splitmix64(np.uint64(seed) + np.uint64(GOLDEN) * ((np.uint64(k) << np.uint64(24)) | (s << np.uint64(4)) |
                                                                  np.uint64(d)))
        i = (((x >> np.uint64(32)) * np.uint64(V)) >> np.uint64(32)).astype(np.int64)
        g0, g1 = got == 0, got == 1
        p[g0] = i[g0]
        got[g0] = 1
        second = g1 & (i != p)
        q[second] = i[second]
        got[second] = 2
    return p, q, got == 2


def jacobi4(A):
    """vp_jacobi<4> over a stack of symmetric matrices [B, 4, 4]: (the rotated a, whose diagonal holds the
    eigenvalues, and v, whose columns are the eigenvectors)."""
    a = np.array(A, np.float64).reshape(-1, 4, 4)
    B = len(a)
    v = np.broadcast_to(np.eye(4), a.shape).copy()
    tot = np.zeros(B)
    for p in range(4):
        for q in range(4):
            tot = tot + a[:, p, q] * a[:, p, q]
    live = np.ones(B, bool)
    for sweep in range(30):
        off = np.zeros(B)
        for p in range(4):
            for q in range(p + 1, 4):
                off = off + a[:, p, q] * a[:, p, q]
        live &= off > 1e-32 * tot
        if not live.any():
            break
        for p in range(4):
            for q in range(p + 1, 4):
                g = 100.0 * np.abs(a[:, p, q])
                app, aqq = np.abs(a[:, p, p]), np.abs(a[:, q, q])
                zero = live & (sweep > 2) & (app + g == app) & (aqq + g == aqq)
                a[zero, p, q] = 0.0
                a[zero, q, p] = 0.0
                idx = np.flatnonzero(live & ~zero & (a[:, p, q] != 0.0))
                if not len(idx):
                    continue
                sub, vs = a[idx], v[idx]
                th = (sub[:, q, q] - sub[:, p, p]) / (2.0 * sub[:, p, q])
                t = np.where(th >= 0, 1.0, -1.0) / (np.abs(th) + np.sqrt(th * th + 1.0))
                c = (1.0 / np.sqrt(t * t + 1.0))[:, None]
                s = t[:, None] * c
                kp, kq = sub[:, :, p].copy(), sub[:, :, q].copy()
                sub[:, :, p], sub[:, :, q] = c * kp - s * kq, s * kp + c * kq
                pk, qk = sub[:, p, :].copy(), sub[:, q, :].copy()
                sub[:, p, :], sub[:, q, :] = c * pk - s * qk, s * pk + c * qk
                kp, kq = vs[:, :, p].copy(), vs[:, :, q].copy()
                vs[:, :, p], vs[:, :, q] = c * kp - s * kq, s * kp + c * kq
                a[idx], v[idx] = sub, vs
    return a, v


def solve(S):
    """The normal matrices' ten sums [B, 10] (00 01 02 03 11 12 13 22 23 33) -> (points [B, 3], finite [B]): the
    eigenvector of the smallest eigenvalue (the lowest index on ties), dehomogenised."""
    S = np.asarray(S, np.float64).reshape(-1, 10)
    ij = [(0, 0, 0), (0, 1, 1), (0, 2, 2), (0, 3, 3), (1, 1, 4), (1, 2, 5), (1, 3, 6), (2, 2, 7), (2, 3, 8), (3, 3, 9)]
    A = np.zeros((len(S), 4, 4))
    for i, j, k in ij:
        A[:, i, j] = A[:, j, i] = S[:, k]
    a, v = jacobi4(A)
    best, h = a[:, 0, 0].copy(), v[:, :, 0].copy()
    for j in range(1, 4):
        m = a[:, j, j] < best
        best[m] = a[m, j, j]
        h[m] = v[m, :, j]
    w = h[:, 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        X = h[:, :3] / w[:, None]
    return X, (w != 0) & np.isfinite(X).all(1)


class Cameras:
    """K, R, t per image and what the rules derive from them: P = K [R | t], the centre C = -R^T t."""

    def __init__(self, Ks, Rs, ts):
        self.K = np.asarray(Ks, np.float64).reshape(-1, 3, 3)
        self.R = np.asarray(Rs, np.float64).reshape(-1, 3, 3)
        self.t = np.asarray(ts, np.float64).reshape(-1, 3)
        self.Rt = np.concatenate([self.R, self.t[:, :, None]], 2)
        self.P = self.K @ self.Rt
        self.C = -np.einsum("aji,aj->ai", self.R, self.t)


def calibrate(K, x, y):
    """cs_verify_essential's calibrated coordinates, K [n, 3, 3] per point."""
    cy = (y - K[:, 1, 2]) / K[:, 1, 1]
    cx = (x - K[:, 0, 2] - K[:, 0, 1] * cy) / K[:, 0, 0]
    return cx, cy


def dlt_rows(cams, a, x, y):
    """The two DLT rows x^ P[2] - P[0], y^ P[2] - P[1] of each observation: [n, 2, 4]."""
    Rt = cams.Rt[a]
    cx, cy = calibrate(cams.K[a], np.asarray(x, np.float64), np.asarray(y, np.float64))
    return np.stack([cx[:, None] * Rt[:, 2] - Rt[:, 0], cy[:, None] * Rt[:, 2] - Rt[:, 1]], 1)


IJ = [(i, j) for i in range(4) for j in range(i, 4)]


def sums(rows):
    """The ten normal-matrix sums of rows [..., m, 4], added in row order."""
    out = np.zeros(rows.shape[:-2] + (10,))
    for r in range(rows.shape[-2]):
        for k, (i, j) in enumerate(IJ):
            out[..., k] = out[..., k] + rows[..., r, i] * rows[..., r, j]
    return out


def score(cams, X, a, x, y, thr2):
    """Per point X [H, 3] and member (a, x, y) [V]: (inlier [H, V], depth [H, V], e2 * depth^2 [H, V])."""
    P = cams.P[a]                                                       # [V, 3, 4]
    u = np.einsum("vij,hj->hvi", P[:, :, :3], X) + P[None, :, :, 3]     # [H, V, 3]
    d = u[..., 2]
    e = (u[..., 0] - x[None] * d) ** 2 + (u[..., 1] - y[None] * d) ** 2
    return (d > 0) & (e < thr2 * (d * d)), d, e


class Band:
    """The smallest distances of the decisions from their boundaries: e2 from maxError^2 (relative), the hypotheses'
    depths (relative to the distance from the camera) and cosines from cosMin."""

    def __init__(self):
        self.e2 = self.depth = self.angle = np.inf

    def add_scores(self, d, e, thr2):
        m = d > 0
        if m.any():
            t = thr2 * d[m] ** 2
            self.e2 = min(self.e2, float(np.min(np.abs(e[m] - t) / t)))


def triangulate(xy, Ks, Rs, ts, offsets, members, numTrials=256, maxError=4.0, minTriAngle=1.5, seed=0, tracks=None):
    """xy[a]: image a's record positions, float32 [n, 2].  tracks: the track indices to state (all by default).
    Returns dict(points [len(tracks), 3], counts, errors [M] and inlier [M] (written for the members of the stated
    tracks; NaN and 0 elsewhere), stats [8] over the stated tracks, band)."""
    cams = Cameras(Ks, Rs, ts)
    S = len(xy)
    offsets = np.asarray(offsets, np.int64)
    members = np.asarray(members, np.int64).reshape(-1, 2)
    M = len(members)
    T = len(offsets) - 1
    tracks = np.arange(T) if tracks is None else np.asarray(tracks, np.int64)
    thr2 = float(maxError) * float(maxError)
    cosMin = math.cos(float(minTriAngle) * (math.pi / 180.0))
    points = np.full((len(tracks), 3), np.nan)
    counts = np.zeros(len(tracks), np.int32)
    errors = np.full(M, np.nan, np.float32)
    inlier = np.zeros(M, bool)
    stats = np.zeros(8, np.int64)
    band = Band()

    # per track: the valid members and the hypotheses that pass the image test; their normal matrices
    work, mats = [], []
    for j, k in enumerate(tracks):
        lo, hi = int(offsets[k]), int(offsets[k + 1])
        if lo < 0 or hi < lo or hi > M:
            stats[1] += 1
            continue
        stats[0] += 1
        pos = np.arange(lo, hi)
        a, f = members[lo:hi, 0], members[lo:hi, 1]
        ok = (a >= 0) & (a < S)
        n = np.array([len(xy[q]) for q in a[ok]], np.int64)
        ok[ok] = (f[ok] >= 0) & (f[ok] < n)
        px = np.array([xy[q][g] for q, g in zip(a[ok], f[ok])], np.float32).reshape(-1, 2)
        fin = np.isfinite(px).all(1)
        ok[ok] = fin
        px = px[fin].astype(np.float64)
        stats[2] += int((~ok).sum())
        errors[pos[~ok]] = np.nan
        inlier[pos[~ok]] = False
        pos, a = pos[ok], a[ok]
        V = len(pos)
        if V < 2:
            hp = hq = hh = np.zeros(0, np.int64)
        elif V * (V - 1) // 2 <= numTrials:
            hp, hq = np.triu_indices(V, 1)
            hh = np.arange(len(hp))
        else:
            hp, hq, good = draw(seed, int(k), np.arange(numTrials), V)
            hh = np.flatnonzero(good)
            hp, hq = hp[good], hq[good]
        stats[3] += len(hh)
        diff = a[hp] != a[hq]
        hp, hq, hh = hp[diff], hq[diff], hh[diff]
        if len(hh):
            rows = np.concatenate([dlt_rows(cams, a[hp], px[hp, 0], px[hp, 1]),
                                   dlt_rows(cams, a[hq], px[hq, 0], px[hq, 1])], 1)
            mats.append(sums(rows))
        work.append((j, pos, a, px, hp, hq, hh, sum(len(m) for m in mats) - len(hh)))
    X_all, ok_all = solve(np.concatenate(mats)) if mats else (np.zeros((0, 3)), np.zeros(0, bool))

    # per track: admissibility, counts, the winner and its refit's normal matrix
    refits = []
    for wi, (j, pos, a, px, hp, hq, hh, at) in enumerate(work):
        X, fine = X_all[at:at + len(hh)], ok_all[at:at + len(hh)]
        dp = np.einsum("hj,hj->h", cams.Rt[a[hp], 2, :3], X) + cams.Rt[a[hp], 2, 3]
        dq = np.einsum("hj,hj->h", cams.Rt[a[hq], 2, :3], X) + cams.Rt[a[hq], 2, 3]
        adm = fine & (dp > 0) & (dq > 0)
        if fine.any():
            for d, q in ((dp, hp), (dq, hq)):
                dist = np.linalg.norm(X[fine] - cams.C[a[q[fine]]], axis=1)
                band.depth = min(band.depth, float(np.min(np.abs(d[fine]) / dist)))
        A, B = X - cams.C[a[hp]], X - cams.C[a[hq]]
        ab, aa, bb = (A * B).sum(1), (A * A).sum(1), (B * B).sum(1)
        if adm.any():
            band.angle = min(band.angle, float(np.min(np.abs(ab[adm] / np.sqrt(aa[adm] * bb[adm]) - cosMin))))
        adm &= ab <= cosMin * np.sqrt(aa * bb)
        stats[4] += int(adm.sum())
        winner = None
        if adm.any():
            Xa = X[adm]
            cnt = np.zeros(len(Xa), np.int64)
            for c0 in range(0, len(Xa), 64):
                inl, d, e = score(cams, Xa[c0:c0 + 64], a, px[:, 0], px[:, 1], thr2)
                band.add_scores(d, e, thr2)
                cnt[c0:c0 + 64] = inl.sum(1)
            w = int(np.argmax(cnt))                                     # the first of equals: the lowest h
            winner = (Xa[w], int(cnt[w]))
        refit = None
        if winner is not None and winner[1] >= 2:
            inl, _, _ = score(cams, winner[0][None], a, px[:, 0], px[:, 1], thr2)
            r = np.flatnonzero(inl[0])
            rows = dlt_rows(cams, a[r], px[r, 0], px[r, 1]).reshape(1, -1, 4)
            refit = len(refits)
            refits.append(sums(rows)[0])
        work[wi] = (j, pos, a, px, winner, refit)
    Y_all, yok = solve(np.array(refits)) if refits else (np.zeros((0, 3)), np.zeros(0, bool))

    # per track: the keep rule and the outputs
    for j, pos, a, px, winner, refit in work:
        X, count, kept = None, 0, False
        if winner is not None:
            X, count = winner
            if refit is not None and yok[refit]:
                inl, d, e = score(cams, Y_all[refit][None], a, px[:, 0], px[:, 1], thr2)
                band.add_scores(d, e, thr2)
                if int(inl.sum()) >= count:
                    X, count, kept = Y_all[refit], int(inl.sum()), True
        has = winner is not None and count >= 2
        if has:
            stats[5] += 1
            stats[6] += kept
            stats[7] += count
            points[j] = X
            counts[j] = count
            inl, d, e = score(cams, X[None], a, px[:, 0], px[:, 1], thr2)
            band.add_scores(d, e, thr2)
            with np.errstate(divide="ignore", invalid="ignore"):
                err = np.where(d[0] > 0, np.sqrt(e[0] / (d[0] * d[0])), np.inf)
            errors[pos] = err.astype(np.float32)
            inlier[pos] = inl[0]
        else:
            errors[pos] = np.nan
            inlier[pos] = False
    return dict(points=points, counts=counts, errors=errors, inlier=inlier, stats=stats, band=band)
