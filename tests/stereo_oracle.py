"""Float64 restatement of dense reconstruction as include/cudasift_b200.h states it: the undistortion of images, the
PatchMatch tables, homography, view cost, aggregation, draws, start, candidate list and selection rule, one half-step
from a given state, the full loop, and the fusion of depth maps.  Everything is vectorised over pixels.  Values that the
library rounds to float (the tables, H, every hypothesis) are rounded here at the same points."""
import numpy as np

GOLD = np.uint64(0x9E3779B97F4A7C15)
VAR_FLOOR = 1.0
OFFSETS = [(-1, 0), (1, 0), (0, -1), (0, 1), (-5, 0), (5, 0), (0, -5), (0, 5)]


def splitmix64(z):
    with np.errstate(over="ignore"):
        z = z + GOLD
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draw(seed, ref, pix, it, slot):
    """u = (splitmix64(seed + GOLD c) >> 11) 2^-53, c = ((ref 2^24 + pix) 64 + it) 16 + slot."""
    pix = np.asarray(pix, np.uint64)
    with np.errstate(over="ignore"):
        c = ((np.uint64(ref) * np.uint64(1 << 24) + pix) * np.uint64(64) + np.uint64(it)) * np.uint64(16) + \
            np.uint64(slot)
        z = splitmix64(np.uint64(seed) + GOLD * c)
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def kinv(K):
    """K^-1 of an upper-triangular K with K[2, 2] = 1, in the closed form the library uses."""
    K = np.asarray(K, np.float64).reshape(9)
    return np.array([[1 / K[0], -K[1] / (K[0] * K[4]), (K[1] * K[5] - K[2] * K[4]) / (K[0] * K[4])],
                     [0, 1 / K[4], -K[5] / K[4]], [0, 0, 1.0]])


def bilinear(img, u, v):
    """The header's bilinear rule in float64 at (u, v) (clamped to the image)."""
    H, W = img.shape
    u = np.clip(u, 0.0, W - 1.0)
    v = np.clip(v, 0.0, H - 1.0)
    x0 = np.minimum(u.astype(np.int64), W - 2)
    y0 = np.minimum(v.astype(np.int64), H - 2)
    fx, fy = u - x0, v - y0
    im = img.astype(np.float64)
    a = im[y0, x0] + fx * (im[y0, x0 + 1] - im[y0, x0])
    b = im[y0 + 1, x0] + fx * (im[y0 + 1, x0 + 1] - im[y0 + 1, x0])
    return a + fy * (b - a)


def undistort(img, K, dist):
    """cs_undistort_images for one image: (output float64, outside count)."""
    H, W = img.shape
    K = np.asarray(K, np.float64).reshape(9)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    b = (y - K[5]) / K[4]
    a = (x - K[2] - K[1] * b) / K[0]
    r2 = a * a + b * b
    s = 1.0 + dist[0] * r2 + dist[1] * r2 * r2
    u = (K[0] * a * s + K[1] * b * s + K[2]).astype(np.float32).astype(np.float64)
    v = (K[4] * b * s + K[5]).astype(np.float32).astype(np.float64)
    out = ~((u >= 0) & (u <= W - 1) & (v >= 0) & (v <= H - 1))
    res = bilinear(img, u, v)
    res[out] = 0.0
    return res, int(out.sum())


class Job:
    """A job's float tables: Kinv (float64), and per source A_s, b_s rounded to float."""

    def __init__(self, Ks, Rs, ts, ref, sources, dmin, dmax):
        self.ref, self.sources = ref, [int(s) for s in sources]
        self.dmin, self.dmax = np.float32(dmin), np.float32(dmax)
        self.Kinv = kinv(Ks[ref])
        self.A, self.b = [], []
        for s in self.sources:
            Rsr = Rs[s] @ Rs[ref].T
            tsr = ts[s] - Rsr @ ts[ref]
            self.A.append((Ks[s] @ Rsr @ self.Kinv).astype(np.float32).astype(np.float64))
            self.b.append((Ks[s] @ tsr).astype(np.float32).astype(np.float64))


def rays(job, x, y):
    return np.stack([x, y, np.ones_like(x)], -1).astype(np.float64) @ job.Kinv.T


def homographies(job, z, n, ray):
    """H_s (float-rounded, as float64) for hypotheses z [P], n [P, 3] (floats) at rays [P, 3]: [S][P, 3, 3]."""
    z = np.asarray(z, np.float64)
    n = np.asarray(n, np.float64)
    den = z * np.sum(n * ray, -1)
    m = (n @ job.Kinv) / den[:, None]
    return [(A[None] + b[None, :, None] * m[:, None, :]).astype(np.float32).astype(np.float64)
            for A, b in zip(job.A, job.b)]


def view_cost(ref, src, H, x, y, radius, step):
    """Per pixel: (cost (2 when invalid), invalid, marginal) of the float homographies H [P, 3, 3] at (x, y).
    Marginal: a decision lies within 1e-3 of its threshold (relative for the variance floor and for w)."""
    Hh, Wh = ref.shape
    Hs, Ws = src.shape
    P = len(x)
    invalid = np.zeros(P, bool)
    marginal = np.zeros(P, bool)
    xf, yf = x.astype(np.float64), y.astype(np.float64)

    def proj(X, Y):
        q = [H[:, k, 0] * X + H[:, k, 1] * Y + H[:, k, 2] for k in range(3)]
        mag = np.abs(H[:, 2, 0] * X) + np.abs(H[:, 2, 1] * Y) + np.abs(H[:, 2, 2])
        return q, mag

    (q0, q1, q2), mag = proj(xf, yf)
    invalid |= ~(q2 > 0)
    marginal |= np.abs(q2) <= 1e-3 * mag
    with np.errstate(divide="ignore", invalid="ignore"):
        uc, vc = q0 / q2, q1 / q2
    inside = (uc >= 0) & (uc <= Ws - 1) & (vc >= 0) & (vc <= Hs - 1)
    invalid |= ~inside
    marginal |= (np.abs(uc) <= 1e-3) | (np.abs(uc - (Ws - 1)) <= 1e-3) | (np.abs(vc) <= 1e-3) | \
        (np.abs(vc - (Hs - 1)) <= 1e-3)
    r00 = ref[y, x].astype(np.float64)
    s00 = bilinear(src, np.nan_to_num(uc), np.nan_to_num(vc))
    sd = np.zeros(P)
    se, sdd, see, sde = sd.copy(), sd.copy(), sd.copy(), sd.copy()
    for j in range(-radius, radius + 1, step):
        yy = np.clip(y + j, 0, Hh - 1)
        for i in range(-radius, radius + 1, step):
            (a0, a1, a2), m2 = proj(xf + i, yf + j)
            invalid |= ~(a2 > 0)
            marginal |= np.abs(a2) <= 1e-3 * m2
            with np.errstate(divide="ignore", invalid="ignore"):
                u, v = np.nan_to_num(a0 / a2), np.nan_to_num(a1 / a2)
            d = ref[yy, np.clip(x + i, 0, Wh - 1)].astype(np.float64) - r00
            e = bilinear(src, u, v) - s00
            sd += d
            se += e
            sdd += d * d
            see += e * e
            sde += d * e
    N = float((2 * radius // step + 1) ** 2)
    md, me = sd / N, se / N
    vd, ve = sdd / N - md * md, see / N - me * me
    invalid |= ~((vd >= VAR_FLOOR) & (ve >= VAR_FLOOR))
    marginal |= (np.abs(vd - VAR_FLOOR) <= 1e-3 * VAR_FLOOR) | (np.abs(ve - VAR_FLOOR) <= 1e-3 * VAR_FLOOR)
    with np.errstate(divide="ignore", invalid="ignore"):
        c = 1.0 - (sde / N - md * me) / np.sqrt(vd * ve)
    c = np.clip(np.nan_to_num(c, nan=2.0), 0.0, 2.0)
    c[invalid] = 2.0
    return c, invalid, marginal


def cost(images, job, x, y, z, n, radius, step, topK):
    """Aggregated cost of hypotheses (z, n) at pixels (x, y): (cost, invalid views per pixel, marginal)."""
    ray = rays(job, x, y)
    Hs = homographies(job, z, n, ray)
    cs, inv, mar = [], 0, np.zeros(len(x), bool)
    for s, H in zip(job.sources, Hs):
        c, i, m = view_cost(images[job.ref], images[s], H, x, y, radius, step)
        cs.append(c)
        inv = inv + i
        mar |= m
    cs = np.sort(np.array(cs), axis=0)[:topK]
    return cs.mean(axis=0), inv, mar


def face(m, ray):
    """normalise(m), negated to face the ray (-ray / |ray| for a zero or perpendicular m), rounded to float."""
    m = np.array(m, np.float64)
    ln = np.linalg.norm(m, axis=-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        m = np.where(ln[:, None] > 0, m / ln[:, None], 0.0)
    d = np.sum(m * ray, -1)
    m = np.where((d > 0)[:, None], -m, m)
    zero = d == 0
    m[zero] = -ray[zero] / np.linalg.norm(ray[zero], axis=-1, keepdims=True)
    return m.astype(np.float32)


def random_hyp(seed, job, W, x, y, it, s0):
    pix = y * W + x
    lo, hi = 1.0 / np.float64(job.dmax), 1.0 / np.float64(job.dmin)
    z = (1.0 / (lo + draw(seed, job.ref, pix, it, s0) * (hi - lo))).astype(np.float32)
    m = np.stack([2.0 * draw(seed, job.ref, pix, it, s0 + 1 + k) - 1.0 for k in range(3)], -1)
    return z, face(m, rays(job, x, y))


def start(images, job, seed, radius, step, topK):
    """Iteration 0: (depth, normal, cost) maps."""
    H, W = images[job.ref].shape
    y, x = [a.reshape(-1) for a in np.mgrid[0:H, 0:W]]
    z, n = random_hyp(seed, job, W, x, y, 0, 0)
    c, _, _ = cost(images, job, x, y, z, n, radius, step, topK)
    return z.reshape(H, W), n.reshape(H, W, 3), c.astype(np.float32).reshape(H, W)


def candidates(job, depth, normal, x, y, it, seed):
    """The candidate list of pixels (x, y) at iteration it from the state (depth, normal): a list of (z, n, valid)
    in the header's order (8 propagations, depth move, normal move, both, random)."""
    H, W = depth.shape
    ray = rays(job, x, y)
    z0, n0 = depth[y, x], normal[y, x]
    out = []
    for dx, dy in OFFSETS:
        xq, yq = x + dx, y + dy
        on = (xq >= 0) & (xq < W) & (yq >= 0) & (yq < H)
        xc, yc = np.clip(xq, 0, W - 1), np.clip(yq, 0, H - 1)
        nq = normal[yc, xc]
        zq = depth[yc, xc].astype(np.float64)
        d = np.sum(nq.astype(np.float64) * ray, -1)
        num = zq * np.sum(nq.astype(np.float64) * rays(job, xc, yc), -1)
        with np.errstate(divide="ignore", invalid="ignore"):
            z = (num / d).astype(np.float32)
        ok = on & (d < 0) & (z >= job.dmin) & (z <= job.dmax)
        out.append((np.where(ok, z, z0), np.where(ok[:, None], nq, n0), ok))
    rho = 2.0 ** -it
    lo, hi = 1.0 / np.float64(job.dmax), 1.0 / np.float64(job.dmin)
    pix = y * W + x

    def moved_depth(slot):
        u = draw(seed, job.ref, pix, it, slot)
        inv = np.clip(1.0 / z0.astype(np.float64) + rho * (2.0 * u - 1.0) * (hi - lo), lo, hi)
        return (1.0 / inv).astype(np.float32)

    def moved_normal(slot):
        m = np.stack([n0[:, k].astype(np.float64) + rho * (2.0 * draw(seed, job.ref, pix, it, slot + k) - 1.0)
                      for k in range(3)], -1)
        return face(m, ray)

    yes = np.ones(len(x), bool)
    out.append((moved_depth(0), n0, yes))
    out.append((z0, moved_normal(1), yes))
    out.append((moved_depth(4), moved_normal(5), yes))
    zr, nr = random_hyp(seed, job, W, x, y, it, 8)
    out.append((zr, nr, yes))
    return out


def colour_pixels(H, W, colour):
    y, x = [a.reshape(-1) for a in np.mgrid[0:H, 0:W]]
    k = ((x + y) & 1) == colour
    return x[k], y[k]


def half_step(images, job, state, it, colour, seed, radius, step, topK, eps=None):
    """One half-step from state = (depth, normal, cost).  Returns the new state (the oracle's own choice).  With eps,
    also per pixel of the colour: the options {current} + candidates, their oracle costs, and the admissible mask
    (cost within eps of the best)."""
    depth, normal, cst = (a.copy() for a in state)
    H, W = depth.shape
    x, y = colour_pixels(H, W, colour)
    cands = candidates(job, state[0], state[1], x, y, it, seed)
    cur_c, _, cur_m = cost(images, job, x, y, depth[y, x], normal[y, x], radius, step, topK)
    best_c = cst[y, x].astype(np.float64).copy()
    best_z, best_n = depth[y, x].copy(), normal[y, x].copy()
    opt_z, opt_n, opt_c, opt_ok, opt_m = [best_z.copy()], [best_n.copy()], [cur_c], [np.ones(len(x), bool)], [cur_m]
    for z, n, ok in cands:
        c, _, m = cost(images, job, x, y, z, n, radius, step, topK)
        c = np.where(ok, c, np.inf)
        better = c < best_c
        best_c = np.where(better, c, best_c)
        best_z = np.where(better, z, best_z)
        best_n = np.where(better[:, None], n, best_n)
        opt_z.append(z)
        opt_n.append(n)
        opt_c.append(c)
        opt_ok.append(ok)
        opt_m.append(m)
    depth[y, x], normal[y, x], cst[y, x] = best_z, best_n, best_c.astype(np.float32)
    if eps is None:
        return depth, normal, cst
    C = np.array(opt_c)
    adm = np.array(opt_ok) & (C <= C.min(axis=0) + eps)
    return (depth, normal, cst), dict(x=x, y=y, z=np.array(opt_z), n=np.array(opt_n), cost=C, admissible=adm,
                                      marginal=np.array(opt_m))


def run(images, job, seed, radius, step, numIterations, topK):
    """The full loop: start, then numIterations iterations of the even and the odd half-step."""
    state = start(images, job, seed, radius, step, topK)
    for it in range(1, numIterations + 1):
        for colour in (0, 1):
            state = half_step(images, job, state, it, colour, seed, radius, step, topK)
    return state


def fuse(images, Ks, Rs, ts, jobs, depth, normal, cst, maxCost, minConsistent, maxReprojError, maxDepthError,
         maxNormalErrorDeg):
    """cs_fuse_depth_maps: per pixel of every job, in ascending (a, pixel) order, (a, pixel, emitted, position, normal,
    intensity, margin): margin is the smallest distance of any decision the pixel depended on from its threshold
    (relative to it), |cost - maxCost| alone for a pixel above maxCost."""
    jobOf = {int(j[0]): k for k, j in enumerate(jobs)}
    minDot = np.cos(np.radians(maxNormalErrorDeg))
    rows = []
    for k in sorted(range(len(jobs)), key=lambda k: jobs[k][0]):
        a, sources = int(jobs[k][0]), [int(s) for s in jobs[k][1]]
        H, W = depth[k].shape
        y, x = [v.reshape(-1) for v in np.mgrid[0:H, 0:W]]
        keep = cst[k].reshape(-1) <= maxCost
        margin = np.abs(cst[k].reshape(-1) - maxCost)
        Ki = kinv(Ks[a])
        z = depth[k].reshape(-1).astype(np.float64)
        Xc = z[:, None] * (np.stack([x, y, np.ones_like(x)], -1) @ Ki.T)
        X = (Xc - ts[a]) @ Rs[a]
        n = normal[k].reshape(-1, 3).astype(np.float64) @ Rs[a]
        sumX, sumN = X.copy(), n.copy()
        sumI = images[a][y, x].astype(np.float64)
        good = np.zeros(len(x), int)
        lower = np.zeros(len(x), bool)
        for b in sources:
            if b not in jobOf:
                continue
            kb = jobOf[b]
            Hb, Wb = depth[kb].shape
            Y = X @ Rs[b].T + ts[b]
            with np.errstate(divide="ignore", invalid="ignore"):
                u = (Ks[b][0] @ Y.T) / Y[:, 2]
                v = (Ks[b][1] @ Y.T) / Y[:, 2]
            qx, qy = np.floor(u + 0.5), np.floor(v + 0.5)
            ok = (Y[:, 2] > 0) & (qx >= 0) & (qx < Wb) & (qy >= 0) & (qy < Hb)
            m_round = np.minimum(np.abs(u + 0.5 - np.round(u + 0.5)), np.abs(v + 0.5 - np.round(v + 0.5)))
            qxi, qyi = np.clip(np.nan_to_num(qx), 0, Wb - 1).astype(int), np.clip(np.nan_to_num(qy), 0, Hb - 1).astype(int)
            cb = cst[kb][qyi, qxi]
            zb = depth[kb][qyi, qxi].astype(np.float64)
            nb = normal[kb][qyi, qxi].astype(np.float64) @ Rs[b]
            dz = np.abs(zb - Y[:, 2]) - maxDepthError * Y[:, 2]
            dot = np.sum(n * nb, -1)
            Xq = (zb[:, None] * (np.stack([qx, qy, np.ones_like(qx)], -1) @ kinv(Ks[b]).T) - ts[b]) @ Rs[b]
            Z = Xq @ Rs[a].T + ts[a]
            with np.errstate(divide="ignore", invalid="ignore"):
                ex = (Ks[a][0] @ Z.T) / Z[:, 2] - x
                ey = (Ks[a][1] @ Z.T) / Z[:, 2] - y
            e2 = ex * ex + ey * ey
            c = ok & (cb <= maxCost) & (dz <= 0) & (dot >= minDot) & (Z[:, 2] > 0) & (e2 <= maxReprojError ** 2)
            with np.errstate(invalid="ignore"):
                mb = np.nanmin(np.stack([np.where(ok, m_round, np.inf), np.where(ok, np.abs(cb - maxCost), np.inf),
                                         np.where(ok, np.abs(dz) / np.maximum(Y[:, 2], 1e-30), np.inf),
                                         np.where(ok, np.abs(dot - minDot), np.inf),
                                         np.where(ok, np.abs(e2 - maxReprojError ** 2) / maxReprojError ** 2, np.inf)]),
                               axis=0)
            margin = np.minimum(margin, np.where(keep, mb, np.inf))
            good += c
            lower |= c & (b < a)
            sumX += np.where(c[:, None], Xq, 0.0)
            sumN += np.where(c[:, None], nb, 0.0)
            sumI += np.where(c, images[b][qyi, qxi].astype(np.float64), 0.0)
        emit = keep & (good >= minConsistent) & ~lower
        views = good + 1
        for p in range(len(x)):
            rows.append((a, int(p), bool(emit[p]), sumX[p] / views[p], sumN[p] / np.linalg.norm(sumN[p]),
                         sumI[p] / views[p], float(margin[p])))
    return rows
