"""Float64 restatement of cs_patch_match_stereo_geometric as include/cudasift_b200.h states it: the geometric error,
the combined view cost, the start rule and one half-step, vectorised over pixels.  Everything the two passes share
(tables, homographies, view costs, draws, facing, propagation) comes from stereo_oracle."""
import numpy as np

import stereo_oracle as so

IT0 = 32                    # the counter iteration of the geometric start; iteration k draws at IT0 + k
MARGIN = 1e-9


class GeomJob(so.Job):
    """A job's tables plus, per source, R_sr, t_sr (float64) and the cameras the geometric error uses."""

    def __init__(self, Ks, Rs, ts, ref, sources, dmin, dmax):
        super().__init__(Ks, Rs, ts, ref, sources, dmin, dmax)
        self.Kr = np.asarray(Ks[ref], np.float64)
        self.Rsr = [Rs[s] @ Rs[ref].T for s in self.sources]
        self.tsr = [ts[s] - R @ ts[ref] for s, R in zip(self.sources, self.Rsr)]
        self.Ks = [np.asarray(Ks[s], np.float64) for s in self.sources]
        self.Kinvs = [so.kinv(Ks[s]) for s in self.sources]


def geom_error(job, k, prior, x, y, z, gmax):
    """Source k's g (as float32 values in float64) for depths z at pixels (x, y), with (capped, marginal) per pixel.
    prior: the source's depth map, or None."""
    X = np.asarray(z, np.float64)[:, None] * so.rays(job, x, y)
    Y = X @ job.Rsr[k].T + job.tsr[k]
    P = len(x)
    e = np.full(P, np.inf)
    marginal = np.abs(Y[:, 2]) <= MARGIN
    if prior is not None:
        Hs, Ws = prior.shape
        with np.errstate(divide="ignore", invalid="ignore"):
            uv = (Y @ job.Ks[k].T)[:, :2] / Y[:, 2:3]
        u, v = uv[:, 0], uv[:, 1]
        marginal |= (np.abs(u + 0.5 - np.round(u + 0.5)) <= MARGIN) | (np.abs(v + 0.5 - np.round(v + 0.5)) <= MARGIN)
        qx, qy = np.floor(u + 0.5), np.floor(v + 0.5)
        ok = (Y[:, 2] > 0) & (qx >= 0) & (qx < Ws) & (qy >= 0) & (qy < Hs)
        zs = prior[np.clip(np.nan_to_num(qy), 0, Hs - 1).astype(int),
                   np.clip(np.nan_to_num(qx), 0, Ws - 1).astype(int)].astype(np.float64)
        with np.errstate(invalid="ignore"):
            ok &= np.isfinite(zs) & (zs > 0)
        Xs = zs[:, None] * (np.stack([u, v, np.ones(P)], -1) @ job.Kinvs[k].T)
        Z = (Xs - job.tsr[k]) @ job.Rsr[k]
        marginal |= ok & (np.abs(Z[:, 2]) <= MARGIN)
        ok &= Z[:, 2] > 0
        with np.errstate(divide="ignore", invalid="ignore"):
            uvr = (Z @ job.Kr.T)[:, :2] / Z[:, 2:3]
            e = np.where(ok, np.hypot(uvr[:, 0] - x, uvr[:, 1] - y), np.inf)
    capped = ~(e < gmax)
    g = np.minimum(e, gmax).astype(np.float32).astype(np.float64)
    return g, capped, marginal


def cost(images, job, priors, x, y, z, n, radius, step, topK, lam, gmax):
    """Combined cost of hypotheses (z, n) at pixels (x, y): (cost, invalid views, capped valid views, marginal) per
    pixel.  priors[image]: depth map or None.  Each view costs c_photo + (float) lam g, c_photo 2 when invalid."""
    ray = so.rays(job, x, y)
    Hs = so.homographies(job, z, n, ray)
    lam32 = float(np.float32(lam))
    cs, inv, cap, mar = [], 0, 0, np.zeros(len(x), bool)
    for k, (s, H) in enumerate(zip(job.sources, Hs)):
        c, i, m = so.view_cost(images[job.ref], images[s], H, x, y, radius, step)
        g, capped, gm = geom_error(job, k, priors[s], x, y, z, gmax)
        cs.append(c + lam32 * g)
        inv = inv + i
        cap = cap + (capped & ~i)
        mar |= m | gm
    cs = np.sort(np.array(cs), axis=0)[:topK]
    return cs.mean(axis=0), inv, cap, mar


def start_rule(job, depth, normal, x, y):
    """Pixels (x, y) whose ref prior (depth [H, W], normal [H, W, 3]) the start takes."""
    z, n = depth[y, x], normal[y, x].astype(np.float64)
    ray = so.rays(job, x, y)
    with np.errstate(invalid="ignore", over="ignore"):
        ok = (z >= job.dmin) & (z <= job.dmax) & np.all(np.isfinite(n), -1)
        ok &= np.sum(n * ray, -1) < 0
        ok &= np.abs(np.sqrt(np.sum(n * n, -1)) - 1.0) <= 1e-3
    return ok


def start(images, job, priors, seed, radius, step, topK, lam, gmax):
    """Iteration 0: (depth, normal, cost, drawn) maps, drawn marking the pixels that took the draws of iteration 32."""
    pd, pn = priors[job.ref]
    H, W = pd.shape
    y, x = [a.reshape(-1) for a in np.mgrid[0:H, 0:W]]
    take = start_rule(job, pd, pn, x, y)
    zr, nr = so.random_hyp(seed, job, W, x, y, IT0, 0)
    z = np.where(take, pd[y, x], zr).astype(np.float32)
    n = np.where(take[:, None], pn[y, x], nr).astype(np.float32)
    c, _, _, _ = cost(images, job, _depths(priors), x, y, z, n, radius, step, topK, lam, gmax)
    return z.reshape(H, W), n.reshape(H, W, 3), c.astype(np.float32).reshape(H, W), ~take.reshape(H, W)


def _depths(priors):
    return {a: (None if p is None else p[0]) for a, p in priors.items()}


def candidates(job, depth, normal, x, y, k, seed):
    """stereo_oracle's candidate list with rho = 2^-k and the draws of counter iteration 32 + k."""
    out = so.candidates(job, depth, normal, x, y, IT0 + k, seed)   # propagation and the random draw: no rho
    H, W = depth.shape
    ray = so.rays(job, x, y)
    z0, n0 = depth[y, x], normal[y, x]
    rho = 2.0 ** -k
    lo, hi = 1.0 / np.float64(job.dmax), 1.0 / np.float64(job.dmin)
    pix = y * W + x

    def moved_depth(slot):
        u = so.draw(seed, job.ref, pix, IT0 + k, slot)
        return (1.0 / np.clip(1.0 / z0.astype(np.float64) + rho * (2.0 * u - 1.0) * (hi - lo), lo, hi)).astype(np.float32)

    def moved_normal(slot):
        m = np.stack([n0[:, c].astype(np.float64) + rho * (2.0 * so.draw(seed, job.ref, pix, IT0 + k, slot + c) - 1.0)
                      for c in range(3)], -1)
        return so.face(m, ray)

    yes = np.ones(len(x), bool)
    out[8] = (moved_depth(0), n0, yes)
    out[9] = (z0, moved_normal(1), yes)
    out[10] = (moved_depth(4), moved_normal(5), yes)
    return out


def half_step(images, job, priors, state, k, colour, seed, radius, step, topK, lam, gmax, eps=None):
    """One half-step from state = (depth, normal, cost), as stereo_oracle.half_step with the combined cost."""
    depth, normal, cst = (a.copy() for a in state)
    H, W = depth.shape
    x, y = so.colour_pixels(H, W, colour)
    pri = _depths(priors)
    cands = candidates(job, state[0], state[1], x, y, k, seed)
    cur_c, _, _, cur_m = cost(images, job, pri, x, y, depth[y, x], normal[y, x], radius, step, topK, lam, gmax)
    best_c = cst[y, x].astype(np.float64).copy()
    best_z, best_n = depth[y, x].copy(), normal[y, x].copy()
    opt_z, opt_n, opt_c, opt_ok, opt_m = [best_z.copy()], [best_n.copy()], [cur_c], [np.ones(len(x), bool)], [cur_m]
    for z, n, ok in cands:
        c, _, _, m = cost(images, job, pri, x, y, z, n, radius, step, topK, lam, gmax)
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


def run(images, job, priors, seed, radius, step, numIterations, topK, lam, gmax):
    """The full pass: the start, then numIterations iterations of the even and the odd half-step."""
    d, n, c, _ = start(images, job, priors, seed, radius, step, topK, lam, gmax)
    state = (d, n, c)
    for k in range(1, numIterations + 1):
        for colour in (0, 1):
            state = half_step(images, job, priors, state, k, colour, seed, radius, step, topK, lam, gmax)
    return state


def consistency(job, priors, depth, gmax=3.0, within=1.0, views=2):
    """Fraction of a map's pixels whose g is <= within px in at least `views` sources, against the priors (truth-free)."""
    H, W = depth.shape
    y, x = [a.reshape(-1) for a in np.mgrid[0:H, 0:W]]
    good = 0
    for k, s in enumerate(job.sources):
        g, _, _ = geom_error(job, k, None if priors[s] is None else priors[s][0], x, y, depth.reshape(-1), gmax)
        good = good + (g <= within)
    return float(np.mean(good >= views))
