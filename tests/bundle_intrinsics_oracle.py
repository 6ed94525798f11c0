"""Self-calibrating bundle adjustment (cs_bundle_adjust_intrinsics, camera block NC = 9) and the undistortion of
records (cs_undistort_records) restated in numpy float64.  Intrinsics extends bundle_oracle.Problem: the radial camera
model, its Jacobians, the robust loss through Ceres's corrector, the focal update with the K ratios held and the LM
loop with the focal test.  The header is the rule; sums run in numpy's order, so results agree with the device to
rounding."""
import numpy as np

import bundle_oracle as bo

LOSSES = {"trivial": 0, "soft_l1": 1, "cauchy": 2}


def loss_rho(loss, c2, s):
    """c^2 rho(s / c^2) and the corrector's scale sqrt(rho'(s / c^2)) per squared norm s."""
    s = np.asarray(s, np.float64)
    if loss == 0:
        return s.copy(), np.ones_like(s)
    u = s / c2
    if loss == 1:
        q = np.sqrt(1.0 + u)
        return c2 * (2.0 * u / (q + 1.0)), np.sqrt(1.0 / q)
    return c2 * np.log1p(u), np.sqrt(1.0 / (1.0 + u))


def distort(K, k, X):
    """Pixels [n, 2] of camera-frame points X [n, 3] under K [3, 3] and k = (k1, k2)."""
    a, b = X[:, 0] / X[:, 2], X[:, 1] / X[:, 2]
    rho2 = a * a + b * b
    D = 1.0 + rho2 * (k[0] + k[1] * rho2)
    ad, bd = D * a, D * b
    return np.stack([K[0, 0] * ad + K[0, 1] * bd + K[0, 2], K[1, 1] * bd + K[1, 2]], 1)


NEWTON = 20


def solve_ru(rd, k):
    """The undistorted radius r_u of r_d by the header's Newton rule, and whether the rule accepts it."""
    ru, ok = rd, False
    for _ in range(NEWTON):
        r2 = ru * ru
        d = 1.0 + r2 * (3.0 * k[0] + 5.0 * k[1] * r2)
        if not d > 0.0:
            break
        step = (ru * (1.0 + r2 * (k[0] + k[1] * r2)) - rd) / d
        ru -= step
        if abs(step) <= 1e-12 * rd:
            ok = True
            break
    r2 = ru * ru
    return ru, bool(ok and 1.0 + r2 * (3.0 * k[0] + 5.0 * k[1] * r2) > 0.0)


def undistort(K, k, xy):
    """cs_undistort_records' rule on float32 positions xy [n, 2]: float32 [n, 2], NaN where the solve fails."""
    x, y = xy[:, 0].astype(np.float64), xy[:, 1].astype(np.float64)
    b = (y - K[1, 2]) / K[1, 1]
    a = (x - K[0, 2] - K[0, 1] * b) / K[0, 0]
    out = np.full((len(xy), 2), np.nan, np.float32)
    for i in range(len(xy)):
        rd = np.sqrt(a[i] * a[i] + b[i] * b[i])
        ru, ok = solve_ru(rd, k)
        s = ru / rd if rd > 0.0 else 1.0
        if ok:
            au, bu = a[i] * s, b[i] * s
            out[i] = (K[0, 0] * au + K[0, 1] * bu + K[0, 2], K[1, 1] * bu + K[1, 2])
    return out


class Intrinsics(bo.Problem):
    """bo.Problem with dists [S, 2] (None: zero), refine (one mask or one per image: bit 0 focal, 1 k1, 2 k2), loss
    (0 trivial, 1 soft-L1, 2 Cauchy) and lossScale.  self.mask is [S, 9]: (w, delta, f, k1, k2)."""

    def __init__(self, xy, Ks, Rs, ts, offsets, members, points, dists=None, refine=3, loss=0, lossScale=1.0,
                 use=None, fixed=None):
        super().__init__(xy, Ks, Rs, ts, offsets, members, points, use=use, fixed=fixed)
        S = self.S
        self.k0 = np.zeros((S, 2)) if dists is None else np.asarray(dists, np.float64).reshape(S, 2).copy()
        ref = np.asarray(refine, np.int64).reshape(-1)
        self.refine = np.full(S, int(ref[0])) if ref.size == 1 else ref
        hasobs = np.zeros(S, bool)
        hasobs[self.a] = True
        im = np.array([[(int(r) >> j) & 1 for j in range(3)] for r in self.refine], bool).reshape(S, 3)
        self.mask = np.concatenate([self.mask, im & hasobs[:, None]], 1)
        self.stats[5] = int(self.mask.sum())
        self.loss, self.c2 = int(loss), float(lossScale) ** 2

    # ---- residuals and Jacobians ----
    def _proj(self, R, t, X, K, k):
        K = self.K if K is None else K
        k = self.k0 if k is None else k
        RX = np.einsum("nij,nj->ni", R[self.a], X[self.k])
        Xc = RX + t[self.a]
        z = Xc[:, 2]
        a, b = Xc[:, 0] / z, Xc[:, 1] / z
        KK, kk = K[self.a], k[self.a]
        rho2 = a * a + b * b
        D = 1.0 + rho2 * (kk[:, 0] + kk[:, 1] * rho2)
        ad, bd = D * a, D * b
        pu, pv = KK[:, 0, 0] * ad + KK[:, 0, 1] * bd, KK[:, 1, 1] * bd
        r = np.stack([pu + KK[:, 0, 2] - self.x, pv + KK[:, 1, 2] - self.y], 1)
        return dict(RX=RX, z=z, a=a, b=b, K=KK, k=kk, rho2=rho2, D=D, pu=pu, pv=pv, r=r)

    def residuals(self, R, t, X, K=None, k=None):
        p = self._proj(R, t, X, K, k)
        return p["r"], p["z"]

    def cost(self, R, t, X, K=None, k=None):
        r, z = self.residuals(R, t, X, K, k)
        rho, _ = loss_rho(self.loss, self.c2, (r * r).sum(1))
        return float(rho.sum()), bool((z > 0).all())

    def jacobians(self, R, t, X, K=None, k=None, robust=True):
        """J_c [N, 2, 9] (w, delta, f, k1, k2), J_p [N, 2, 3], r [N, 2]; scaled by sqrt(rho') when robust."""
        p = self._proj(R, t, X, K, k)
        a, b, z, KK, kk, rho2, D = p["a"], p["b"], p["z"], p["K"], p["k"], p["rho2"], p["D"]
        Dp = 2.0 * (kk[:, 0] + 2.0 * kk[:, 1] * rho2)
        Daa, Dab, Dbb = D + Dp * a * a, Dp * a * b, D + Dp * b * b
        du = np.stack([np.stack([KK[:, 0, 0] * Daa + KK[:, 0, 1] * Dab, KK[:, 0, 0] * Dab + KK[:, 0, 1] * Dbb], 1),
                       np.stack([KK[:, 1, 1] * Dab, KK[:, 1, 1] * Dbb], 1)], 1)            # [N, 2, 2]
        gr = np.stack([du[:, :, 0] / z[:, None], du[:, :, 1] / z[:, None],
                       -(du[:, :, 0] * a[:, None] + du[:, :, 1] * b[:, None]) / z[:, None]], 2)   # [N, 2, 3]
        Jc = np.zeros((self.N, 2, 9))
        Jc[:, :, :3] = np.cross(p["RX"][:, None, :], gr)
        Jc[:, :, 3:6] = gr
        Jc[:, 0, 6], Jc[:, 1, 6] = p["pu"] / KK[:, 0, 0], p["pv"] / KK[:, 0, 0]
        Jc[:, 0, 7], Jc[:, 1, 7] = (KK[:, 0, 0] * a + KK[:, 0, 1] * b) * rho2, KK[:, 1, 1] * b * rho2
        Jc[:, :, 8] = Jc[:, :, 7] * rho2[:, None]
        Jp = np.einsum("nqi,nij->nqj", gr, R[self.a])
        r = p["r"]
        if robust:
            _, w = loss_rho(self.loss, self.c2, (r * r).sum(1))
            Jc, Jp, r = Jc * w[:, None, None], Jp * w[:, None, None], r * w[:, None]
        return Jc, Jp, r

    @staticmethod
    def apply9(R, t, K, k, mask, dc):
        """The candidate (R, t, K, k) of the step dc [S, 9]."""
        R1, t1 = bo.Problem.apply(R, t, mask[:, :6], dc[:, :6])
        K1, k1 = K.copy(), k.copy()
        for a in range(len(K)):
            if mask[a, 6]:
                f = K[a, 0, 0] + dc[a, 6]
                s = f / K[a, 0, 0]
                K1[a, 0, 0], K1[a, 0, 1], K1[a, 1, 1] = f, K[a, 0, 1] * s, K[a, 1, 1] * s
            for j in range(2):
                if mask[a, 7 + j]:
                    k1[a, j] = k[a, j] + dc[a, 7 + j]
        return R1, t1, K1, k1

    # ---- the linear solve ----
    def solve(self, Jc, Jp, r, lam, maxLinear, tol):
        """bo.Problem.solve's Schur + PCG step with the camera block of Jc [N, 2, C] (C = 9 here, self.mask [S, C]):
        (ok, dc [S, C], dp [T, 3], CG iterations).  The same statement and the same numpy order, every 6 a C."""
        S, T, C = self.S, self.T, Jc.shape[2]
        U = np.zeros((S, C, C)); gc = np.zeros((S, C))
        V = np.zeros((T, 3, 3)); gp = np.zeros((T, 3))
        np.add.at(U, self.a, np.einsum("nqi,nqj->nij", Jc, Jc))
        np.add.at(gc, self.a, np.einsum("nqi,nq->ni", Jc, r))
        np.add.at(V, self.k, np.einsum("nqi,nqj->nij", Jp, Jp))
        np.add.at(gp, self.k, np.einsum("nqi,nq->ni", Jp, r))
        Wo = np.einsum("nqi,nqj->nij", Jc, Jp)                              # [N, C, 3]
        Vi = {}
        for k in self.parts:
            L = bo.chol_ok(bo.damp(V[k], lam))
            if L is None:
                return False, None, None, 0
            Vi[int(k)] = bo.chol_solve(L, np.eye(3))
        q = np.zeros((T, 3))
        for k in self.parts:
            q[k] = Vi[int(k)] @ gp[k]
        rhs = -gc.copy()
        np.add.at(rhs, self.a, np.einsum("nij,nj->ni", Wo, q[self.k]))
        Wak = [{} for _ in range(S)]                                        # per image: track -> W_ak
        for n in range(self.N):
            a, k = int(self.a[n]), int(self.k[n])
            Wak[a][k] = Wak[a].get(k, 0) + Wo[n]
        Us = np.zeros((S, C, C)); Ls = []
        for a in range(S):
            m = self.mask[a]
            u = bo.damp(U[a], lam)
            Mb = u.copy()
            for k, w in Wak[a].items():
                Mb -= w @ Vi[k] @ w.T
            fm = np.outer(m, m)
            u = np.where(fm, u, np.eye(C)); Mb = np.where(fm, Mb, np.eye(C))
            L = bo.chol_ok(Mb)
            if L is None:
                return False, None, None, 0
            Us[a] = u
            Ls.append(L)
        rhs = np.where(self.mask, rhs, 0.0)

        def Sx(p):
            h = np.zeros((T, 3))
            np.add.at(h, self.k, np.einsum("nij,ni->nj", Wo, p[self.a]))
            y = np.zeros((T, 3))
            for k in self.parts:
                y[k] = Vi[int(k)] @ h[k]
            Wy = np.zeros((S, C))
            np.add.at(Wy, self.a, np.einsum("nij,nj->ni", Wo, y[self.k]))
            return np.where(self.mask, np.einsum("aij,aj->ai", Us, p) - Wy, 0.0)

        def Minv(v):
            return np.array([bo.chol_solve(Ls[a], v[a]) for a in range(S)]).reshape(S, C)

        x = np.zeros((S, C)); res = rhs.copy(); z = Minv(res); p = np.zeros((S, C))
        bb = float((rhs * rhs).sum()); rr = bb; rz = float((res * z).sum()); beta = 0.0
        it = 0
        self.cg_history = []
        while it < maxLinear and not (rr <= tol * tol * bb):
            p = z + beta * p
            qv = Sx(p)
            pq = float((p * qv).sum())
            self.cg_history.append((rr, tol * tol * bb, pq))
            if not (pq > 0.0):
                break
            alpha = rz / pq
            x = x + alpha * p
            res = res - alpha * qv
            z = Minv(res)
            it += 1
            rr = float((res * res).sum())
            rzn = float((res * z).sum())
            beta, rz = rzn / rz, rzn
        self.cg_history.append((rr, tol * tol * bb, np.nan))
        h = -gp.copy()
        np.add.at(h, self.k, -np.einsum("nij,ni->nj", Wo, x[self.a]))
        dp = np.zeros((T, 3))
        for k in self.parts:
            dp[k] = Vi[int(k)] @ h[k]
        return True, x, dp, it

    # ---- the LM loop ----
    def run(self, maxIterations=50, maxLinear=100, tol=1e-6):
        """Returns (K, k, R, t, X, cost (initial, final), trace [iterations, 4], accepted); self.history as
        bo.Problem.run's."""
        R, t, X, K, k = self.R0.copy(), self.t0.copy(), self.X0.copy(), self.K.copy(), self.k0.copy()
        cost = self.cost(R, t, X, K, k)[0] if self.N else 0.0
        cost0, lam, trace, accepted, self.history = cost, 1e-3, [], 0, []
        for it in range(maxIterations if self.N else 0):
            Jc, Jp, r = self.jacobians(R, t, X, K, k)
            ok, dc, dp, cgit = self.solve(Jc, Jp, r, lam, maxLinear, tol)
            cand, behind, badf = np.nan, True, False
            if ok:
                R1, t1, K1, k1 = self.apply9(R, t, K, k, self.mask, dc)
                X1 = X.copy()
                X1[self.parts] = X[self.parts] + dp[self.parts]
                badf = bool((self.mask[:, 6] & ~(K1[:, 0, 0] > 0)).any())
                cand, front = self.cost(R1, t1, X1, K1, k1)
                behind = not front
            acc = ok and not behind and not badf and cand < cost
            trace.append((cand, lam, cgit, float(acc)))
            self.history.append(dict(cost=cost, cand=cand, cg=list(self.cg_history) if ok else []))
            if acc:
                stop = cost - cand <= 1e-10 * cost
                R, t, X, K, k, cost, lam = R1, t1, X1, K1, k1, cand, lam / 10.0
                accepted += 1
                if stop:
                    break
            else:
                lam *= 10.0
                if lam > 1e16:
                    break
        return K, k, R, t, X, (cost0, cost), np.array(trace).reshape(-1, 4), accepted

    def outputs9(self, K, k, R, t, X, maxError):
        """errors float32 [M] and inlier [M] under the NC = 9 member rule, and the members written."""
        err = np.full(self.M, np.nan, np.float32)
        inl = np.zeros(self.M, bool)
        written = np.zeros(self.M, bool)
        for kk in range(self.T):
            if not self.wellformed[kk]:
                continue
            lo, hi = int(self.offsets[kk]), int(self.offsets[kk + 1])
            written[lo:hi] = True
            if not np.isfinite(X[kk]).all():
                continue
            for m in range(lo, hi):
                if not self.valid[m]:
                    continue
                a, f = int(self.members[m, 0]), int(self.members[m, 1])
                Xc = R[a] @ X[kk] + t[a]
                px = distort(K[a], k[a], Xc[None])[0]
                e2 = float(((px - self.xy[a][f].astype(np.float64)) ** 2).sum())
                inl[m] = Xc[2] > 0 and e2 < maxError * maxError
                err[m] = np.float32(np.sqrt(e2)) if Xc[2] > 0 else np.inf
        return err, inl, written
