"""Bundle adjustment (cs_bundle_adjust) restated in numpy float64: the used observations, the gauge, the residual and
Jacobians, the damped normal equations, the Schur complement with the block-Jacobi preconditioned CG and its stop
rule, the back-substitution, the LM loop and the per-member outputs.  The header at cs_bundle_adjust is the rule; sums
here run in numpy's order, so results agree with the device to rounding."""
import numpy as np

import triangulate_oracle as to


def rodrigues(w):
    """exp([w]x): I + A [w]x + B [w]x^2, A = sin th / th, B = 2 sin^2(th / 2) / th^2 (1 and 1/2 at th = 0)."""
    th2 = float(w @ w)
    A, B = 1.0, 0.5
    if th2 != 0.0:
        th = np.sqrt(th2)
        A, B = np.sin(th) / th, 2.0 * np.sin(0.5 * th) ** 2 / th2
    W = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    return np.eye(3) + A * W + B * (W @ W)


def free_mask(code):
    m = np.ones(6, bool)
    if code == 1:
        m[:] = False
    elif code >= 2:
        m[3 + code - 2] = False
    return m


def chol_ok(A):
    """Cholesky factor of A, or None when a pivot is not > 0 or not finite (the header's rule)."""
    n = len(A)
    L = np.zeros_like(A)
    for j in range(n):
        d = A[j, j] - L[j, :j] @ L[j, :j]
        if not (d > 0.0) or not np.isfinite(d):
            return None
        L[j, j] = np.sqrt(d)
        for i in range(j + 1, n):
            L[i, j] = (A[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
    return L


def chol_solve(L, b):
    z = np.linalg.solve(L, b)
    return np.linalg.solve(L.T, z)


def damp(H, lam):
    H = H.copy()
    d = np.diagonal(H).copy()
    H[np.arange(len(d)), np.arange(len(d))] = d + lam * np.clip(d, 1e-6, 1e32)
    return H


class Problem:
    """The observations a call uses.  xy[a] float32 [n_a, 2] record positions; Ks, Rs [S, 3, 3], ts [S, 3]; offsets,
    members as cs_build_tracks; points [T, 3]; use bool [M] or None; fixed uint8 [S] or None."""

    def __init__(self, xy, Ks, Rs, ts, offsets, members, points, use=None, fixed=None):
        self.K = np.asarray(Ks, np.float64).reshape(-1, 3, 3)
        R0 = np.asarray(Rs, np.float64).reshape(-1, 3, 3)
        t0 = np.asarray(ts, np.float64).reshape(-1, 3)
        self.S = S = len(self.K)
        off = np.asarray(offsets, np.int64)
        mem = np.asarray(members, np.int64).reshape(-1, 2)
        self.T, self.M = len(off) - 1, len(mem)
        self.X0 = np.asarray(points, np.float64).reshape(-1, 3).copy()
        self.xy, self.offsets, self.members = xy, off, mem
        self.fixed = np.zeros(S, np.uint8) if fixed is None else np.asarray(fixed, np.uint8)
        st = np.zeros(8, np.int64)
        k_, a_, m_, x_, y_ = [], [], [], [], []
        self.wellformed = np.zeros(self.T, bool)
        self.valid = np.zeros(self.M, bool)
        for k in range(self.T):
            lo, hi = int(off[k]), int(off[k + 1])
            if lo < 0 or hi < lo or hi > self.M:
                st[1] += 1
                continue
            st[0] += 1
            self.wellformed[k] = True
            X = self.X0[k]
            fin = np.isfinite(X).all()
            cand = []
            for m in range(lo, hi):
                a, f = int(mem[m, 0]), int(mem[m, 1])
                ok = 0 <= a < S and 0 <= f < len(xy[a]) and np.isfinite(xy[a][f]).all()
                if not ok:
                    st[2] += 1
                    continue
                self.valid[m] = True
                if not fin or (use is not None and not use[m]):
                    continue
                if not (R0[a][2] @ X + t0[a][2] > 0.0):
                    continue
                cand.append((m, a, float(xy[a][f][0]), float(xy[a][f][1])))
            if len(cand) >= 2:
                st[3] += len(cand)
                st[4] += 1
                for m, a, x, y in cand:
                    k_.append(k); a_.append(a); m_.append(m); x_.append(x); y_.append(y)
        self.k, self.a, self.m = np.array(k_, np.int64), np.array(a_, np.int64), np.array(m_, np.int64)
        self.x, self.y = np.array(x_, np.float64), np.array(y_, np.float64)
        self.N = len(self.k)
        self.parts = np.unique(self.k)
        hasobs = np.zeros(S, bool)
        hasobs[self.a] = True
        self.mask = np.array([free_mask(int(self.fixed[a])) & hasobs[a] for a in range(S)]).reshape(S, 6)
        st[5] = int(self.mask.sum())
        self.stats = st
        self.R0, self.t0 = R0, t0

    # ---- residuals and Jacobians ----
    def residuals(self, R, t, X):
        """r [N, 2] and the depth [N]."""
        RX = np.einsum("nij,nj->ni", R[self.a], X[self.k])
        Xc = RX + t[self.a]
        z = Xc[:, 2]
        a, b = Xc[:, 0] / z, Xc[:, 1] / z
        K = self.K[self.a]
        r = np.stack([K[:, 0, 0] * a + K[:, 0, 1] * b + K[:, 0, 2] - self.x, K[:, 1, 1] * b + K[:, 1, 2] - self.y], 1)
        return r, z

    def jacobians(self, R, t, X):
        """J_c [N, 2, 6] (w then delta), J_p [N, 2, 3], r [N, 2]."""
        RX = np.einsum("nij,nj->ni", R[self.a], X[self.k])
        Xc = RX + t[self.a]
        z = Xc[:, 2]
        a, b = Xc[:, 0] / z, Xc[:, 1] / z
        K = self.K[self.a]
        r, _ = self.residuals(R, t, X)
        gx = np.stack([K[:, 0, 0] / z, K[:, 0, 1] / z, -(K[:, 0, 0] * a + K[:, 0, 1] * b) / z], 1)
        gy = np.stack([np.zeros_like(z), K[:, 1, 1] / z, -K[:, 1, 1] * b / z], 1)
        gr = np.stack([gx, gy], 1)                                          # [N, 2, 3]
        Jc = np.concatenate([np.cross(RX[:, None, :], gr), gr], 2)
        Jp = np.einsum("nqi,nij->nqj", gr, R[self.a])
        return Jc, Jp, r

    def cost(self, R, t, X):
        r, z = self.residuals(R, t, X)
        return float((r * r).sum()), bool((z > 0).all())

    # ---- the linear solve ----
    def solve(self, Jc, Jp, r, lam, maxLinear, tol):
        """The Schur + PCG step of the header: (ok, dc [S, 6], dp [T, 3], CG iterations)."""
        S, T = self.S, self.T
        U = np.zeros((S, 6, 6)); gc = np.zeros((S, 6))
        V = np.zeros((T, 3, 3)); gp = np.zeros((T, 3))
        np.add.at(U, self.a, np.einsum("nqi,nqj->nij", Jc, Jc))
        np.add.at(gc, self.a, np.einsum("nqi,nq->ni", Jc, r))
        np.add.at(V, self.k, np.einsum("nqi,nqj->nij", Jp, Jp))
        np.add.at(gp, self.k, np.einsum("nqi,nq->ni", Jp, r))
        Wo = np.einsum("nqi,nqj->nij", Jc, Jp)                              # [N, 6, 3]
        Vi = {}
        for k in self.parts:
            L = chol_ok(damp(V[k], lam))
            if L is None:
                return False, None, None, 0
            Vi[int(k)] = chol_solve(L, np.eye(3))
        q = np.zeros((T, 3))
        for k in self.parts:
            q[k] = Vi[int(k)] @ gp[k]
        rhs = -gc.copy()
        np.add.at(rhs, self.a, np.einsum("nij,nj->ni", Wo, q[self.k]))
        Wak = [{} for _ in range(S)]                                        # per image: track -> W_ak
        for n in range(self.N):
            a, k = int(self.a[n]), int(self.k[n])
            Wak[a][k] = Wak[a].get(k, 0) + Wo[n]
        Us = np.zeros((S, 6, 6)); Ls = []
        for a in range(S):
            m = self.mask[a]
            u = damp(U[a], lam)
            Mb = u.copy()
            for k, w in Wak[a].items():
                Mb -= w @ Vi[k] @ w.T
            fm = np.outer(m, m)
            u = np.where(fm, u, np.eye(6)); Mb = np.where(fm, Mb, np.eye(6))
            L = chol_ok(Mb)
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
            Wy = np.zeros((S, 6))
            np.add.at(Wy, self.a, np.einsum("nij,nj->ni", Wo, y[self.k]))
            return np.where(self.mask, np.einsum("aij,aj->ai", Us, p) - Wy, 0.0)

        def Minv(v):
            return np.array([chol_solve(Ls[a], v[a]) for a in range(S)]).reshape(S, 6)

        x = np.zeros((S, 6)); res = rhs.copy(); z = Minv(res); p = np.zeros((S, 6))
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

    def dense_step(self, Jc, Jp, r, lam):
        """The same step from the full damped normal equations over the free parameters (np.linalg.solve)."""
        S, T = self.S, self.T
        cols = [(a, i) for a in range(S) for i in range(6) if self.mask[a, i]]
        cidx = {c: j for j, c in enumerate(cols)}
        pidx = {int(k): len(cols) + 3 * j for j, k in enumerate(self.parts)}
        n = len(cols) + 3 * len(self.parts)
        J = np.zeros((2 * self.N, n))
        for o in range(self.N):
            a, k = int(self.a[o]), int(self.k[o])
            for i in range(6):
                if self.mask[a, i]:
                    J[2 * o:2 * o + 2, cidx[(a, i)]] = Jc[o, :, i]
            J[2 * o:2 * o + 2, pidx[k]:pidx[k] + 3] = Jp[o]
        H = damp(J.T @ J, lam)
        step = np.linalg.solve(H, -J.T @ r.reshape(-1))
        dc = np.zeros((S, 6)); dp = np.zeros((T, 3))
        for (a, i), j in cidx.items():
            dc[a, i] = step[j]
        for k, j in pidx.items():
            dp[k] = step[j:j + 3]
        return dc, dp

    @staticmethod
    def apply(R, t, mask, dc):
        R1, t1 = R.copy(), t.copy()
        for a in range(len(R)):
            if not mask[a].any():
                continue
            R1[a] = rodrigues(dc[a, :3]) @ R[a]
            t1[a] = np.where(mask[a, 3:], t[a] + dc[a, 3:], t[a])
        return R1, t1

    # ---- the LM loop ----
    def run(self, maxIterations=50, maxLinear=100, tol=1e-6):
        """Returns (R, t, X, cost (initial, final), trace [iterations, 4], accepted, history): history holds per
        iteration the margins of its decisions (for the tests' band)."""
        R, t, X = self.R0.copy(), self.t0.copy(), self.X0.copy()
        cost, _ = self.cost(R, t, X) if self.N else (0.0, True)
        cost0, lam, trace, accepted, self.history = cost, 1e-3, [], 0, []
        for it in range(maxIterations if self.N else 0):
            Jc, Jp, r = self.jacobians(R, t, X)
            ok, dc, dp, cgit = self.solve(Jc, Jp, r, lam, maxLinear, tol)
            cand, behind = np.nan, True
            if ok:
                R1, t1 = self.apply(R, t, self.mask, dc)
                X1 = X.copy()
                X1[self.parts] = X[self.parts] + dp[self.parts]
                cand, front = self.cost(R1, t1, X1)
                behind = not front
            acc = ok and not behind and cand < cost
            trace.append((cand, lam, cgit, float(acc)))
            self.history.append(dict(cost=cost, cand=cand, cg=list(self.cg_history) if ok else []))
            if acc:
                stop = cost - cand <= 1e-10 * cost
                R, t, X, cost, lam = R1, t1, X1, cand, lam / 10.0
                accepted += 1
                if stop:
                    break
            else:
                lam *= 10.0
                if lam > 1e16:
                    break
        return R, t, X, (cost0, cost), np.array(trace).reshape(-1, 4), accepted

    def outputs(self, R, t, X, maxError):
        """errors float32 [M] and inlier [M] for the members of well-formed tracks (others None-marked by -1)."""
        cams = to.Cameras(self.K, R, t)
        err = np.full(self.M, np.nan, np.float32)
        inl = np.zeros(self.M, bool)
        written = np.zeros(self.M, bool)
        for k in range(self.T):
            if not self.wellformed[k]:
                continue
            lo, hi = int(self.offsets[k]), int(self.offsets[k + 1])
            written[lo:hi] = True
            if not np.isfinite(X[k]).all():
                continue
            ms = [m for m in range(lo, hi) if self.valid[m]]
            if not ms:
                continue
            a = self.members[ms, 0]
            xy = np.array([self.xy[int(aa)][int(f)] for aa, f in self.members[ms]], np.float64).reshape(-1, 2)
            i, d, e = to.score(cams, X[k][None], a, xy[:, 0], xy[:, 1], maxError * maxError)
            inl[ms] = i[0]
            with np.errstate(divide="ignore", invalid="ignore"):
                err[ms] = np.where(d[0] > 0, np.sqrt(e[0] / (d[0] * d[0])), np.inf).astype(np.float32)
        return err, inl, written
