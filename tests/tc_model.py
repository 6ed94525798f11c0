"""Restatement of the tensor matcher's certification (csrc/match_tc.cu) in numpy, for both rules it serves.

TEST INFRASTRUCTURE ONLY.  Every quantity is computed the way the kernels compute it:

  * the exact score: the reference's sequential k = 0..127 FP32 FMA chain, each step one correctly rounded fmaf
    (fma32 below: the float64 sum of the exact product and the accumulator, corrected where rounding it twice to FP32
    would differ from rounding once);
  * the split: hi = fp16(2^12 x), lo = fp16(2^12 x - hi), and the approximate score sum hi*hi + hi*lo + lo*hi (in
    float64: every product is exact and the sum's error is far below the budgets here);
  * the row norms and bmax as t3_prep_kernel forms them: per 8-value chunk an fmaf chain from 0, the 16 chunk sums added
    in order, sqrtf, times 1.0001f; bmax the largest norm over the candidate rows;
  * delta = 2 (T3_C1 |a| bmax + T3_C2 (|a| + bmax)) in FP32, as t3_resolve_kernel computes it;
  * per (row, partition) the three largest positive 4-candidate group maxima and the ids of the first two, inserted
    in increasing group order with the epilogue's strict updates;
  * the pools (the reference rule's L = {G[0..7], S[0]}, the top-2 rule's T = {G[0..7], S[0..7]}), rowOk, cert, use1,
    use2, the re-scored candidate list in the kernel's order and the rule applied to their exact scores.

The tensor cores' own accumulation is the adversary: an approximate score may lie anywhere within ACCUM_BUDGET * |a||b|
of the split-FP16 value.  decide() takes one such perturbation; fallback_bounds() gives, for all of them at once, the
interval [rows certainly uncertified, rows possibly uncertified] from the monotone bounds of the tables."""
import numpy as np

T3_C1, T3_C2 = np.float32(4.0e-5), np.float32(1.0e-9)
SCALE = 4096.0
LIMIT = 8.0
ACCUM_BUDGET = 2.0 ** -15          # the share of T3_C1 the comments give the tensor cores' accumulation
T3_MT = T3_N = 128
T3_SEG = 6                         # t3_resolve_kernel: segments fetched unrolled before the loop

F32, F64 = np.float32, np.float64


# ---------------------------------------------------------------------------------------------------- arithmetic
def fma32(a, b, c):
    """fmaf(a, b, c) elementwise on float32 arrays: one rounding.  a*b is exact in float64; where the float64 sum lands
    exactly on a midpoint between two floats while its rounding error e is not zero, the sum is moved one float64 ulp
    toward the true value before the rounding to float32."""
    p = a.astype(F64) * b.astype(F64)
    c64 = c.astype(F64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)                      # TwoSum: s + e == p + c exactly
    r = s.astype(F32)
    rd = r.astype(F64)
    with np.errstate(invalid="ignore", over="ignore"):
        other = np.nextafter(r, np.where(s > rd, F32(np.inf), F32(-np.inf))).astype(F64)
        tie = (s != rd) & (s == (rd + other) * 0.5) & (e != 0)
    if tie.any():
        s = np.where(tie, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def exact_scores(a, b):
    """[len(a), len(b)] FP32 scores of the reference's chain (matching.cu:338-351)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    acc = np.zeros((len(a), len(b)), F32)
    for k in range(128):
        acc = fma32(a[:, k:k + 1], b[None, :, k], acc)
    return acc


def chain_pairs(a, b):
    """The chain for row pairs (a[i], b[i])."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    acc = np.zeros(len(a), F32)
    for k in range(128):
        acc = fma32(a[:, k], b[:, k], acc)
    return acc


def split(x):
    xs = np.asarray(x, F32) * F32(SCALE)
    hi = xs.astype(np.float16)
    lo = (xs - hi.astype(F32)).astype(np.float16)
    return hi, lo


def gated(x):
    """t3_split_chunk's test: a set with a value outside |x| < 8 (NaN, Inf included) takes the exact way."""
    return not bool(np.all(np.abs(np.asarray(x, F32)) < F32(LIMIT)))


def approx_scaled(a, b):
    """sum hi*hi + hi*lo + lo*hi in float64, still scaled by 2^24 (the accumulators' scale)."""
    ah, al = (v.astype(F64) for v in split(a))
    bh, bl = (v.astype(F64) for v in split(b))
    return ah @ bh.T + (ah @ bl.T + al @ bh.T)


def prep_norms(x):
    """The row norms of t3_prep_kernel: fmaf chain per chunk of 8, chunk sums added in order, sqrtf * 1.0001f."""
    x = np.asarray(x, F32)
    t = np.zeros(len(x), F32)
    for c in range(16):
        sq = np.zeros(len(x), F32)
        for i in range(8):
            v = x[:, 8 * c + i]
            sq = fma32(v, v, sq)
        t = (t + sq).astype(F32)
    return (np.sqrt(t).astype(F32) * F32(1.0001)).astype(F32)


def delta32(normA, bmax):
    normA, bmax = np.asarray(normA, F32), F32(bmax)
    eps = (T3_C1 * normA * bmax).astype(F32) + (T3_C2 * (normA + bmax).astype(F32)).astype(F32)
    return (F32(2.0) * eps.astype(F32)).astype(F32)


def eps64(na, nb):
    """The error bound eps = T3_C1 |a||b| + T3_C2 (|a| + |b|) in float64."""
    return float(T3_C1) * na * nb + float(T3_C2) * (na + nb)


# ---------------------------------------------------------------------------------------------------- schedule
def idivup(a, b):
    return -(-a // b)


def t3_schedule(total, sms):
    grid = min(total, sms)
    U = idivup(total, grid)
    return U, idivup(total, U)


def t3_plan(n1, n2v, sms):
    """(n_mt, n_nt, total, U, grid) of one direction, as match_tc.cu's t3_plan."""
    n_mt, n_nt = idivup(n1, T3_MT), idivup(n2v, T3_N)
    total = n_mt * n_nt
    U, grid = t3_schedule(total, sms)
    return n_mt, n_nt, total, U, grid


def segments(n1, n2v, sms):
    """Per row tile the CTAs [c0, c1] whose units it spans (the segments the resolve merges), and whether a CTA
    boundary falls on the tile's end."""
    n_mt, n_nt, total, U, grid = t3_plan(n1, n2v, sms)
    out = []
    for mt in range(n_mt):
        u0, u1 = mt * n_nt, mt * n_nt + n_nt - 1
        out.append((u0 // U, u1 // U, (u1 + 1) % U == 0))
    return out


def b_role_copy(n, nv):
    """t3_setup: a set gets its own B-role copy when its tail rows [nv, n) lie in a tile that the B role reads."""
    return n != nv and nv % T3_N != 0


# ---------------------------------------------------------------------------------------------------- tables
def tables(approx, n2cand):
    """Per (row, partition) G >= S >= Th and the group ids I1, I2 of the epilogue + segment merge, from the scaled
    approximate scores [n1, >= n2cand] (float64; rounded to the FP32 accumulators here).  Candidates from n2cand on are
    the B operand's zero rows: their score is 0 and never enters a table."""
    n1 = approx.shape[0]
    ng = idivup(n2cand, T3_N) * (T3_N // 4)
    v = np.zeros((n1, ng * 4), F64)
    v[:, :n2cand] = approx[:, :n2cand]
    gm = v.astype(F32).reshape(n1, ng, 4).max(-1)
    G = np.zeros((n1, 8), F32); S = np.zeros((n1, 8), F32); Th = np.zeros((n1, 8), F32)
    I1 = np.full((n1, 8), -1, np.int64); I2 = np.full((n1, 8), -1, np.int64)
    gpart = gm.reshape(n1, ng // 8, 8)
    for k in range(ng // 8):
        x = gpart[:, k, :]
        gid = 8 * k + np.arange(8)[None, :]
        t, u2 = x > G, x > S
        Th = np.maximum(Th, np.minimum(S, x))
        I2 = np.where(u2, np.where(t, I1, gid), I2)
        S = np.maximum(S, np.minimum(G, x))
        I1 = np.where(t, gid, I1)
        G = np.maximum(G, x)
    un = F32(1.0 / 16777216.0)
    return G * un, S * un, Th * un, I1, I2


def _second_largest(vals):
    s = np.sort(vals, axis=1)
    return s[:, -1], s[:, -2]


def decide(G, S, Th, I1, I2, delta, knn):
    """(rowOk, cert [n1, 8], use1, use2) of t3_resolve_kernel, in FP32."""
    delta = delta[:, None]
    if knn:
        _, m2 = _second_largest(np.concatenate([G, S], 1))
    else:
        _, m2 = _second_largest(np.concatenate([G, S[:, :1]], 1))
    m2 = m2[:, None]
    rowOk = (m2 > F32(2) * delta) & (m2 < F32(3.0e38))
    if knn:
        low = (m2 - delta).astype(F32)
        cert = (Th <= 0) | (Th < low)
        use1 = rowOk & (I1 >= 0) & (G >= low)
        use2 = rowOk & (I2 >= 0) & (S >= low)
    else:
        rel = rowOk & (G >= (m2 - delta).astype(F32))
        base = np.concatenate([np.minimum(m2, G[:, :1]), G[:, 1:]], 1)
        low = (base - delta).astype(F32)
        cert = ~rel | (Th <= 0) | (Th < low)
        use1 = rel & (I1 >= 0)
        use2 = rel & (I2 >= 0) & (S >= low)
    ok = rowOk[:, 0] & cert.all(1)
    return ok, use1, use2


def candidates(use1, use2, I1, I2, r):
    """The kernel's candidate list of row r: the first groups in partition order, then the second groups."""
    groups = [int(I1[r, p]) for p in range(8) if use1[r, p]] + [int(I2[r, p]) for p in range(8) if use2[r, p]]
    return [4 * g + c for g in groups for c in range(4)]


def rule_ref(cands, ex_row, n2):
    """The reference rule on the re-scored candidates: (score, match, ambiguity) of the per-partition rule and the
    8-way merge (matching.cu:354-359, 378-390)."""
    pmx, psec, pidx = [F32(0)] * 8, [F32(0)] * 8, [-1] * 8
    for p2 in cands:
        sc = ex_row[p2] if p2 < n2 else F32(0)
        p = (p2 >> 2) & 7
        if not sc > 0:
            continue
        if sc > pmx[p]:
            psec[p], pmx[p], pidx[p] = pmx[p], sc, p2
        else:
            if sc == pmx[p] and p2 < pidx[p]:
                pidx[p] = p2
            psec[p] = max(psec[p], sc)
    mx, sec, idx = pmx[0], psec[0], pidx[0]
    for y in range(8):
        if idx != pidx[y]:
            if pmx[y] > mx:
                sec, mx, idx = max(mx, sec), pmx[y], pidx[y]
            elif pmx[y] > sec:
                sec = pmx[y]
    return F32(mx), idx, F32(sec) / (F32(mx) + F32(1e-6))


def rule_knn(cands, ex_row, n2):
    """The top-2 rule: larger score first, then the lower index; only positive scores."""
    s1, j1, s2, j2 = F32(0), -1, F32(0), -1
    for p2 in cands:
        if p2 >= n2:
            continue
        s = ex_row[p2]
        if s > s1 or (s == s1 and p2 < j1):
            s2, j2, s1, j1 = s1, j1, s, p2
        elif s > s2 or (s == s2 and p2 < j2):
            s2, j2 = s, p2
    return (j1, j2), (s1, s2)


class Direction:
    """One direction (rows a against candidates b) under the model: the rule (knn or the reference rule), its
    candidate count (n2v = 32 floor(n2 / 32) for the reference rule, n2 for knn), norms, bmax, delta, the scaled
    approximate scores and the per-pair accumulation budget."""

    def __init__(self, a, b, knn):
        self.a, self.b = np.asarray(a, F32), np.asarray(b, F32)
        self.knn = knn
        self.n1, self.n2 = len(a), len(b)
        self.ncand = self.n2 if knn else (self.n2 // 32) * 32
        bc = self.b[:self.ncand]
        self.normA = prep_norms(self.a)
        self.bmax = F32(prep_norms(bc).max()) if self.ncand else F32(0)
        self.delta = delta32(self.normA, self.bmax)
        self.approx = approx_scaled(self.a, bc) if self.ncand else np.zeros((self.n1, 0))
        na = np.sqrt((self.a.astype(F64) ** 2).sum(1))
        nb = np.sqrt((bc.astype(F64) ** 2).sum(1))
        self.budget = ACCUM_BUDGET * np.outer(na, nb) * 2.0 ** 24

    def perturbations(self, ex=None, seed=0):
        """Admissible accumulator errors: none, all +budget, all -budget, uniform and random-sign draws, and (with the
        exact scores) the exact best candidate of each row pushed down while every other one is pushed up."""
        rng = np.random.default_rng(seed)
        B = self.budget
        out = {"none": 0.0, "up": B, "down": -B, "uniform": rng.uniform(-1, 1, B.shape) * B,
               "sign": np.where(rng.random(B.shape) < 0.5, -B, B)}
        if ex is not None and self.ncand:
            best = np.argmax(ex[:, :self.ncand], 1)
            t = B.copy()
            t[np.arange(self.n1), best] *= -1
            out["against-best"] = t
        return out

    def run(self, pert=0.0):
        """(ok [n1], per row the re-scored candidate list) under one perturbation."""
        G, S, Th, I1, I2 = tables(self.approx + pert, self.ncand)
        ok, use1, use2 = decide(G, S, Th, I1, I2, self.delta, self.knn)
        return ok, [candidates(use1, use2, I1, I2, r) if ok[r] else None for r in range(self.n1)]

    def fallback_bounds(self):
        """[rows uncertified under every admissible perturbation, rows uncertified under some].  G, S and Th are
        monotone in the approximate scores, so the tables of approx -/+ budget bound them; the bounds are padded by
        2^-10 of the budget for the FP32 rounding of the accumulators."""
        if not self.ncand:
            return self.n1, self.n1
        pad = self.budget * (1 + 2.0 ** -10)
        lo = tables(self.approx - pad, self.ncand)[:3]
        hi = tables(self.approx + pad, self.ncand)[:3]
        d = self.delta[:, None]
        two = F32(2)

        def m2_of(G, S):
            pool = np.concatenate([G, S], 1) if self.knn else np.concatenate([G, S[:, :1]], 1)
            return _second_largest(pool)[1][:, None]
        m2lo, m2hi = m2_of(lo[0], lo[1]), m2_of(hi[0], hi[1])
        okSure = (m2lo > two * d) & (m2hi < F32(3.0e38))
        okMaybe = m2hi > two * d
        Glo, Ghi, Thlo, Thhi = lo[0], hi[0], lo[2], hi[2]
        if self.knn:
            certSure = (Thhi <= 0) | (Thhi < (m2lo - d).astype(F32))
            certMaybe = (Thlo <= 0) | (Thlo < (m2hi - d).astype(F32))
        else:
            relNever = ~okMaybe | (Ghi < (m2lo - d).astype(F32))
            relMaybeNot = ~okSure | (Glo < (m2hi - d).astype(F32))
            lowLo = (np.concatenate([np.minimum(m2lo, Glo[:, :1]), Glo[:, 1:]], 1) - d).astype(F32)
            lowHi = (np.concatenate([np.minimum(m2hi, Ghi[:, :1]), Ghi[:, 1:]], 1) - d).astype(F32)
            certSure = relNever | (Thhi <= 0) | (Thhi < lowLo)
            certMaybe = relMaybeNot | (Thlo <= 0) | (Thlo < lowHi)
        sure = okSure[:, 0] & certSure.all(1)
        maybe = okMaybe[:, 0] & certMaybe.all(1)
        return int((~maybe).sum()), int((~sure).sum())
