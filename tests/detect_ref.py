"""Restatement of the detector (FindPointsMultiNew, cudaSiftD.cu:1292-1431) on one pyramid level, vectorised over
pixels and extrema, with the exact set of records a correct kernel may write.

Input: the octave's base level as the pipeline left it (Extractor.read_level) and the octave index of its Laplace
taps (numOctaves - level).  The 7 DoG planes come from oracle.dog, which tests/test_pyramid_gpu.py pins bit for bit.

- Extrema are exact: |c| > thresh and the strict 26-neighbour rule as the reference states it (fminf / fmaxf, so a NaN
  neighbour is ignored), interior pixels only.
- The cap of `limit` extrema per 30x8 cell and scale is exact: extrema are ranked before refinement, column-major with
  rows ascending (cap32.cu).
- The refinement (refine_extremum, sift_arith.cuh) replays every _rn operation in float32; fma32 rounds once.  The
  MUFU results are not reproducible on a CPU, so each one stands for every float32 value within its documented error
  of the exact result:
    __fdividef(x, y)   2 ulp for 2^-126 <= |y| <= 2^126; 0 above; x * (+-inf) or the IEEE quotient below
    exp2f              2 ulp
    powf (d2_pow_table) 4 ulp (2^0 = 1 exactly)
  Everything downstream is replayed once per candidate value (at most 5), so xpos, ypos and sharpness each get an
  exact set of admissible float32 values, scale an exact interval, edgeness an exact set.  A keep decision that a
  MUFU result can tip (the |p| <= 0.5 branch, sc >= lowestScale) makes the extremum "marginal": its record may be
  present or absent and must match one of the outcomes.
"""
import numpy as np

import oracle

F32 = np.float32
D2_STRIP = 244          # CS_D2_STRIP: tested DoG columns per detector strip
D2_LCAP = 510           # candidate list capacity per step (detect2.cu)
D2_KQ = 32              # keypoints parked per item (detect2.cu)
NUM_SCALES = 5
EDGE_LIMIT = F32(10.0)
FACTOR = F32(F32(1.0) / F32(NUM_SCALES))
HS_OF_BATCH = {1: 12, 2: 32, 8: 96}   # rows per detector stream the pipeline picks for a batch (pipeline2.cu)
# (width, height, octaves): the last strip of level 0 has 1, 2, 3, 4, 243 or 244 columns, and of level 1 too; heights
# 193..196 leave 2hs - 1, 2hs, 1 and 2 rows to the last item at every hs; 491 x 195 x 7 octaves ends in a 7 x 3 level,
# 247 x 400 x 7 octaves in a 3 x 6 level (tests/test_detect_cpu.py checks this list against cs_detector_items)
SEAM_SHAPES = [(491, 195, 7), (492, 196, 5), (493, 193, 5), (494, 194, 5), (489, 195, 5), (490, 196, 5),
               (496, 193, 5), (498, 194, 5), (500, 195, 5), (247, 400, 7)]
ULP_FDIVIDEF, ULP_EXP2F, ULP_POWF = 2, 2, 4


# ------------------------------------------------------------------------------------------------------- arithmetic
def f32(x):
    return np.asarray(x, np.float64).astype(np.float32)


def fma32(a, b, c):
    """float32 fma with one rounding: the float64 product of two float32 values is exact; the float64 sum may round,
    and TwoSum recovers its error, which decides a float32 tie that the float64 rounding created."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bp = s - c
        e = (p - bp) + (c - (s - bp))              # p + c = s + e exactly (finite s)
        r = s.astype(np.float32)
        r64 = r.astype(np.float64)
        fin = np.isfinite(s) & np.isfinite(r64) & (e != 0)
        other = np.nextafter(r, np.where(s > r64, F32(np.inf), F32(-np.inf)).astype(np.float32))
        tie = fin & (r64 != s) & (s == 0.5 * (r64 + other.astype(np.float64)))
        # s is a float32 midpoint only because the float64 sum rounded: the exact sum lies on e's side of it
        r = np.where(tie, np.where(e > 0, np.maximum(r, other), np.minimum(r, other)), r)
    return r.astype(np.float32)


def _ulp_of(r):
    """Spacing of float32 at the exact value r (float64): 2^(e-23) for |r| in [2^e, 2^(e+1))."""
    m, e = np.frexp(np.abs(r))
    return np.ldexp(1.0, np.maximum(e - 24, -149))


def mufu(r, ulps):
    """(..., 2*ulps+3) float32 values within `ulps` ulp of the exact result r (float64): the admissible results of a
    MUFU-based function.  Slots outside the bound repeat the rounded value; a non-finite r gives itself."""
    r = np.asarray(r, np.float64)
    f = r.astype(np.float32)
    out = [f]
    up, dn = f.copy(), f.copy()
    for _ in range(ulps + 1):
        up = np.nextafter(up, F32(np.inf))
        dn = np.nextafter(dn, F32(-np.inf))
        out += [up, dn]
    c = np.stack(out, -1)
    with np.errstate(invalid="ignore"):
        ok = np.abs(c.astype(np.float64) - r[..., None]) <= ulps * _ulp_of(r)[..., None]
    ok &= np.isfinite(c)
    c = np.where(ok | ~np.isfinite(r)[..., None], c, f[..., None])
    return np.where(np.isfinite(r)[..., None], c, f[..., None]).astype(np.float32)


def fdividef(x, y):
    """Admissible results of __fdividef(x, y), elementwise over float32 arrays: (..., 7)."""
    x = np.asarray(x, np.float32)
    y = np.asarray(y, np.float32)
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        c = mufu(x64 / y64, ULP_FDIVIDEF)
        ay = np.abs(y64)
        huge = ay > 2.0 ** 126
        tiny = ay < 2.0 ** -126
        # |y| > 2^126: 0 (a NaN or infinite x: NaN).  |y| < 2^-126: the reciprocal flushes to +-inf (x * inf), or the
        # IEEE quotient.
        zero = np.where(np.isfinite(x), F32(0.0) * np.sign(x) * np.sign(y), F32(np.nan)).astype(np.float32)
        c = np.where(huge[..., None], zero[..., None], c)
        rinf = (x * (F32(1.0) / np.where(y == 0, y, F32(0.0) * np.sign(y)).astype(np.float32))).astype(np.float32)
        ieee = (x / y).astype(np.float32)
        alt = np.stack([rinf, ieee] + [ieee] * (c.shape[-1] - 2), -1)
        c = np.where(tiny[..., None], alt, c)
    return c.astype(np.float32)


def exp2f(x):
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore"):
        return mufu(np.exp2(x.astype(np.float64)), ULP_EXP2F)


def pow_table():
    """Admissible d2_pow_table[s] = powf(2, s / 5f): (5, 11) float32."""
    e = f32(np.arange(NUM_SCALES, dtype=np.float32) / F32(NUM_SCALES)).astype(np.float64)
    t = mufu(np.exp2(e), ULP_POWF)
    t[0] = F32(1.0)
    return t


# ---------------------------------------------------------------------------------------------------------- extrema
def dog_planes(level, numOctaves, lev_index):
    return oracle.dog(level, numOctaves, numOctaves - lev_index)


def extrema(dog, thresh):
    """Boolean (5, h, w): the reference's extrema of DoG planes 1..5 (scale 0..4), interior pixels only."""
    _, h, w = dog.shape
    ext = np.zeros((NUM_SCALES, h, w), bool)
    if h < 3 or w < 3:
        return ext
    thresh = F32(thresh)
    for s in range(NUM_SCALES):
        c = dog[s + 1, 1:h - 1, 1:w - 1]
        mn = np.full(c.shape, np.inf, np.float32)
        mx = np.full(c.shape, -np.inf, np.float32)
        for p in range(3):
            for dy in range(3):
                for dx in range(3):
                    if p == 1 and dy == 1 and dx == 1:
                        continue
                    v = dog[s + p, dy:dy + h - 2, dx:dx + w - 2]
                    mn = np.fmin(mn, v)
                    mx = np.fmax(mx, v)
        with np.errstate(invalid="ignore"):
            ext[s, 1:h - 1, 1:w - 1] = (c < np.fmin(-thresh, mn)) | (c > np.fmax(thresh, mx))
    return ext


def cap(scale, gy, gx, limit):
    """Keep mask of the cap: rank < limit per (scale, 30x8 cell), ranked column-major with rows ascending."""
    if len(gx) == 0:
        return np.zeros(0, bool)
    cell = (scale.astype(np.int64) * (1 << 20) + (gy >> 3)) * (1 << 20) + gx // 30
    order = np.lexsort((gy, gx, cell))
    cs = cell[order]
    start = np.r_[0, np.nonzero(np.diff(cs))[0] + 1]
    first = np.repeat(start, np.diff(np.r_[start, len(cs)]))
    rank = np.empty(len(gx), np.int64)
    rank[order] = np.arange(len(gx)) - first
    return rank < limit


def flags(dog, thresh):
    """The detector's candidate flags (5, h, w): |c| > thresh, and for columns 1..6 of a lane's 8 (dc = gx - x0 of the
    strip), a sign-wise win over the left and right neighbours.  Only their counts per step are used (list overflow)."""
    _, h, w = dog.shape
    thresh = F32(thresh)
    c = dog[1:6]
    with np.errstate(invalid="ignore"):
        f = np.abs(c) > thresh
        l = np.concatenate([c[:, :, :1], c[:, :, :-1]], 2)
        r = np.concatenate([c[:, :, 1:], c[:, :, -1:]], 2)
        win = np.where(c > 0, (c > l) & (c > r), (c < l) & (c < r))
    gx = np.arange(w)
    dc = np.where(gx >= 1, (gx - 1) % D2_STRIP + 1, 0)
    d = dc % 8
    inner = (d >= 1) & (d <= 6)
    return f & (win | ~inner[None, None, :])


# ------------------------------------------------------------------------------------------------------- refinement
def _gather(dog, s, y, x):
    v = np.empty((3, 3, 3, len(x)), np.float32)
    for p in range(3):
        for dy in range(3):
            for dx in range(3):
                v[p, dy, dx] = dog[s + p, y + dy - 1, x + dx - 1]
    return v


def refine(dog, s, gy, gx, lowestScale):
    """The admissible outcomes of refine_extremum for extrema at (scale s, gy, gx).  Returns a dict of arrays over
    the extrema: must (kept under every admissible MUFU result), may (kept under some), edge (N, 7) set, and per
    branch b in (newton, fallback): ok_b (branch possible and kept under some result), x_b / y_b / sharp_b value sets,
    scale interval lo_b / hi_b."""
    n = len(gx)
    v = _gather(dog, s, gy, gx)
    with np.errstate(all="ignore"):
        val = v[1, 1, 1]
        two = val + val
        dxx = (two - v[1, 1, 0]) - v[1, 1, 2]
        dyy = (two - v[1, 0, 1]) - v[1, 2, 1]
        dxy = F32(0.25) * (((v[1, 2, 2] + v[1, 0, 0]) - v[1, 0, 2]) - v[1, 2, 0])
        tra = dxx + dyy
        det = fma32(dxx, dyy, -(dxy * dxy))
        tra2 = tra * tra
        edge_ok = tra2 < EDGE_LIMIT * det
        edge = fdividef(tra2, det)
        dx = F32(0.5) * (v[1, 1, 2] - v[1, 1, 0])
        dy = F32(0.5) * (v[1, 2, 1] - v[1, 0, 1])
        ds = F32(0.5) * (v[0, 1, 1] - v[2, 1, 1])
        dss = (two - v[2, 1, 1]) - v[0, 1, 1]
        dxs = F32(0.25) * (((v[2, 1, 2] + v[0, 1, 0]) - v[0, 1, 2]) - v[2, 1, 0])
        dys = F32(0.25) * (((v[2, 2, 1] + v[0, 0, 1]) - v[2, 0, 1]) - v[0, 2, 1])
        idxx = fma32(dyy, dss, -(dys * dys))
        idxy = fma32(dys, dxs, -(dxy * dss))
        idxs = fma32(dxy, dys, -(dyy * dxs))
        det3 = fma32(idxs, dxs, fma32(idxx, dxx, idxy * dxy))
        idet = fdividef(F32(1.0), det3)                                  # (N, K)
        idyy = fma32(dxx, dss, -(dxs * dxs))
        idys = fma32(dxy, dxs, -(dxx * dys))
        idss = det
        C = lambda a: a[:, None]
        pdx = idet * C(fma32(ds, idxs, fma32(dx, idxx, dy * idxy)))
        pdy = idet * C(fma32(ds, idys, fma32(dy, idyy, dx * idxy)))
        pds = idet * C(fma32(idss, ds, fma32(dx, idxs, dy * idys)))
        out_ = (pdx < -0.5) | (pdx > 0.5) | (pdy < -0.5) | (pdy > 0.5) | (pds < -0.5) | (pds > 0.5)
        P = pow_table()[s]                                               # (N, T)
        L = F32(lowestScale)

        def scales(pds_):
            """sc for every pds value, exp2f and pow result: (N, ...) -> min, max over the result axes, and
            whether sc >= lowestScale always / ever holds, per pds value."""
            e = exp2f(pds_ * FACTOR)                                     # (N, K, J)
            sc = P[:, None, None, :] * e[..., None]                      # (N, K, J, T)
            sc = sc.reshape(sc.shape[0], sc.shape[1], sc.shape[2] * sc.shape[3])
            return np.min(sc, -1), np.max(sc, -1), np.all(sc >= L, -1), np.any(sc >= L, -1)

        gxf, gyf = C(gx.astype(np.float32)), C(gy.astype(np.float32))
        # Newton branch: candidate k where no |p| > 0.5
        newton_k = ~out_
        lo_n, hi_n, all_n, any_n = scales(pds)
        dsum = fma32(C(ds), pds, fma32(C(dx), pdx, C(dy) * pdy))
        res = dict(edge=edge, edge_ok=edge_ok, newton_k=newton_k,
                   x_n=(gxf + pdx).astype(np.float32), y_n=(gyf + pdy).astype(np.float32),
                   sharp_n=fma32(dsum, F32(0.5), C(val)), lo_n=lo_n, hi_n=hi_n, keep_n_all=all_n, keep_n_any=any_n)
        # fallback branch: pdx, pdy, pds each over their own admissible quotients
        fx, fy, fs = fdividef(dx, dxx), fdividef(dy, dyy), fdividef(ds, dss)
        K = fx.shape[1]
        a_, b_, c_ = (np.arange(K ** 3) // K ** 2, (np.arange(K ** 3) // K) % K, np.arange(K ** 3) % K)
        dsum_f = fma32(C(ds), fs[:, c_], fma32(C(dx), fx[:, a_], C(dy) * fy[:, b_]))
        lo_f, hi_f, all_f, any_f = scales(fs)
        res.update(x_f=(gxf + fx).astype(np.float32), y_f=(gyf + fy).astype(np.float32),
                   sharp_f=fma32(dsum_f, F32(0.5), C(val)), lo_f=lo_f.min(1), hi_f=hi_f.max(1),
                   keep_f_all=all_f.all(1), keep_f_any=any_f.any(1))
        may_newton = edge_ok & newton_k.any(1)
        may_fallback = edge_ok & out_.any(1)
        ok_n = may_newton & (newton_k & any_n).any(1)
        ok_f = may_fallback & res["keep_f_any"]
        must = edge_ok & ~(newton_k & ~all_n).any(1) & ~(out_.any(1) & ~res["keep_f_all"])
        res.update(ok_n=ok_n, ok_f=ok_f, may=ok_n | ok_f, must=must,
                   marginal=(ok_n | ok_f) & ~must | (ok_n & ok_f & (newton_k.any(1) & out_.any(1))))
    return res


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def _member(got, cand):
    """Per row: is got (N,) bit-equal to one of cand (N, K)?"""
    return (_bits(cand) == _bits(got)[:, None]).any(1)


def admissible(r, i, rec):
    """Per record: do its fields lie in the admissible sets of extremum i (index arrays into refine's result) under
    one branch?  rec: level-coordinate fields x, y, scale, sharpness, edgeness (float32 arrays)."""
    x, y, sc, sh, ed = (np.asarray(rec[k], np.float32) for k in ("x", "y", "scale", "sharpness", "edgeness"))
    ok_e = _member(ed, r["edge"][i])
    nk = r["newton_k"][i] & r["keep_n_any"][i]
    same = lambda a, g: (_bits(a[i]) == _bits(g)[:, None])
    with np.errstate(invalid="ignore"):
        in_sc = (sc[:, None] >= r["lo_n"][i]) & (sc[:, None] <= r["hi_n"][i])
    ok_n = r["ok_n"][i] & (nk & same(r["x_n"], x) & same(r["y_n"], y) & same(r["sharp_n"], sh) & in_sc).any(1)
    with np.errstate(invalid="ignore"):
        in_f = (sc >= r["lo_f"][i]) & (sc <= r["hi_f"][i])
    ok_f = (r["ok_f"][i] & _member(x, r["x_f"][i]) & _member(y, r["y_f"][i]) & _member(sh, r["sharp_f"][i]) & in_f)
    return ok_e & (ok_n | ok_f)


def widest_ulp(r, idx):
    """Widest admissible scale interval of the extrema idx, in ulp of the scale."""
    if len(idx) == 0:
        return 0.0
    with np.errstate(invalid="ignore"):
        lo = np.where(r["newton_k"][idx], r["lo_n"][idx], np.inf).min(1)
        hi = np.where(r["newton_k"][idx], r["hi_n"][idx], -np.inf).max(1)
        lo = np.where(r["ok_f"][idx], np.minimum(lo, r["lo_f"][idx]), lo)
        hi = np.where(r["ok_f"][idx], np.maximum(hi, r["hi_f"][idx]), hi)
        w = (hi.astype(np.float64) - lo) / _ulp_of(hi.astype(np.float64))
    w = w[np.isfinite(w)]
    return float(w.max(initial=0.0))


# ------------------------------------------------------------------------------------------------------------ level
class Level:
    """The restatement on one level: the extrema, the capped set, and the admissible records.

    ext_*: every extremum (scale, gy, gx); kept: the cap's mask over them; r: refine() over the kept extrema;
    must / may / marginal over the kept extrema."""

    def __init__(self, level, numOctaves, lev_index, thresh, lowestScale=0.0, limit=32, want_flags=False):
        self.lev_index = lev_index
        self.h, self.w = level.shape
        dog = dog_planes(level, numOctaves, lev_index)
        ext = extrema(dog, thresh)
        s, gy, gx = np.nonzero(ext)
        self.n_extrema = len(gx)
        keep = cap(s, gy, gx, limit)
        self.dropped = int((~keep).sum())
        self.s, self.gy, self.gx = s[keep], gy[keep], gx[keep]
        self.r = refine(dog, self.s, self.gy, self.gx, lowestScale)
        self.must, self.may, self.marginal = self.r["must"], self.r["may"], self.r["marginal"]
        self.flags = flags(dog, thresh) if want_flags else None

    def key(self):
        return (self.s.astype(np.int64) << 40) | (self.gy.astype(np.int64) << 20) | self.gx

    def check(self, scale, gy, gx, rec, exact_set=True):
        """Records with decoded integer positions against the restatement.  exact_set: the decoded set must be the
        kept set up to marginal extrema (False: a subset, e.g. under a maxPts clamp).  Returns statistics."""
        key = (np.asarray(scale, np.int64) << 40) | (np.asarray(gy, np.int64) << 20) | np.asarray(gx, np.int64)
        assert len(np.unique(key)) == len(key), "two records of one extremum"
        mine = self.key()
        order = np.argsort(mine)
        pos = np.searchsorted(mine[order], key)
        pos = np.minimum(pos, max(len(mine) - 1, 0))
        found = (len(mine) > 0) & (mine[order][pos] == key) if len(key) else np.zeros(0, bool)
        assert found.all(), ("records at non-extrema or capped extrema", np.nonzero(~found)[0][:5],
                             np.asarray(gx)[~found][:5], np.asarray(gy)[~found][:5], np.asarray(scale)[~found][:5])
        idx = order[pos]
        assert self.may[idx].all(), ("records of rejected extrema", idx[~self.may[idx]][:5])
        if exact_set:
            hit = np.zeros(len(mine), bool)
            hit[idx] = True
            miss = self.must & ~hit
            assert not miss.any(), ("kept extrema without a record", self.gx[miss][:5], self.gy[miss][:5],
                                    self.s[miss][:5])
        ok = admissible(self.r, idx, rec)
        assert ok.all(), ("fields outside the admissible sets", np.nonzero(~ok)[0][:5],
                          {k: np.asarray(v)[~ok][:3] for k, v in rec.items()})
        return dict(records=len(idx), marginal=int(self.marginal.sum()), widest_ulp=widest_ulp(self.r, idx))

    def locate(self, rec):
        """(scale, gy, gx) of records without a tag (the oracle's, the round-1 kernels'): the extremum whose admissible
        sets hold the record; -1 where none does."""
        x, y = _bits(rec["x"]), _bits(rec["y"])
        table = {}
        r = self.r
        for i in np.nonzero(self.may)[0]:
            pairs = set(zip(_bits(r["x_n"][i]).tolist(), _bits(r["y_n"][i]).tolist()))
            pairs |= {(a, b) for a in _bits(r["x_f"][i]).tolist() for b in _bits(r["y_f"][i]).tolist()}
            for p in pairs:
                table.setdefault(p, []).append(i)
        out = np.full(len(x), -1, np.int64)
        for j, p in enumerate(zip(x.tolist(), y.tolist())):
            for i in table.get(p, []):
                one = {k: np.asarray(v)[j:j + 1] for k, v in rec.items()}
                if admissible(r, np.array([i]), one)[0]:
                    out[j] = i
                    break
        ok = out >= 0
        i = np.maximum(out, 0)
        return np.where(ok, self.s[i], -1), np.where(ok, self.gy[i], -1), np.where(ok, self.gx[i], -1)

    def step_stats(self, hs):
        """Per detector item and step of this level (items as build_detector_items makes them for one image): the
        largest number of flagged (pixel, scale) pairs in one step, and the largest number of keypoints (may) in one
        item."""
        h, w = self.h, self.w
        if w < 3 or h < 3:
            return 0, 0
        strips = -(-(w - 2) // D2_STRIP)
        rows = h - 2
        fl = self.flags.sum(0)                                            # (h, w)
        cum = np.concatenate([np.zeros((h, 1), np.int64), np.cumsum(fl, 1)], 1)
        kx = self.gx[self.may]
        ky = self.gy[self.may]
        max_flag = max_kp = 0
        for r0 in range(0, rows, 2 * hs):
            ry0 = 1 + r0
            left = rows - r0
            hsi = hs if left >= 2 * hs else (left + 1) // 2
            for st in range(strips):
                x0 = st * D2_STRIP
                a, b = x0 + 1, min(x0 + D2_STRIP, w - 2)
                per_row = cum[:, b + 1] - cum[:, a]
                for k in range(1, hsi + 1):
                    ya, yb = ry0 - 1 + k, ry0 + hsi - 1 + k
                    c = (per_row[ya] if ya <= h - 2 else 0) + (per_row[yb] if yb <= h - 2 else 0)
                    max_flag = max(max_flag, int(c))
                inx = (kx >= a) & (kx <= b) & (ky >= ry0) & (ky <= min(ry0 + 2 * hsi - 1, h - 2))
                max_kp = max(max_kp, int(inx.sum()))
        return max_flag, max_kp
