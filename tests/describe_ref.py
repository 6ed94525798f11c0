"""Float64 restatement of the describe stage (cudasift_b200/csrc/describe.cu, describe_kernel), vectorised over
keypoints, with the decision margins and error bounds a test needs to tell a real disagreement from rounding.

Input: one pyramid level (float32, h x w) and keypoints in level coordinates (px, py, pscale), as the detector
leaves them.  What is float32 in the kernel and decides a discrete outcome is computed in float32, op for op: the
sample coordinates, fast_atan2, angf and angi (so quirks Q21 and Q22 come out as the kernel's).  Weights, histograms,
votes and normalisations are float64.

Texture fetches follow oracle_tex2d (oracle/sift_oracle.c): 1.8 fixed point, clamp addressing, exact weighted sum
rounded once.  tests/test_tex_gpu.py pins that rule to the hardware up to the final rounding of the fetched value, so
every fetch is allowed one ulp of its value.

__sinf / __cosf (MUFU) are not reproducible on a CPU.  CUDA documents an absolute error of at most 2^-21.41 on
[-pi, pi]; theta = orientation * 2*3.1415/360 lies in [0, 2*pi), where the hardware's range reduction (a float32
multiply by 1/(2*pi)) adds at most 2^-22.  SIN_ERR = 2^-20 bounds both.  Propagated through the sample-coordinate
formula it gives, per fetch, how far the GPU's coordinate can be from ours; a fetch whose fixed-point coordinate lies
closer than that to a 1/256 grid line is "grid-ambiguous", and the value one grid step over bounds what it can read.
"""
import numpy as np

U = 2.0 ** -24                 # float32 unit roundoff
SIN_ERR = 2.0 ** -20           # |__sinf(t) - sin(t)|, |__cosf(t) - cos(t)| for t in [0, 2*pi), see above
ATAN_SLACK = 4e-6              # rad: fast_atan2 rounding jitter under a perturbed input (16 ulp of pi)
BIN_SLACK = 1e-5               # 16*atan2f/3.1416 + 16.5 in float32 (atan2f 2 ulp, three roundings) vs float64
F32 = np.float32
PI_Q14 = float(F32(3.1416))    # quirk Q14: the orientation bin uses 3.1416 (float32 constant)
THETA_K = F32(F32(F32(2.0) * F32(3.1415)) / F32(360.0))
ANGF_K = F32(F32(4.0) / F32(3.1415))
R32 = 1.0 / np.sqrt(128.0)


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32)


def fma32(a, b, c):
    """float32 fma: exact float64 product and sum, one rounding to float32."""
    return f32(np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64))


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


# ------------------------------------------------------------------------------------------------------------ texture
def _fixed(c):
    """1.8 fixed-point coordinate floor((c - 0.5) * 256 + 0.5) as float64, and the distance of the unrounded value to
    the grid line below it (lo) and above it (hi), in 1/256 texel units."""
    r = (np.asarray(c, np.float32).astype(np.float64) - 0.5) * 256.0 + 0.5
    F = np.floor(r)
    bad = ~((F > -1.0e9) & (F < 1.0e9))            # NaN / huge coordinates read as 0 (oracle_tex2d)
    F = np.where(bad, 0.0, F)
    lo = np.where(bad, np.inf, r - F)
    hi = np.where(bad, np.inf, F + 1.0 - r)
    return F, lo, hi


def _tex_fixed(img, FX, FY):
    h, w = img.shape
    i0 = np.floor(FX / 256.0)
    j0 = np.floor(FY / 256.0)
    A = (FX - i0 * 256.0).astype(np.int64)
    B = (FY - j0 * 256.0).astype(np.int64)
    i0 = i0.astype(np.int64)
    j0 = j0.astype(np.int64)
    i1 = np.clip(i0 + 1, 0, w - 1)
    j1 = np.clip(j0 + 1, 0, h - 1)
    i0 = np.clip(i0, 0, w - 1)
    j0 = np.clip(j0, 0, h - 1)
    w11 = (A * B + 128) >> 8
    w10, w01 = A - w11, B - w11
    w00 = 256 - A - B + w11
    im = img.astype(np.float64)
    t00, t10, t01, t11 = im[j0, i0], im[j0, i1], im[j1, i0], im[j1, i1]
    s = w00 * t00 + w10 * t10 + w01 * t01 + w11 * t11
    return f32(s * (1.0 / 256.0)), (t00 == t10) & (t00 == t01) & (t00 == t11)


def tex2d(img, x, y):
    """oracle_tex2d, vectorised: float32 coordinates in, float32 values out."""
    FX, _, _ = _fixed(x)
    FY, _, _ = _fixed(y)
    return _tex_fixed(img, FX, FY)[0]


def tex2d_bounded(img, x, y, dcx, dcy=None):
    """(value, bound, ambiguous, rounding part of bound): bound covers coordinates off by up to dcx / dcy pixels
    (one fixed-point step at most) plus one ulp of the fetched value (the hardware's final rounding; none when the four texels are equal, as the
    exact result is then a texel value)."""
    FX, lox, hix = _fixed(x)
    FY, loy, hiy = _fixed(y)
    v, const = _tex_fixed(img, FX, FY)
    ux = np.broadcast_to(np.asarray(dcx, np.float64) * 256.0, FX.shape)
    uy = ux if dcy is None else np.broadcast_to(np.asarray(dcy, np.float64) * 256.0, FY.shape)
    assert np.all(ux < 0.5) and np.all(uy < 0.5), "coordinate uncertainty reaches a whole fixed-point step"
    sx = np.where(lox < ux, -1.0, np.where(hix < ux, 1.0, 0.0))
    sy = np.where(loy < uy, -1.0, np.where(hiy < uy, 1.0, 0.0))
    amb = (sx != 0) | (sy != 0)
    bound = np.where(const, 0.0, ulp32(v))
    rbound = bound.copy()
    if amb.any():
        idx = np.nonzero(amb)
        fx, fy, ax, ay, v0 = FX[idx], FY[idx], sx[idx], sy[idx], v[idx].astype(np.float64)
        dmax = np.zeros(len(fx))
        for mx, my in ((1, 0), (0, 1), (1, 1)):
            alt = _tex_fixed(img, fx + mx * ax, fy + my * ay)[0].astype(np.float64)
            dmax = np.maximum(dmax, np.abs(alt - v0) + ulp32(alt))
        bound[idx] += dmax
    return v, bound, amb, rbound


# -------------------------------------------------------------------------------------------------------- orientation
def _smooth(h):
    return 6.0 * h + 4.0 * (np.roll(h, 1, -1) + np.roll(h, -1, -1)) + (np.roll(h, 2, -1) + np.roll(h, -2, -1))


def _interp(sm, b):
    """Orientation in degrees of a peak at bin b (parabolic interpolation, describe.cu:143-145)."""
    n = np.arange(sm.shape[0])
    v1, v2, m = sm[n, (b + 1) & 31], sm[n, (b + 31) & 31], sm[n, b]
    with np.errstate(invalid="ignore", divide="ignore"):
        peak = b + 0.5 * (v1 - v2) / ((2.0 * m - v1) - v2)
    return 11.25 * np.where(peak < 0.0, peak + 32.0, peak), (2.0 * m - v1) - v2


def orientations(img, px, py, pscale):
    """Orientation histogram, peaks and secondaries of describe_kernel for keypoints at (px, py, pscale).

    Returns a dict of arrays over keypoints:
      sm (N, 32)          smoothed histogram (float64)
      tol (N, 32)         bound on |sm_gpu - sm| (float32 arithmetic, texture rounding, samples near a bin edge)
      ori (N, 32)         interpolated orientation (degrees) if bin b were the peak; ori_tol its bound
      ori1, ori2, has2    the float64 decision (ori2 NaN without a secondary; Q1 is the caller's)
      cand1, cand2 (N,32) bins that can be the primary / secondary peak within tol
      has2_certain        the secondary decision holds for every sm within tol
      near_tie            more than one primary candidate, or an uncertain / ambiguous secondary
      bin_margin (N,121)  distance of 16*atan2/3.1416 + 16.5 from an integer, per sample
      peak_gap            best peak - runner-up;  ratio_margin  maxval2 / maxval1 - 0.8
      peak_cmp (N, 2, 2)  sm - smm and sm - smp at the chosen peaks (the `sm > smm && sm >= smp` test)
    """
    px = np.asarray(px, np.float32)
    py = np.asarray(py, np.float32)
    ps = np.asarray(pscale, np.float32)
    N = len(px)
    k = np.arange(121)
    yd, xd = k // 11, k % 11
    xf = f32(xd[None, :] + f32(px[:, None].astype(np.float64) - 4.5))
    yf = f32(yd[None, :] + f32(py[:, None].astype(np.float64) - 4.5))
    one = np.float32(1.0)
    ax, ea, _, _ = tex2d_bounded(img, f32(xf + one), yf, 0.0)
    bx, eb, _, _ = tex2d_bounded(img, f32(xf - one), yf, 0.0)
    cy, ec, _, _ = tex2d_bounded(img, xf, f32(yf + one), 0.0)
    dy_, ed, _, _ = tex2d_bounded(img, xf, f32(yf - one), 0.0)
    dx = f32(ax.astype(np.float64) - bx).astype(np.float64)
    dy = f32(cy.astype(np.float64) - dy_).astype(np.float64)
    eps = np.maximum(ea + eb, ec + ed)
    t = 16.0 * np.arctan2(dy, dx) / PI_Q14 + 16.5
    binv = np.trunc(t).astype(np.int64)
    binv[binv > 31] = 0
    binv[binv < 0] = 0
    frac = t - np.floor(t)
    bin_margin = np.minimum(frac, 1.0 - frac)
    grad = np.sqrt(dx * dx + dy * dy)
    i2s = -1.0 / (4.5 * ps.astype(np.float64) ** 2)
    g11 = np.exp(((np.arange(11) - 5.0) ** 2)[None, :] * i2s[:, None])
    gw = g11[:, xd] * g11[:, yd]
    wts = grad * gw
    # a sample whose bin the GPU may decide differently: within BIN_SLACK, or within reach of the texture rounding
    with np.errstate(divide="ignore", invalid="ignore"):
        dang = np.where(grad > 2.0 * eps, 1.5 * eps / np.maximum(grad - 1.5 * eps, 1e-300), np.inf)
    amb = bin_margin < BIN_SLACK + 16.0 / PI_Q14 * dang
    flat = (np.arange(N)[:, None] * 32 + binv).ravel()
    hist = np.bincount(flat, wts.ravel(), minlength=N * 32).reshape(N, 32)
    sm = _smooth(hist)
    werr = (gw * 1.5 * eps).sum(1) + (wts * amb).sum(1)                    # weight a sample may gain, lose or move
    tol = 64.0 * U * sm + 16.0 * werr[:, None] + 1e-30
    smm, smp = np.roll(sm, 1, -1), np.roll(sm, -1, -1)
    tm, tp = np.roll(tol, 1, -1), np.roll(tol, -1, -1)
    is_peak = (sm > smm) & (sm >= smp)
    may_peak = (sm + tol > smm - tm) & (sm + tol >= smp - tp)
    sure_peak = (sm - tol > smm + tm) & (sm - tol >= smp + tp)
    pk = np.where(is_peak, sm, 0.0)
    order = np.argsort(-pk, axis=1, kind="stable")           # ties: lowest index first
    i1, i2 = order[:, 0], order[:, 1]
    n = np.arange(N)
    m1, m2 = pk[n, i1], pk[n, i2]
    has1 = m1 > 0.0
    i1 = np.where(has1, i1, -1)
    m2 = np.where(m2 > 0.0, m2, 0.0)
    i2 = np.where(m2 > 0.0, i2, -1)
    has2 = m2 > 0.8 * np.where(has1, m1, 0.0)
    ori = np.empty((N, 32))
    den = np.empty((N, 32))
    for b in range(32):
        ori[:, b], den[:, b] = _interp(sm, np.full(N, b))
    # |d peak| <= 4 T / d for sm errors T (|peak offset| <= 1/2 and d = 2m - v1 - v2 >= |v1 - v2|), plus the
    # float32 roundings of the offset, of i + offset (ulp(32)) and of 11.25 * peak (ulp(360))
    T = np.maximum(np.maximum(tol, tm), tp)
    with np.errstate(divide="ignore", invalid="ignore"):
        ori_tol = 11.25 * (4.0 * T / np.maximum(den - 4.0 * T, 1e-300) + 4.0 * 2.0 ** -19) + 2.0 ** -14
    ori_tol = np.where(den > 4.0 * T, ori_tol, np.inf)
    lo = np.where(sure_peak, sm - tol, -np.inf)
    hi = np.where(may_peak, sm + tol, -np.inf)
    los, his = -np.sort(-lo, 1), -np.sort(-hi, 1)
    m1_lo, m1_hi, m2_lo, m2_hi = los[:, 0], his[:, 0], los[:, 1], his[:, 1]
    cand1 = may_peak & (hi >= m1_lo[:, None])
    cand2 = may_peak & (hi >= m2_lo[:, None])
    # the secondary is never the primary's bin: exclude it unless the primary is itself a near-tie
    cand2 &= ~(cand1 & (cand1.sum(1) == 1)[:, None])
    sure2 = m2_lo > 0.8 * m1_hi * (1 + 4 * U)
    sure_not2 = m2_hi < 0.8 * m1_lo * (1 - 4 * U)
    # a window without any peak (all sm equal, e.g. exactly flat): the kernel gives NaN, no secondary
    flat_win = (sm.max(1) == 0.0) & (werr == 0.0)
    sure_not2 |= flat_win
    ori1 = np.where(has1, ori[n, np.maximum(i1, 0)], np.nan)
    ori2 = np.where(has2, ori[n, np.maximum(i2, 0)], np.nan)
    has2_certain = sure2 | sure_not2
    near_tie = (cand1.sum(1) > 1) | ~has2_certain | (has2 & (cand2.sum(1) > 1))
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio_margin = np.where(m1 > 0, m2 / m1 - 0.8, -0.8)
    cmp = np.stack([np.stack([sm[n, j] - smm[n, j], sm[n, j] - smp[n, j]], 1)
                    for j in (np.maximum(i1, 0), np.maximum(i2, 0))], 1)
    return dict(sm=sm, tol=tol, ori=ori, ori_tol=ori_tol, ori1=ori1, ori2=ori2, has1=has1, has2=has2, i1=i1, i2=i2,
                cand1=cand1, cand2=cand2, has2_certain=has2_certain, near_tie=near_tie, flat=flat_win,
                bin_margin=bin_margin, peak_gap=m1 - m2, ratio_margin=ratio_margin, peak_cmp=cmp)


def match_orientation(o, got, cand):
    """Per keypoint: does `got` (degrees) equal the orientation of one of the candidate bins within its bound?"""
    d = np.abs(got[:, None].astype(np.float64) - o["ori"]) % 360.0
    d = np.minimum(d, 360.0 - d)
    return (cand & (d <= o["ori_tol"])).any(1)


# --------------------------------------------------------------------------------------------------------- descriptor
def fast_atan2(y, x):
    """describe.cu fast_atan2, float32 op for op."""
    y = np.asarray(y, np.float32)
    x = np.asarray(x, np.float32)
    absx, absy = np.abs(x), np.abs(y)
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.minimum(absx, absy) / np.maximum(absx, absy)
    s = a * a
    r = fma32(s, F32(-0.0464964749), F32(0.15931422))
    r = fma32(s, r, F32(-0.327622764))
    r = s * r
    r = fma32(r, a, a)
    r = np.where(absy > absx, F32(1.57079637) - r, r).astype(np.float32)
    r = np.where(x < 0, F32(3.14159274) - r, r).astype(np.float32)
    return np.where(y < 0, -r, r).astype(np.float32)


def _gauss16():
    t = np.arange(16) - 7.5
    return np.exp(-t * t / 128.0)


def _normalise(v):
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        t1 = np.fmin(v * (1.0 / np.sqrt((v * v).sum(1)))[:, None], 0.2)
        return t1, t1 * (1.0 / np.sqrt((t1 * t1).sum(1)))[:, None]


def _propagate(v, B, NB):
    """Bound on |normalise(v + b) - normalise(v)| for |b_e| <= B_e and ||b||_2 <= NB, elementwise, through both
    normalisations and the clamp (1-Lipschitz), plus the float32 norm arithmetic (tree sums, rsqrtf: 16 u relative
    per stage).  For x' = x + b:  |x'_e/|x'| - x_e/|x|| <= (B_e + |x_e|/|x| NB) / (|x| - NB), and the whole unit
    vector moves by at most |b|/|x| + |x'| ||x'| - |x|| / (|x'| |x|) <= 2 NB / |x|."""
    def step(x, b, nb):
        nx = np.sqrt((x * x).sum(1))[:, None]
        nb = np.minimum(nb[:, None], np.sqrt((b * b).sum(1))[:, None])
        with np.errstate(divide="ignore", invalid="ignore"):
            out = np.where(nx > nb, (b + np.abs(x) / nx * nb) / (nx - nb), np.inf)
            out = np.minimum(out, 2.0 * nb / nx) + 16.0 * U * np.abs(x) / nx
            nout = 2.0 * nb[:, 0] / nx[:, 0] + 16.0 * U
        return out, nout
    t1, _ = _normalise(v)
    d1, n1 = step(v, B, NB)
    return step(t1, d1 * (1 + 1e-12), n1 * (1 + 1e-12))[0]


def descriptors(img, px, py, pscale, orientation, sin_err=SIN_ERR, q22_carry=True):
    """The 128-D descriptors of describe_kernel for keypoints at (px, py, pscale) with the given float32
    orientations (degrees).  sin_err: bound on the sin/cos error against the correctly rounded sin(theta) used here
    (SIN_ERR for the GPU's __sinf/__cosf; about one ulp for libm's sinf).  q22_carry=False: the variant that drops
    the angi == 8 votes instead of carrying them into the next cell.

    Returns a dict:
      desc (N, 128)      float64 descriptor
      bound (N, 128)     bound on |desc_gpu - desc| (rounding + texture + grid-ambiguous fetches), given which side
                         of the discontinuity near angle pi each sample in `jumps` lands on: see within_bound()
      jumps              per row, the samples that may land on either side, as 128-vectors of the vote they move
      loose_bound        the bound without that knowledge (each such move counted elementwise and in norm)
      round_bound        the part of bound due to float32 rounding and the texture's final rounding alone
      amb_rows (N,)      rows with at least one grid-ambiguous fetch;  amb_fetch (N,) their count
      q21 (N,)           rows with an exactly zero gradient (NaN vote, quirk Q21: constant 1/sqrt(128) row)
      q21_maybe (N,)     rows where a perturbation within bounds could make a gradient exactly zero
      q22 (N,)           votes through quirk Q22 (angi == 8 with a nonzero spatial weight into a cell)
    """
    px = np.asarray(px, np.float32)
    py = np.asarray(py, np.float32)
    ps = np.asarray(pscale, np.float32)
    N = len(px)
    theta = f32(THETA_K * np.asarray(orientation, np.float32))
    sina = f32(np.sin(theta.astype(np.float64)))
    cosa = f32(np.cos(theta.astype(np.float64)))
    scale = f32(F32(0.75) * ps)
    ssina, scosa = f32(scale * sina), f32(scale * cosa)
    s = np.arange(256)
    y, x = s // 16, s % 16
    tt = (x - 7.5).astype(np.float32)[None, :]
    yy = (y - 7.5).astype(np.float32)[None, :]
    P, Q = px[:, None], py[:, None]
    xpos = f32(fma32(-ssina[:, None], yy, f32(f32(tt * scosa[:, None]) + P)) + F32(0.5))
    ypos = f32(fma32(scosa[:, None], yy, fma32(tt, ssina[:, None], Q)) + F32(0.5))
    S, C = sina[:, None], cosa[:, None]
    # coordinate uncertainty per axis: sin/cos error through scale * (|tt| + |yy|) and the +-cos/sin offset, and one
    # rounding flip per float32 operation whose result has the coordinate's magnitude (+ P, fma, + 0.5, +- cos/sin:
    # four, each at most an ulp of the largest such intermediate)
    dsin = sin_err * (scale[:, None].astype(np.float64) * (np.abs(tt) + np.abs(yy)) + 1.0)
    reach = 16.0 * scale[:, None] + 2.0
    dcx = (dsin + 4.0 * ulp32(np.abs(P).astype(np.float64) + reach)) * (1.0 + 1e-6)
    dcy = (dsin + 4.0 * ulp32(np.abs(Q).astype(np.float64) + reach)) * (1.0 + 1e-6)
    fa, ea, ma, ra = tex2d_bounded(img, f32(xpos + C), f32(ypos + S), dcx, dcy)
    fb, eb, mb, rb = tex2d_bounded(img, f32(xpos - C), f32(ypos - S), dcx, dcy)
    fc, ec, mc, rc = tex2d_bounded(img, f32(xpos - S), f32(ypos + C), dcx, dcy)
    fd, ed, md, rd = tex2d_bounded(img, f32(xpos + S), f32(ypos - C), dcx, dcy)
    dx = f32(fa.astype(np.float64) - fb)
    dy = f32(fc.astype(np.float64) - fd)
    dx64, dy64 = dx.astype(np.float64), dy.astype(np.float64)
    amb_n = ma.astype(int) + mb + mc + md
    # a perturbed subtraction also rounds differently: one more ulp of the difference, unless nothing moved
    udx, udy = ulp32(dx), ulp32(dy)
    eps = np.maximum(ea + eb + np.where(ea + eb > 0, udx, 0), ec + ed + np.where(ec + ed > 0, udy, 0))
    eps_round = np.maximum(ra + rb + np.where(ra + rb > 0, udx, 0), rc + rd + np.where(rc + rd > 0, udy, 0))
    g16 = _gauss16()
    gw = g16[y] * g16[x]
    g = np.sqrt(dx64 * dx64 + dy64 * dy64)
    grad = gw[None, :] * g
    at = fast_atan2(dy, dx)
    angf = fma32(at, ANGF_K, F32(4.0))
    nan = np.isnan(angf)
    angi = np.where(nan, 0, np.trunc(np.where(nan, 0, angf))).astype(np.int64)
    af = f32(angf - angi.astype(np.float32)).astype(np.float64)
    angp = np.where(angi < 7, angi + 1, 0)
    # spatial weights: the sample's cell (hori, veri) and its right / lower neighbours (describe.cu:191-205)
    hori, veri = (x + 2) // 4 - 1, (y + 2) // 4 - 1
    horf = (x - 1.5) * 0.25 - hori
    verf = (y - 1.5) * 0.25 - veri
    cells, sws = [], []
    for dv, dh in ((0, 0), (1, 0), (0, 1), (1, 1)):
        cv, ch = veri + dv, hori + dh
        sw = (verf if dv else 1.0 - verf) * (horf if dh else 1.0 - horf)
        ok = (cv >= 0) & (cv <= 3) & (ch >= 0) & (ch <= 3)
        cells.append(np.where(ok, 4 * cv + ch, -1))
        sws.append(np.where(ok, sw, 0.0))
    rows = np.arange(N)[:, None] * 129
    L = 129 * N                        # per row 128 bins + a sink for dropped votes
    acc = np.zeros(L)
    gsum = np.zeros(L)
    cnt = np.zeros(L)
    q22 = np.zeros(N, np.int64)
    # perturbation of a sample's gradient within eps: smooth change, or a jump where the vote function is
    # discontinuous (angf = 8: the Q22 carry; angle = +-pi: the wrap) or the gradient may vanish
    dist_disc = np.minimum(np.abs(np.abs(at.astype(np.float64)) - np.pi), np.abs(at.astype(np.float64) - 3.1415))

    # A smooth move changes each of the (at most four) bins it reaches by `smooth`.  A jump moves at most the whole
    # vote `big`: elementwise it can land on any bin it reaches, but in norm it moves at most 2 * big (what leaves
    # one bin plus what arrives in another).  Near the discontinuity with a well-defined angle (dth < 0.3 rad, so
    # angf stays within 0.4 of 0 or 8) the bins it reaches are 7, 0 and 1 of the cell and bin 0 of the next cell;
    # a gradient that may vanish can reach any of the cell's bins.
    def perturbation(e):
        with np.errstate(divide="ignore", invalid="ignore"):
            dth = np.where(g > 2.0 * 1.5 * e, 1.5 * e / (g - 1.5 * e), np.inf) + ATAN_SLACK
        jump = ~(dth < dist_disc) | nan
        local = jump & (dth < 0.3) & ~nan
        smooth = np.where(jump & ~local, 0.0, 1.5 * e + (g + 1.5 * e) * float(ANGF_K) * np.where(jump & ~local, 0.0, dth))
        return jump, local, smooth, np.where(jump & ~nan, (g + 1.5 * e) * (1.0 + 2e-4), 0.0)
    pert, pert_r = np.zeros(L), np.zeros(L)         # smooth moves, elementwise
    pj, pj_r = np.zeros(L), np.zeros(L)             # jumps, elementwise
    jmp, jmp_r = np.zeros(L), np.zeros(L)           # jumps, norm (per row, at slot 0)
    flips = []                                      # local jumps of the full bound: (row, sample, from, to, weight)
    for c, sw in zip(cells, sws):
        valid = (c >= 0)[None, :] & (sw > 0)[None, :]
        base = rows + np.where(c >= 0, 8 * c, 0)[None, :]
        g2 = grad * sw[None, :]
        sink = rows + 128
        i8 = angi == 8
        if q22_carry:
            lo_idx = np.where(i8 & (c == 15)[None, :], sink, base + angi)
        else:
            lo_idx = np.where(i8, sink, base + angi)
        q22 += (valid & i8).sum(1)
        lo_idx = np.where(valid, lo_idx, sink)
        hi_idx = np.where(valid, base + angp, sink)
        with np.errstate(invalid="ignore"):
            acc += np.bincount(lo_idx.ravel(), ((1.0 - af) * g2).ravel(), minlength=L)
            acc += np.bincount(hi_idx.ravel(), (af * g2).ravel(), minlength=L)
        gg = np.abs(g2) * (1.0 + np.abs(af))
        gsum += np.bincount(lo_idx.ravel(), np.where(nan, 0, gg).ravel(), minlength=L)
        gsum += np.bincount(hi_idx.ravel(), np.where(nan, 0, gg).ravel(), minlength=L)
        cnt += np.bincount(lo_idx.ravel(), minlength=L) + np.bincount(hi_idx.ravel(), minlength=L)
        for e, out, pout, jout in ((eps, pert, pj, jmp), (eps_round, pert_r, pj_r, jmp_r)):
            jump, local, smooth, big = perturbation(e)
            wv = gw[None, :] * sw[None, :]
            if not valid.any():
                continue
            sm_w = wv * smooth
            for j in range(-1, 3):          # a smooth move reaches the two bins and one either side
                idx = np.where(valid & ~jump, base + (angi + j) % 8, sink)
                out += np.bincount(idx.ravel(), sm_w.ravel(), minlength=L)
            # a local jump of the full bound is enumerated by within_bound(): the vote sits either at angle bin 0 of
            # this cell (angi 7 or 0) or at angle bin 0 of the next cell (angi 8, the Q22 carry; dropped past cell 15
            # or without the carry), and moves smoothly around either place
            enum = local if out is pert else np.zeros_like(local)
            nxt = base + 8 if q22_carry else np.broadcast_to(sink, base.shape)
            nxt = np.where((c < 15)[None, :], nxt, sink)
            for tgt in (base + 7, base, base + 1, nxt):
                out += np.bincount(np.where(valid & enum, tgt, sink).ravel(), sm_w.ravel(), minlength=L)
            if enum.any():
                r_, s_ = np.nonzero(valid & enum)
                here, there = base[r_, s_], nxt[r_, s_]
                at_next = angi[r_, s_] == 8
                flips.append((r_, s_, np.where(at_next, there, here), np.where(at_next, here, there),
                              (g2 * (1.0 + np.abs(af)))[r_, s_] * (1.0 + 2e-4)))
            jw = (wv * big * ~enum).ravel()
            for j in range(9):               # bin 8: angle bin 0 of the next cell (the Q22 carry)
                reach = (j in (7, 0, 1, 8)) | ~local
                idx = np.where(valid & jump & reach & ((j < 8) | (c < 15)[None, :]), base + j, sink)
                pout += np.bincount(idx.ravel(), jw, minlength=L)
            jout += np.bincount(np.where(valid & jump, rows, sink).ravel(), 2.0 * jw, minlength=L)
    v = acc.reshape(N, 129)[:, :128]
    G = gsum.reshape(N, 129)[:, :128]
    n_terms = cnt.reshape(N, 129)[:, :128]
    # float32 rounding of one vote: gauss (__expf, 2 ulp each), grad (sqrt, fma, mul), three spatial / angle
    # products and 1 - af: 16 u of its spatial-weighted gradient; summation: (terms + 8) u of the sum of magnitudes
    R = (n_terms + 8.0 + 16.0) * U * G
    q21 = np.isnan(v).any(1)
    t1, desc = _normalise(v)
    vz = np.where(np.isnan(v), 0.0, v)
    # norm of the perturbation: the elementwise bound of the smooth part and rounding, plus 2 * big per jump
    def parts(sm_, j_, jn):
        Bsm = R + sm_.reshape(N, 129)[:, :128]
        return Bsm + j_.reshape(N, 129)[:, :128], np.sqrt((Bsm * Bsm).sum(1)) + jn.reshape(N, 129)[:, 0]
    Bt, NBt = parts(pert, pj, jmp)
    bound = _propagate(vz, Bt, NBt)
    round_bound = _propagate(vz, *parts(pert_r, pj_r, jmp_r))
    # per row: the local jumps as 128-vectors (one per sample: all its cells flip together)
    jumps = [np.zeros((0, 128)) for _ in range(N)]
    if flips:
        r_, s_, fr, to, w_ = (np.concatenate(a) for a in zip(*flips))
        for r in np.unique(r_):
            m = r_ == r
            ss = np.unique(s_[m])
            D = np.zeros((len(ss), 129))
            k = np.searchsorted(ss, s_[m])
            np.add.at(D, (k, fr[m] - r * 129), -w_[m])
            np.add.at(D, (k, to[m] - r * 129), w_[m])
            jumps[r] = D[:, :128]
    # without enumeration (rows with more than MAX_FLIPS such samples): each flip elementwise at its two bins, and
    # 2 * weight in norm
    Bl, NBl = Bt.copy(), NBt.copy()
    for D, r in zip(jumps, range(N)):
        if len(D):
            Bl[r] += np.abs(D).sum(0)
            NBl[r] += np.abs(D).sum()
    # a zero gradient within reach of the perturbation makes the row's Q21 status uncertain
    zero_ok = (np.abs(dx64) <= np.maximum(ea + eb, 0)) & (np.abs(dy64) <= np.maximum(ec + ed, 0))
    q21_maybe = (zero_ok & ~nan).any(1)
    bound[q21] = 0.0
    round_bound[q21] = 0.0
    amb_rows = amb_n.sum(1) > 0
    return dict(desc=desc, bound=bound, round_bound=round_bound, amb_rows=amb_rows, amb_fetch=amb_n.sum(1), q21=q21,
                q21_maybe=q21_maybe & ~q21, q22=q22, raw=v, jumps=jumps, B=Bt, NB=NBt,
                loose_bound=_propagate(vz, Bl, NBl))


MAX_FLIPS = 14


def within_bound(d, got, rows=None):
    """Per row: is the kernel's descriptor `got` within the bound of one of the 2^K descriptors the restatement
    allows, K being the row's samples that a perturbation within bounds can carry across the vote function's
    discontinuity near angle pi?  Returns (ok, bound of the accepted or closest variant (elementwise max), K)."""
    rows = np.arange(len(got)) if rows is None else rows
    ok = np.zeros(len(rows), bool)
    bmax = np.full(len(rows), np.inf)
    K = np.array([len(d["jumps"][r]) for r in rows])
    for i, r in enumerate(rows):
        D = d["jumps"][r]
        if len(D) > MAX_FLIPS:
            b = d["loose_bound"][r]
            ok[i] = np.all(np.abs(got[i] - d["desc"][r]) <= b)
            bmax[i] = b.max()
            continue
        Z = ((np.arange(2 ** len(D))[:, None] >> np.arange(len(D))[None, :]) & 1).astype(np.float64)
        vz = d["raw"][r][None, :] + Z @ D
        _, dz = _normalise(vz)
        bz = _propagate(vz, np.broadcast_to(d["B"][r], vz.shape), np.full(len(vz), d["NB"][r]))
        fit = np.all(np.abs(got[i][None, :] - dz) <= bz, 1)
        ok[i] = fit.any()
        bmax[i] = bz[fit].max(1).min() if fit.any() else bz.max(1).min()
    return ok, bmax, K
