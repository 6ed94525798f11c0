"""cs_texture_mesh_photo's rules 3a to 3c restated in float64 (numpy element-wise operations, each rounded once, in the
header's order), in the device's lane and butterfly order: the samples of every passing (face, image) pair with their
Sobel magnitudes and intensities, the GMI or area data term, the best 8 candidates with their means, and the
median/MAD outlier test; the labelling, charts and atlas are texture_oracle.texture's, unchanged.  The passing pairs
are texture_oracle.candidates' own, asked one image at a time, so rule 3's tests are stated once."""
import numpy as np

import texture_oracle as to

MCAND = to.MCAND
LANES = 32


def sobel(img):
    """G [H, W]: the Sobel magnitude over 8 at every pixel, indices clamped to the image."""
    I = np.asarray(img, np.float32).astype(np.float64)
    H, W = I.shape
    x, y = np.arange(W), np.arange(H)
    xm, xp, ym, yp = np.maximum(x - 1, 0), np.minimum(x + 1, W - 1), np.maximum(y - 1, 0), np.minimum(y + 1, H - 1)
    P = lambda ys, xs: I[ys][:, xs]
    gx = ((P(ym, xp) - P(ym, xm)) + 2.0 * (P(y, xp) - P(y, xm))) + (P(yp, xp) - P(yp, xm))
    gy = ((P(yp, xm) - P(ym, xm)) + 2.0 * (P(yp, x) - P(ym, x))) + (P(yp, xp) - P(ym, xp))
    return np.sqrt(gx * gx + gy * gy) / 8.0


def lane_sums(vals):
    """The device's sum of vals (in box-index order, zeros where a pixel is no sample): lane j adds the entries
    i = j mod 32 in ascending i, then the xor butterfly 16, 8, 4, 2, 1; lane 0's value."""
    v = np.asarray(vals, np.float64)
    rows = -(-len(v) // LANES)
    pad = np.zeros(rows * LANES)
    pad[:len(v)] = v
    acc = np.zeros(LANES)
    for r in pad.reshape(rows, LANES):
        acc = acc + r
    return float(to._butterfly(acc)[0])


def box(u, v, W, H):
    """Rule 2's clipped bounding box (xlo, xhi, ylo, yhi) of a face's corners u, v [3]; empty when xlo > xhi or
    ylo > yhi."""
    xlo = max(0.0, np.ceil(min(min(u[0], u[1]), u[2])))
    xhi = min(W - 1.0, np.floor(max(max(u[0], u[1]), u[2])))
    ylo = max(0.0, np.ceil(min(min(v[0], v[1]), v[2])))
    yhi = min(H - 1.0, np.floor(max(max(v[0], v[1]), v[2])))
    return int(xlo), int(xhi), int(ylo), int(yhi)


def visible(keys, f):
    """The box pixels that are samples of face f: their key names f."""
    return (keys & np.uint64(0xFFFFFFFF)) == np.uint64(f)


def centroid_pixel(uc, vc):
    return int(np.floor(uc + 0.5)), int(np.floor(vc + 0.5))


def best8(c):
    """A face's kept candidates: the best MCAND by (q descending, image ascending)."""
    return sorted(c, key=lambda e: (-e[0], e[1]))[:MCAND]


def sample(f, buf, G, I, u, v, uc, vc):
    """Rule 3a for face f in one image: (n, g, mu)."""
    H, W = I.shape
    xlo, xhi, ylo, yhi = box(u, v, W, H)
    n = 0
    if xlo <= xhi and ylo <= yhi:
        keys = buf[ylo:yhi + 1, xlo:xhi + 1].reshape(-1)
        mask = visible(keys, f)
        n = int(mask.sum())
    if n == 0:
        px, py = centroid_pixel(uc, vc)
        return 0, float(G[py, px]), float(I[py, px])
    g = lane_sums(np.where(mask, G[ylo:yhi + 1, xlo:xhi + 1].reshape(-1), 0.0))
    i = lane_sums(np.where(mask, I[ylo:yhi + 1, xlo:xhi + 1].reshape(-1), 0.0))
    return n, g / float(n), i / float(n)


def quality(area, g, dataTerm):
    """Rule 3b's q: the area, or the area times (g + 1)."""
    return area * (g + 1.0) if dataTerm else area


def median(x):
    s = sorted(x)
    m = len(s)
    return s[m // 2] if m % 2 else (s[m // 2 - 1] + s[m // 2]) * 0.5


def spread(mad, minSigma):
    return max(1.4826 * mad, minSigma)


def outliers(c, outlierK, minSigma):
    """Rule 3c on one face's kept candidates c [(q, image, mu)]: (survivors in order, tested, best removed)."""
    m = len(c)
    if not outlierK > 0 or m < 3:
        return c, False, False
    mu = [e[2] for e in c]
    med = median(mu)
    lim = outlierK * spread(median([abs(x - med) for x in mu]), minSigma)
    keep = [e for e in c if not abs(e[2] - med) > lim]
    return keep, True, abs(mu[0] - med) > lim


def passing(candidates, cams, bufs, verts, tris, maxViewAngleDeg, depthTol):
    """Per image a: (a, the faces that pass every test of rule 3 with their area q = 0.5 |A|, the corners' u and v
    [T, 3], the centroid's u and v [T]), from texture_oracle's rule 3 (candidates) on image a alone."""
    X = np.asarray(verts, np.float32).astype(np.float64)
    tr = np.asarray(tris, np.int64)
    cen = ((X[tr[:, 0]] + X[tr[:, 1]]) + X[tr[:, 2]]) / 3.0
    for a, (K, R, t, W, H) in enumerate(cams):
        lists, _ = candidates([cams[a]], [bufs[a]], X, tr, maxViewAngleDeg, depthTol)
        U, V, _ = to.project(K, R, t, X[tr])
        Uc, Vc, _ = to.project(K, R, t, cen)
        yield a, [(f, c[0][0]) for f, c in enumerate(lists) if c], U, V, Uc, Vc


def photo_candidates(images, cams, bufs, verts, tris, maxViewAngleDeg, depthTol, dataTerm, outlierK, minSigma,
                     candidates=None):
    """Rules 3a to 3c: per face its (q, image) candidates after the outlier test, the passing pairs, and the five
    counters of stats [11..15].  candidates is rule 3 of cs_texture_mesh (texture_oracle.candidates)."""
    T = len(tris)
    lists = [[] for _ in range(T)]
    total = samples = fallbacks = 0
    for a, ok, U, V, Uc, Vc in passing(candidates or to.candidates, cams, bufs, verts, tris, maxViewAngleDeg,
                                       depthTol):
        G, I = sobel(images[a]), np.asarray(images[a], np.float32).astype(np.float64)
        for f, area in ok:
            n, g, mu = sample(f, bufs[a], G, I, U[f], V[f], Uc[f], Vc[f])
            samples += n
            fallbacks += n == 0
            lists[f].append((float(quality(area, g, dataTerm)), a, mu))
        total += len(ok)
    out, tested, removed, best = [], 0, 0, 0
    for c in lists:
        kept = best8(c)
        keep, t, b = outliers(kept, outlierK, minSigma)
        tested += t
        removed += len(kept) - len(keep)
        best += b
        out.append(keep)
    return out, total, [samples, fallbacks, tested, removed, best]


def texture_photo(images, Ks, Rs, ts, verts, tris, dataTerm=1, outlierK=3.0, outlierMinSigma=4.0, lam=0.5,
                  maxViewAngleDeg=75.0, depthTol=0.01, bufs=None, **kw):
    """The whole call: texture_oracle.texture's dict with rule 3 replaced and stats [16]; 'means' holds each face's
    surviving (q, image, mu).  texture_oracle.texture looks its rule 3 up as the module's `candidates`, which stands
    for rules 3a to 3c for the length of the call."""
    extra = {}
    rule3 = to.candidates

    def select(cams, bf, X, tr, angle, tol):
        c, total, counters = photo_candidates(images, cams, bf, X, tr, angle, tol, dataTerm, outlierK,
                                              outlierMinSigma, rule3)
        extra.update(counters=counters, means=c)
        return [[(q, a) for q, a, _ in e] for e in c], total

    to.candidates = select
    try:
        r = to.texture(images, Ks, Rs, ts, verts, tris, lam=lam, maxViewAngleDeg=maxViewAngleDeg, depthTol=depthTol,
                       bufs=bufs, **kw)
    finally:
        to.candidates = rule3
    r["stats"] = list(r["stats"]) + extra.get("counters", [0] * 5)
    r["means"] = extra.get("means")
    return r
