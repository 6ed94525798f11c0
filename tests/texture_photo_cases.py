"""One case per rule of cs_texture_mesh_photo (rules 3a to 3c; tests/test_texture_photo_*.py): sub-pixel faces that fall
back to the centroid pixel, faces whose samples reach the image border (clamped Sobel taps), faces partly hidden behind
an occluder, equal q, a flat view against a faintly textured one (the GMI floor), and the outlier test at m = 2, m = 3, even m, MAD = 0, the best candidate removed, a distance of
exactly K s, and more than 8 passing images.  Each returns texture_cases' dict, with kw holding the photo settings
(dataTerm, outlierK, outlierMinSigma) beside the texturing arguments.

The sampling cases are soups of separate triangles seen by identical pixel cameras (texture_cases.pix) with different
random images, at lambda 0: every view of a face has the same area, so GMI's g decides the label, the image-ascending
tie decides it under the area term, and the outlier test sees random means.  The outlier cases are a pixel grid seen by
pixel cameras of decreasing focal length (so the views rank by camera) with constant images: each mean is the image's
value exactly."""
import numpy as np

import texture_cases as tc

PHOTO = dict(dataTerm=1, outlierK=3.0, outlierMinSigma=4.0)


def _case(imgs, Ks, v, t, **kw):
    n = len(imgs)
    return tc._case(imgs, Ks, [np.eye(3)] * n, [np.zeros(3)] * n, v, t, **(PHOTO | kw))


def _soup(corners, depth=1.0, f=100.0, cx=32.0, cy=32.0):
    """Separate triangles from their pixel corners [N, 3, 2], turned to face the pixel camera."""
    c = np.asarray(corners, np.float64)
    P = tc._at_pixels(c[..., 0].reshape(-1), c[..., 1].reshape(-1), f, cx, cy, depth)
    t = np.arange(len(P)).reshape(-1, 3)
    X = P[t]
    n = np.cross(X[:, 1] - X[:, 0], X[:, 2] - X[:, 0])
    away = (n * X.mean(1)).sum(1) > 0                   # the camera sits at the origin
    t[away] = t[away][:, ::-1]
    return P, t


def _same_views(v, t, shape, k=3, seed=0, **kw):
    """k identical pixel cameras (cx = cy = 32) with random images."""
    return _case(tc._images([shape] * k, seed), [tc.pix(100.0, 32.0, 32.0)] * k, v, t, lam=0.0, **kw)


def subpixel(n=80, seed=40):
    """Rule 3a's fallback: n triangles inside single pixel cells (no pixel centre covered, an empty box), with
    centroids that round up, down or across to a neighbouring pixel."""
    rng = np.random.default_rng(seed)
    cells = rng.choice(48 * 48, n, replace=False)
    x, y = 8 + cells % 48, 8 + cells // 48
    off = rng.uniform(0.05, 0.95, (n, 3, 2))
    c = np.stack([x, y], 1)[:, None, :] + off
    return _same_views(*_soup(c), (64, 64), seed=seed + 1)


def border(seed=42):
    """Rule 3a's clamped Sobel taps: triangles of 3 to 6 pixels along every border and in every corner of 64 x 64
    images, so samples lie in row and column 0 and 63."""
    rng = np.random.default_rng(seed)
    c = []
    for k in range(0, 60, 6):
        s = rng.uniform(3, 6)
        c += [[(k, 0), (k + s, 0), (k, s)], [(63 - k, 63), (63 - k - s, 63), (63 - k, 63 - s)],
              [(0, k + 1), (s, k + 1), (0, k + 1 + s)], [(63, 62 - k), (63 - s, 62 - k), (63, 62 - k - s)]]
    c += [[(0, 0), (2.5, 0), (0, 2.5)], [(63, 63), (60.5, 63), (63, 60.5)]]
    return _same_views(*_soup(np.clip(np.array(c, np.float64), 0, 63)), (64, 64), seed=seed + 1)


def occluded(seed=44):
    """Rule 3a's depth-buffer samples: 12 back triangles at depth 2, each with a front square at depth 1 over part of
    its inside (away from its corners and centroid), so some of its box pixels name the square."""
    b, f = [], []
    for k in range(12):
        x, y = 4 + 14 * (k % 4), 4 + 18 * (k // 4)
        b.append([(x, y), (x + 13, y), (x, y + 16)])
        f += [[(x + 7, y + 0.5), (x + 11, y + 0.5), (x + 11, y + 2.5)], [(x + 7, y + 0.5), (x + 11, y + 2.5),
                                                                         (x + 7, y + 2.5)]]
    v, t = tc.join(_soup(b, depth=2.0), _soup(f, depth=1.0))
    return _same_views(v, t, (64, 64), seed=seed + 1)


def equal_q(seed=46):
    """Rules 3a and 3b's ties: views 0 and 1 are the same camera and the same image, so their q are equal under both
    data terms and the lower image wins; view 2 differs."""
    v, t = tc.pixel_grid(8, 8, 6, 6, 8, cx=32.0, cy=32.0)
    imgs = tc._images([(64, 64)] * 2, seed)
    return _case([imgs[0], imgs[0].copy(), imgs[1]], [tc.pix(100.0, 32.0, 32.0)] * 3, v, t, lam=0.5)


def ranked(values, lam=0.5, imgs=None, **kw):
    """Rule 3c: a 4 x 4-cell grid seen by pixel cameras of focal length 100, 98, 96, ... (view k ranks k-th at every
    face by area) with constant images of the given values (or the images given)."""
    v, t = tc.pixel_grid(16, 16, 4, 4, 8, cx=32.0, cy=32.0)
    n = len(values)
    if imgs is None:
        imgs = [np.full((64, 64), x, np.float32) for x in values]
    return _case(imgs, [tc.pix(100.0 - 2.0 * k, 32.0, 32.0) for k in range(n)], v, t, lam=lam, **kw)


def textureless(seed=48):
    """Rule 3b's floor: view 0 is flat (g = 0), view 1 has a faint texture (g well under 0.04, less than view 0's
    area gain of (100 / 98)^2), so with the floor of 1 view 0 still wins by area under GMI; without it view 0's q would
    be 0."""
    rng = np.random.default_rng(seed)
    faint = (100.0 + rng.uniform(-0.01, 0.01, (64, 64))).astype(np.float32)
    return ranked([100.0, 100.0], imgs=[np.full((64, 64), 100.0, np.float32), faint])


def m2():
    """m = 2: not tested, however far apart."""
    return ranked([100.0, 200.0])


def m3():
    """m = 3: med 104, MAD 4, K s = 17.79; 180 leaves."""
    return ranked([100.0, 104.0, 180.0])


def even_m():
    """m = 6: med (100 + 110) * 0.5 = 105, MAD (5 + 5) * 0.5 = 5, K s = 22.24; 130 leaves (with the upper middle
    values, med 110 and MAD 10, nothing would)."""
    return ranked([100.0, 110.0, 100.0, 115.0, 100.0, 130.0])


def mad0():
    """MAD = 0: s is the floor 4, K s = 12; 110 stays, 130 leaves."""
    return ranked([100.0, 100.0, 110.0, 100.0, 130.0])


def best_removed():
    """The best view is the outlier: the face starts at view 1, D normalised by view 1's q."""
    return ranked([200.0, 100.0, 101.0, 100.0, 102.0])


def at_limit():
    """|mu - med| = K s exactly: med 100, MAD 0, K s = 3 x 4 = 12, and 112 stays."""
    return ranked([100.0, 100.0, 112.0, 100.0])


def capped():
    """More than 8 passing images: the best 8 alternate 100 and 200 (med 150, MAD 50: nothing leaves); over all 10,
    with the last two at 100, med would be 100 and MAD 0, and every 200 would leave."""
    return ranked([100.0, 200.0] * 4 + [100.0, 100.0])


CASES = {"subpixel": subpixel, "border": border, "occluded": occluded, "equal_q": equal_q, "textureless": textureless,
         "m2": m2, "m3": m3, "even_m": even_m, "mad0": mad0, "best_removed": best_removed, "at_limit": at_limit,
         "capped": capped}
