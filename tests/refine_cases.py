"""Meshes and views for photometric mesh refinement (cs_mesh_refine): the scene of stereo_cases as texture_cases' grids
with every interior vertex jittered along its rectangle's normal, rendered by stereo_cases.render with a coarse texture
so the NCC basin is a few pixels wide, and one small case per rule (fixed vertices, an occluder, windows cut by the
border and by holes, a flat texture at the variance floor, a repeated pair, a line search that rejects).  Each
generator returns a dict: imgs (float32 [H, W] list), Ks, Rs, ts, v (float32 [V, 3]), t (int32 [T, 3]), pairs
(int32 [n, 2]) and kw, the call's arguments by refine_oracle.refine's names; the scene also carries its rectangles
and each vertex's rectangle, for the distance to the true planes."""
import numpy as np

import stereo_cases as sc
import texture_cases as tc

TEXELS = 6.0                     # texture samples per world unit: coarse, so the basin spans a few pixels


def scene(n=6, width=160, height=120, cell=0.3, jitter=0.15, seed=0, texels=TEXELS):
    """The scene's rectangles as grids of cell-sized squares, every interior vertex moved along its rectangle's normal
    by up to jitter * cell (the borders stay on their planes and are fixed: each rectangle is an open grid), seen by n
    renders; pairs (a, a + 1) and (a + 1, a)."""
    Ks, Rs, ts, views = sc.render(n, width, height, seed=seed, texels=texels)
    C = np.mean([-R.T @ t for R, t in zip(Rs, ts)], axis=0)
    rng = np.random.default_rng(seed + 100)
    vs, tr, rect, k = [], [], [], 0
    rects = sc.scene()
    for ri, r in enumerate(rects):
        toward = r["c"] - tc.BOX_CENTRE if 2 <= r["face"] <= 6 else C - r["c"]
        P, t, border = tc._grid(r, cell, toward)
        off = np.where(border, 0.0, rng.uniform(-jitter * cell, jitter * cell, len(P)))
        vs.append(P + off[:, None] * r["n"][None, :])
        tr.append(t + k)
        rect.append(np.full(len(P), ri))
        k += len(P)
    pairs = [(a, a + 1) for a in range(n - 1)] + [(a + 1, a) for a in range(n - 1)]
    return dict(imgs=[v[0] for v in views], Ks=Ks, Rs=Rs, ts=ts, v=np.concatenate(vs).astype(np.float32),
                t=np.concatenate(tr).astype(np.int32), pairs=np.array(pairs, np.int32), rect=np.concatenate(rect),
                rects=rects, kw={})


def plane_rms(v, rect, rects, mask):
    """The RMS distance of the vertices v[mask] to the planes of their rectangles."""
    d = np.array([np.dot(v[i].astype(np.float64) - rects[rect[i]]["c"], rects[rect[i]]["n"])
                  for i in np.nonzero(mask)[0]])
    return float(np.sqrt(np.mean(d * d))) if len(d) else 0.0


def _case(imgs, Ks, Rs, ts, v, t, pairs, **kw):
    return dict(imgs=[np.ascontiguousarray(im, np.float32) for im in imgs], Ks=np.asarray(Ks, np.float64),
                Rs=np.asarray(Rs, np.float64), ts=np.asarray(ts, np.float64), v=np.asarray(v, np.float32),
                t=np.asarray(t, np.int32), pairs=np.asarray(pairs, np.int32).reshape(-1, 2), kw=kw)


def _smooth(shape, seed, sigma=3.0, scale=60.0):
    """A smooth random image on 0..255 (a box-blurred noise field), so bilinear reads have useful gradients."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(0, 1, shape)
    r = int(sigma)
    for ax in (0, 1):
        a = sum(np.roll(a, s, ax) for s in range(-r, r + 1)) / (2 * r + 1)
    return (128.0 + scale * (a - a.mean()) / (a.std() + 1e-9)).astype(np.float32)


def _views(target, offsets, W=96, H=80, seed=0):
    return tc.oblique(target, W, H, offsets, seed=seed)


def _bumpy(nx=10, ny=8, step=6.0, seed=0, amp=2.0):
    """A pixel grid (texture_cases.pixel_grid) with random depth bumps, facing the cameras at z ~ 100."""
    rng = np.random.default_rng(seed)
    v, t = tc.pixel_grid(20, 20, nx, ny, step, cx=50.0, cy=45.0)
    v[:, 2] += rng.uniform(-amp, amp, len(v))
    return v, t


def fixed_vertices():
    """Rule 1: a bumpy grid with a fin on an interior edge (three faces on it: its two vertices fixed), a face on a
    boundary edge, and unused vertices; two views both ways."""
    v, t = _bumpy(seed=1)
    n = len(v)
    a, b = 23, 24                                   # an interior row edge of the 11-wide vertex grid
    fin = 0.5 * (v[a] + v[b]) + np.array([0.5, -1.0, -6.0])
    v = np.concatenate([v, [fin], np.array([[1e3, 1e3, 1e3], [-5.0, 2.0, 90.0]])])
    t = np.concatenate([t, [[a, b, n]]])
    Ks, Rs, ts = _views([0.0, 0.0, 100.0], [(-25, 5, -180), (25, -5, -180)], seed=2)
    imgs = [_smooth((80, 96), 3), _smooth((80, 96), 4)]
    return _case(imgs, Ks, Rs, ts, v, t, [(0, 1), (1, 0)])


def occluder():
    """Rule 3's visibility: a small grid close to camera 1 hides part of the bumpy grid from it, so pixels of camera
    0 whose points camera 1 cannot see stay unmapped."""
    v, t = _bumpy(seed=5)
    w, u = tc.pixel_grid(30, 30, 2, 2, 4, cx=50.0, cy=45.0, depth=0.6)
    v, t = tc.join((v, t), (w, u))
    Ks, Rs, ts = _views([0.0, 0.0, 100.0], [(0, 0, -200), (30, 10, -170)], seed=6)
    imgs = [_smooth((80, 96), 7), _smooth((80, 96), 8)]
    return _case(imgs, Ks, Rs, ts, v, t, [(0, 1)])


def windows_cut():
    """Rule 4: a grid that runs past the border of image 0 (windows cut by the border) with holes (faces removed),
    whose windows are cut by the unmapped pixels; windowRadius 3."""
    v, t = tc.pixel_grid(-10, 10, 12, 10, 7, cx=50.0, cy=45.0)
    rng = np.random.default_rng(9)
    v[:, 2] += rng.uniform(-1.5, 1.5, len(v))
    t = np.delete(t, [30, 31, 75, 120, 121, 122], axis=0)
    Ks, Rs, ts = _views([0.0, 0.0, 100.0], [(10, 0, -90), (-20, 10, -180)], seed=10)
    imgs = [_smooth((80, 96), 11), _smooth((80, 96), 12)]
    return _case(imgs, Ks, Rs, ts, v, t, [(0, 1), (1, 0)], windowRadius=3)


def flat():
    """Rule 4's floor: image 1 is flat over one half (variance below 1 grey level^2), image 0 textured."""
    v, t = _bumpy(seed=13)
    Ks, Rs, ts = _views([0.0, 0.0, 100.0], [(-20, 0, -190), (20, 5, -185)], seed=14)
    a, b = _smooth((80, 96), 15), _smooth((80, 96), 16)
    b[:, :48] = 100.0 + 0.2 * (np.arange(48) % 2)
    return _case([a, b], Ks, Rs, ts, v, t, [(0, 1), (1, 0)])


def repeated():
    """Rule 6's pair order: the same pair twice and three images, windowRadius 1."""
    v, t = _bumpy(seed=17)
    Ks, Rs, ts = _views([0.0, 0.0, 100.0], [(-20, 0, -190), (20, 5, -185), (0, 25, -180)], seed=18)
    imgs = [_smooth((80, 96), 19), _smooth((80, 96), 20), _smooth((80, 96), 21)]
    return _case(imgs, Ks, Rs, ts, v, t, [(0, 1), (2, 0), (0, 1)], windowRadius=1)


def rejects():
    """Rule 8's line search: a step of 1 (two mean edge lengths a vertex at most) overshoots, is rejected and
    halves."""
    c = repeated()
    c["kw"] = dict(windowRadius=2, step=1.0, smoothness=0.5)
    return c


CASES = {"fixed_vertices": fixed_vertices, "occluder": occluder, "windows_cut": windows_cut, "flat": flat,
         "repeated": repeated, "rejects": rejects}
