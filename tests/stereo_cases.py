"""Scenes for dense reconstruction (cs_patch_match_stereo, cs_fuse_depth_maps, cs_undistort_images): numpy ray casting
of a piecewise-planar scene -- a ground plane, a box, and a slanted plane in front of a back wall -- textured with
synth.synth_image by world coordinates, seen by cameras from triangulate_cases.look_at with skewed, unequal
intrinsics.  Each render returns the image, the true depth and camera-frame normal per pixel and the world point."""
import numpy as np

from cudasift_b200 import synth
from triangulate_cases import look_at

TEXELS = 32.0                    # texture samples per world unit


def _texture():
    return synth.synth_image(1024, 1024, seed=77, shapes=500, small=300, noise=20.0, sigma=1.5).astype(np.float64)


def _rect(c, u, v, hu, hv, face):
    c, u, v = (np.asarray(a, np.float64) for a in (c, u, v))
    u, v = u / np.linalg.norm(u), v / np.linalg.norm(v)
    return dict(c=c, u=u, v=v, n=np.cross(u, v), hu=hu, hv=hv, face=face)


def scene():
    """The rectangles of the scene (world Y up): ground, back wall, five faces of a box, a slanted plane."""
    rs = [_rect((0, 0, 2), (1, 0, 0), (0, 0, 1), 9, 9, 0), _rect((0, 3.5, 5), (1, 0, 0), (0, 1, 0), 9, 4, 1)]
    b, h = np.array([-0.9, 0.5, 1.6]), 0.5
    for k, (n, u, v) in enumerate([((0, 0, -1), (1, 0, 0), (0, 1, 0)), ((1, 0, 0), (0, 0, 1), (0, 1, 0)),
                                   ((-1, 0, 0), (0, 0, 1), (0, 1, 0)), ((0, 1, 0), (1, 0, 0), (0, 0, 1)),
                                   ((0, 0, 1), (1, 0, 0), (0, 1, 0))]):
        rs.append(_rect(b + h * np.array(n, float), u, v, h, h, 2 + k))
    a = np.radians(35.0)
    rs.append(_rect((1.1, 0.9, 1.2), (np.cos(a), 0, np.sin(a)), (0, 1, 0.3), 0.7, 0.6, 7))
    return rs


def cameras(n, width, height, seed=0):
    """n cameras on an arc in front of the scene looking at it, with skewed, unequal intrinsics."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = [], [], []
    for a in range(n):
        ang = np.radians(-25 + 50 * a / max(n - 1, 1)) + rng.uniform(-0.03, 0.03)
        C = np.array([5.5 * np.sin(ang), 2.0 + rng.uniform(-0.4, 0.4), 1.8 - 5.5 * np.cos(ang)])
        R = look_at(C, np.array([0.0, 0.9, 2.2]) + rng.uniform(-0.2, 0.2, 3), rng.uniform(-0.1, 0.1))
        f = width * rng.uniform(0.85, 1.0)
        K = np.array([[f, rng.uniform(-2, 2), width / 2 + rng.uniform(-6, 6)],
                      [0, f * rng.uniform(0.93, 1.07), height / 2 + rng.uniform(-6, 6)], [0, 0, 1.0]])
        Ks.append(K)
        Rs.append(R)
        ts.append(-R @ C)
    return np.array(Ks), np.array(Rs), np.array(ts)


def _sample(tex, u, v):
    H, W = tex.shape
    u = np.clip(u, 0, W - 1.001)
    v = np.clip(v, 0, H - 1.001)
    x0, y0 = np.floor(u).astype(int), np.floor(v).astype(int)
    fx, fy = u - x0, v - y0
    return ((1 - fy) * ((1 - fx) * tex[y0, x0] + fx * tex[y0, x0 + 1]) +
            fy * ((1 - fx) * tex[y0 + 1, x0] + fx * tex[y0 + 1, x0 + 1]))


def cast(K, R, t, width, height, dist=(0.0, 0.0), tex=None, texels=TEXELS):
    """The render of camera (K, R, t): (image float32, depth, normal [H, W, 3] in the camera frame facing the camera,
    world points [H, W, 3]).  With dist (k1, k2), pixel (x, y) shows what the pinhole camera sees at the undistortion
    of (x, y) (the forward model's inverse, by fixed-point iteration).  texels: texture samples per world unit."""
    tex = _texture() if tex is None else tex
    ys, xs = np.mgrid[0:height, 0:width].astype(np.float64)
    b = (ys - K[1, 2]) / K[1, 1]
    a = (xs - K[0, 2] - K[0, 1] * b) / K[0, 0]
    k1, k2 = dist
    if k1 or k2:
        ad, bd = a.copy(), b.copy()
        for _ in range(50):
            r2 = a * a + b * b
            s = 1 + k1 * r2 + k2 * r2 * r2
            a, b = ad / s, bd / s
    rays_c = np.stack([a, b, np.ones_like(a)], -1)
    rays = rays_c @ R                              # world directions (R^T d)
    C = -R.T @ t
    best = np.full((height, width), np.inf)
    nrm = np.zeros((height, width, 3))
    val = np.zeros((height, width))
    for r in scene():
        den = rays @ r["n"]
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = ((r["c"] - C) @ r["n"]) / den
        P = C + lam[..., None] * rays
        du, dv = (P - r["c"]) @ r["u"], (P - r["c"]) @ r["v"]
        hit = (lam > 1e-6) & (np.abs(du) <= r["hu"]) & (np.abs(dv) <= r["hv"]) & (lam < best)
        best[hit] = lam[hit]
        off = 130.0 * r["face"]
        val[hit] = _sample(tex, ((du[hit] + r["hu"]) * texels + off % 600) % (tex.shape[1] - 1),
                           ((dv[hit] + r["hv"]) * texels + off % 400) % (tex.shape[0] - 1))
        nrm[hit] = r["n"]
    X = C + best[..., None] * rays
    depth = best                                    # the z of lam * (a, b, 1) is lam
    n_c = nrm @ R.T
    flip = np.sum(n_c * rays_c, -1) > 0
    n_c[flip] = -n_c[flip]
    return val.astype(np.float32), depth, n_c, X


def render(n, width, height, seed=0, dists=None, texels=TEXELS):
    """n views of the scene: Ks, Rs, ts and per view (image, depth, normal, world points)."""
    Ks, Rs, ts = cameras(n, width, height, seed)
    tex = _texture()
    views = [cast(Ks[a], Rs[a], ts[a], width, height, (0.0, 0.0) if dists is None else dists[a], tex, texels)
             for a in range(n)]
    return Ks, Rs, ts, views


def visible_in(views, Ks, Rs, ts, a, b, tol=0.01):
    """Pixels of view a whose surface point view b sees (in its image and not occluded, within a relative tol)."""
    X = views[a][3]                                 # infinite where the ray misses the scene
    with np.errstate(divide="ignore", invalid="ignore"):
        Y = X @ Rs[b].T + ts[b]
        z = Y[..., 2]
        u = (Y @ Ks[b].T)
        px, py = u[..., 0] / z, u[..., 1] / z
    H, W = views[b][1].shape
    ok = (z > 0) & (px >= 0) & (px <= W - 1) & (py >= 0) & (py <= H - 1)
    qx = np.clip(np.rint(np.nan_to_num(px)), 0, W - 1).astype(int)
    qy = np.clip(np.rint(np.nan_to_num(py)), 0, H - 1).astype(int)
    return ok & (np.abs(views[b][1][qy, qx] - z) <= tol * z)
