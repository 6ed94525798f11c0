"""Meshes and views for mesh texturing (cs_texture_mesh): the rectangles of stereo_cases.scene() as grids of triangles
facing outward (the box's faces away from its centre, the other rectangles towards the cameras), with a jittered
variant, seen by stereo_cases.render's views; a sphere seen by a ring of cameras; and a flat grid facing a camera."""
import numpy as np

import stereo_cases as sc
from triangulate_cases import look_at

BOX_CENTRE = np.array([-0.9, 0.5, 1.6])


def _grid(r, cell, toward):
    nu, nv = max(2, int(np.ceil(2 * r["hu"] / cell))), max(2, int(np.ceil(2 * r["hv"] / cell)))
    a, b = np.meshgrid(np.linspace(-r["hu"], r["hu"], nu + 1), np.linspace(-r["hv"], r["hv"], nv + 1))
    P = r["c"] + a.reshape(-1, 1) * r["u"] + b.reshape(-1, 1) * r["v"]
    idx = np.arange((nu + 1) * (nv + 1)).reshape(nv + 1, nu + 1)
    q00, q10, q01, q11 = idx[:-1, :-1], idx[:-1, 1:], idx[1:, :-1], idx[1:, 1:]
    t = np.concatenate([np.stack([q00, q10, q11], -1).reshape(-1, 3), np.stack([q00, q11, q01], -1).reshape(-1, 3)])
    if np.dot(r["n"], toward) < 0:          # (u, v, n) is right-handed: the triangles above face +n
        t = t[:, ::-1]
    border = np.zeros((nv + 1, nu + 1), bool)
    border[[0, -1], :] = True
    border[:, [0, -1]] = True
    return P, t, border.reshape(-1)


def scene_mesh(cell=0.6, jitter=0.0, seed=0, Rs=None, ts=None):
    """The scene as one triangle soup of separate rectangles (vertices float32 [V, 3], triangles int32 [T, 3]).
    jitter moves every interior vertex by up to jitter * cell in 3-D."""
    if Rs is None:
        _, Rs, ts = sc.cameras(6, 160, 120)
    C = np.mean([-R.T @ t for R, t in zip(Rs, ts)], axis=0)
    rng = np.random.default_rng(seed)
    vs, tr, n = [], [], 0
    for r in sc.scene():
        toward = r["c"] - BOX_CENTRE if 2 <= r["face"] <= 6 else C - r["c"]
        P, t, border = _grid(r, cell, toward)
        if jitter:
            P = P + np.where(border[:, None], 0.0, rng.uniform(-jitter * cell, jitter * cell, P.shape))
        vs.append(P)
        tr.append(t + n)
        n += len(P)
    return np.concatenate(vs).astype(np.float32), np.concatenate(tr).astype(np.int32)


def scene_views(n=6, width=160, height=120, seed=0):
    """stereo_cases.render's views: (images float32 [H, W] list, Ks, Rs, ts, views)."""
    Ks, Rs, ts, views = sc.render(n, width, height, seed=seed)
    return [v[0] for v in views], Ks, Rs, ts, views


def ring_cameras(n, width, height, centre, radius, seed=0):
    """n cameras on a tilted ring around centre looking at it."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = [], [], []
    for a in range(n):
        ang = 2 * np.pi * a / n + rng.uniform(-0.05, 0.05)
        C = centre + radius * np.array([np.cos(ang), 0.35 * np.sin(3 * ang), np.sin(ang)])
        R = look_at(C, centre + rng.uniform(-0.05, 0.05, 3), rng.uniform(-0.1, 0.1))
        f = width * rng.uniform(0.9, 1.1)
        Ks.append(np.array([[f, 0.0, width / 2 + rng.uniform(-3, 3)], [0, f, height / 2 + rng.uniform(-3, 3)],
                            [0, 0, 1.0]]))
        Rs.append(R)
        ts.append(-R @ C)
    return np.array(Ks), np.array(Rs), np.array(ts)


def flat_grid(n=8, step=10.0, jitter=0.0, seed=0):
    """A z = 5 grid of n x n cells, each `step` pixels wide, seen straight on by one camera (K = diag(5, 5, 1) with the
    principal point at (20, 20)): its vertices project to integer pixels, so its edges pass through pixel centres, or
    near them with jitter (the border stays put).  Returns (verts,
    tris, K, R, t, W, H, (x_lo, x_hi, y_lo, y_hi) the grid's pixel rectangle)."""
    rng = np.random.default_rng(seed)
    W = H = int(n * step + 40)
    K = np.array([[5.0, 0, 20.0], [0, 5.0, 20.0], [0, 0, 1.0]])
    a, b = np.meshgrid(np.arange(n + 1) * step, np.arange(n + 1) * step)
    px = np.stack([a.reshape(-1), b.reshape(-1)], 1)
    inner = (a.reshape(-1) > 0) & (a.reshape(-1) < n * step) & (b.reshape(-1) > 0) & (b.reshape(-1) < n * step)
    if jitter:
        px = px + np.where(inner[:, None], rng.uniform(-jitter * step, jitter * step, px.shape), 0.0)
    z = 5.0
    X = np.concatenate([px, np.full((len(px), 1), z)], 1)        # u = (5 x + 20 z) / z = x + 20
    idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1)
    q00, q10, q01, q11 = idx[:-1, :-1], idx[:-1, 1:], idx[1:, :-1], idx[1:, 1:]
    t = np.concatenate([np.stack([q00, q11, q10], -1).reshape(-1, 3), np.stack([q00, q01, q11], -1).reshape(-1, 3)])
    return (X.astype(np.float32), t.astype(np.int32), K, np.eye(3), np.zeros(3), W, H,
            (20, 20 + int(n * step), 20, 20 + int(n * step)))
