"""Meshes and views for mesh texturing (cs_texture_mesh): the rectangles of stereo_cases.scene() as grids of triangles
facing outward (the box's faces away from its centre, the other rectangles towards the cameras), with a jittered
variant, seen by stereo_cases.render's views; a sphere seen by a ring of cameras; a flat grid facing a camera; and
one case per rule of cs_texture_mesh with its images, cameras and arguments (pixel grids, occluders, coplanar copies,
many and mixed-size views, labelling, charts, atlas packing, and more than 2^21 faces)."""
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


# ---- cases that reach each rule of cs_texture_mesh (tests/test_texture_rules_*.py) -------------------------------------
# Each generator returns a dict: imgs (float32 [H, W] list), Ks, Rs, ts, v (float32 [V, 3]), t (int32 [T, 3]) and kw,
# the call's arguments by texture_oracle.texture's names (lam, maxViewAngleDeg, depthTol, padding, atlasWidth,
# maxSweeps); groups, when present, the texture_group_bytes caps to run it under as well.
# A pixel camera pix(f, cx, cy) has K = [[f, 0, cx], [0, f, cy], [0, 0, 1]], R = I and t = 0.  The point at depth
# z = depth f that it sees at pixel (x, y) is ((x - cx) depth, (y - cy) depth, depth f): at depth 1 and 2 every
# coordinate of an integer pixel is an integer, and the projection gives the pixel back exactly.


def pix(f=100.0, cx=64.0, cy=64.0):
    return np.array([[f, 0, cx], [0, f, cy], [0, 0, 1.0]])


def _case(imgs, Ks, Rs, ts, v, t, **kw):
    return dict(imgs=[np.ascontiguousarray(im, np.float32) for im in imgs], Ks=np.asarray(Ks, np.float64),
                Rs=np.asarray(Rs, np.float64), ts=np.asarray(ts, np.float64), v=np.asarray(v, np.float32),
                t=np.asarray(t, np.int32), kw=kw)


def _images(shapes, seed):
    rng = np.random.default_rng(seed)
    return [rng.uniform(0, 255, s).astype(np.float32) for s in shapes]


def _at_pixels(px, py, f, cx, cy, depth):
    return np.stack([(px - cx) * depth, (py - cy) * depth, np.full(len(px), depth * f)], 1)


def pixel_grid(x0, y0, nx, ny, step, f=100.0, cx=64.0, cy=64.0, depth=1.0, jitter=0.0, seed=0):
    """An nx x ny grid of cells `step` pixels wide whose vertices pix(f, cx, cy) sees at pixels (x0 + i step,
    y0 + j step) and depth depth * f, triangulated as flat_grid (facing the camera); jitter moves the interior
    vertices in the image plane by up to jitter * step.  Returns (verts float64 [V, 3], tris int64 [T, 3])."""
    rng = np.random.default_rng(seed)
    a, b = np.meshgrid(x0 + np.arange(nx + 1) * step, y0 + np.arange(ny + 1) * step)
    px, py = a.reshape(-1).astype(np.float64), b.reshape(-1).astype(np.float64)
    if jitter:
        i, j = np.meshgrid(np.arange(nx + 1), np.arange(ny + 1))
        inner = ((i > 0) & (i < nx) & (j > 0) & (j < ny)).reshape(-1)
        px = px + np.where(inner, rng.uniform(-jitter * step, jitter * step, len(px)), 0.0)
        py = py + np.where(inner, rng.uniform(-jitter * step, jitter * step, len(py)), 0.0)
    idx = np.arange((nx + 1) * (ny + 1)).reshape(ny + 1, nx + 1)
    q00, q10, q01, q11 = idx[:-1, :-1], idx[:-1, 1:], idx[1:, :-1], idx[1:, 1:]
    t = np.concatenate([np.stack([q00, q11, q10], -1).reshape(-1, 3), np.stack([q00, q01, q11], -1).reshape(-1, 3)])
    return _at_pixels(px, py, f, cx, cy, depth), t


def join(*parts):
    """One mesh of several (verts, tris) parts, vertex ids offset."""
    vs, ts, n = [], [], 0
    for v, t in parts:
        vs.append(np.asarray(v, np.float64))
        ts.append(np.asarray(t, np.int64) + n)
        n += len(v)
    return np.concatenate(vs), np.concatenate(ts)


def oblique(target, W, H, offsets, seed=0):
    """Cameras at target + offset looking at target (focal about W, images W x H), one per offset."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = [], [], []
    for o in offsets:
        C = np.asarray(target, np.float64) + np.asarray(o, np.float64)
        R = look_at(C, np.asarray(target, np.float64), rng.uniform(-0.2, 0.2))
        Ks.append(np.array([[W * rng.uniform(0.9, 1.1), 0, W / 2 + rng.uniform(-2, 2)],
                            [0, W * rng.uniform(0.9, 1.1), H / 2 + rng.uniform(-2, 2)], [0, 0, 1.0]]))
        Rs.append(R)
        ts.append(-R @ C)
    return Ks, Rs, ts


def _with(K0, more):
    """The pixel camera K0 first, then oblique()'s cameras."""
    Ks, Rs, ts = more
    return [K0] + list(Ks), [np.eye(3)] + list(Rs), [np.zeros(3)] + list(ts)


def _relabel(v, t, seed, unused=0):
    """Vertex ids permuted, `unused` extra vertices (every third NaN) that no face uses, and the faces in random
    order."""
    rng = np.random.default_rng(seed)
    extra = rng.uniform(-50, 50, (unused, 3))
    extra[::3] = np.nan
    allv = np.concatenate([v, extra])
    perm = rng.permutation(len(allv))               # old vertex i is new vertex perm[i]
    nv = np.empty_like(allv)
    nv[perm] = allv
    return nv, perm[t][rng.permutation(len(t))]


def topology():
    """Rule 1: a pixel grid with one edge held by 3 faces and one by 4 (fins towards the camera), an isolated face
    repeated with its corners rotated (adjacent to its copy across all three edges), boundary edges; the vertex ids
    permuted, unused vertices with NaN coordinates, the faces in random order; the pixel camera and 3 oblique ones."""
    v, t = pixel_grid(20, 20, 8, 8, 10)
    extra, n = [], len(v)
    for (a, b), k in (((10, 20), 1), ((40, 41), 2)):    # (10, 20) is a grid diagonal, (40, 41) a row edge
        for j in range(k):
            extra.append(0.5 * (v[a] + v[b]) + np.array([0.3 + j, -0.7 - j, -4.0 - 2.0 * j]))
            t = np.concatenate([t, [[a, b, n]]])
            n += 1
    extra += list(_at_pixels(np.array([104.0, 112, 112]), np.array([24.0, 32, 24]), 100.0, 64.0, 64.0, 0.9))
    t = np.concatenate([t, [[n, n + 1, n + 2], [n + 1, n + 2, n]]])
    v, t = _relabel(np.concatenate([v, extra]), t, seed=3, unused=40)
    Ks, Rs, ts = _with(pix(), oblique([-4.0, -4.0, 100.0], 160, 120, [(-60, 20, -180), (70, -30, -170),
                                                                       (10, 80, -160)], seed=1))
    return _case(_images([(120, 120)] + [(120, 160)] * 3, seed=4), Ks, Rs, ts, v, t, lam=0.5)


def occluder(jitter=0.0):
    """Rule 2: an occluder grid at depth 100 whose vertices the pixel camera sees at integer pixels (or near them with
    jitter), in front of separate faces at depth 200.  Each back face has its corners on an occluder cell's corner
    (x, y) and on the cell's edges from it ((x + 10, y) and (x, y + 10), or (x + 6, y) and (x, y + 6)), and its
    centroid (x + 10/3, y + 10/3) or (x + 2, y + 2) rounds to a pixel on the cell's diagonal: all four of its sample
    pixels lie on the occluder's edges and vertices.  A pixel the rasteriser drops there leaves the sample unoccluded,
    and with all four dropped the back face becomes a candidate of the pixel camera."""
    v, t = pixel_grid(20, 20, 8, 8, 10, jitter=jitter, seed=5)
    pts = []
    for i in range(8):
        for j in range(8):
            x, y, s = 20 + 10 * i, 20 + 10 * j, 10 if (i + j) % 2 else 6
            pts += [(x, y), (x, y + s), (x + s, y)]
    pts = np.array(pts, np.float64)
    v, t = join((v, t), (_at_pixels(pts[:, 0], pts[:, 1], 100.0, 64.0, 64.0, 2.0), np.arange(len(pts)).reshape(-1, 3)))
    Ks, Rs, ts = _with(pix(), oblique([-4.0, -4.0, 100.0], 120, 120, [(-30, 20, -200)], seed=2))
    return _case(_images([(120, 120), (120, 120)], seed=6), Ks, Rs, ts, v, t, lam=0.5)


def coplanar(depthTol=0.0):
    """Rule 2 at depthTol 0: a tilted jittered grid and a second copy of every face on its own copies of the
    vertices, corners rotated, the faces in random order.  The copies' float64 depths may differ in their last bits
    and round to the same float: the tie order (the lower face wins) and the float rounding of the stored depth
    decide which copy sees itself."""
    rng = np.random.default_rng(7)
    v, t = pixel_grid(20, 20, 6, 6, 12, jitter=0.3, seed=7)
    v[:, 2] += 0.13 * v[:, 0] - 0.21 * v[:, 1] + rng.uniform(-1.0, 1.0, len(v))
    v = v.astype(np.float32).astype(np.float64)
    v, t = join((v, t), (v, t[:, [1, 2, 0]]))
    Ks, Rs, ts = _with(pix(), oblique([-8.0, -8.0, 100.0], 160, 120, [(-50, 30, -180), (60, -20, -170)], seed=3))
    return _case(_images([(120, 120)] + [(120, 160)] * 2, seed=8), Ks, Rs, ts, v, t[rng.permutation(len(t))],
                 lam=0.5, depthTol=depthTol)


def raster_edges():
    """Rule 2's faces without pixels, and clipped boxes: a grid in the plane y = 0 through camera 0's centre (its
    principal row 64, a power of two, so every projected v is exactly 64 and A == 0); a plane crossing camera 1's
    Y_z = 0; two faces larger than every image; small faces straddling each border and corner of camera 0's image."""
    a, b = np.meshgrid(np.linspace(-2, 2, 7), np.linspace(2, 6, 7))
    P = np.stack([a.reshape(-1), np.zeros(49), b.reshape(-1)], 1)
    idx = np.arange(49).reshape(7, 7)
    g = np.concatenate([np.stack([idx[:-1, :-1], idx[1:, 1:], idx[:-1, 1:]], -1).reshape(-1, 3),
                        np.stack([idx[:-1, :-1], idx[:-1, 1:], idx[1:, 1:]], -1).reshape(-1, 3)[::2]])
    a, b = np.meshgrid(np.linspace(-3, 3, 9), np.linspace(-2, 2, 5))
    Q = np.stack([a.reshape(-1), b.reshape(-1) + 0.5, 6.0 + 2.5 * a.reshape(-1)], 1)
    idx = np.arange(45).reshape(5, 9)
    q = np.concatenate([np.stack([idx[:-1, :-1], idx[1:, 1:], idx[:-1, 1:]], -1).reshape(-1, 3),
                        np.stack([idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:]], -1).reshape(-1, 3)])
    big = np.array([[-30.0, -30, 8], [30, -30, 8], [-30, 30, 8], [30, 30, 8]])
    bt = np.array([[0, 3, 1], [0, 2, 3]])
    s = []                                          # camera 0: 128 x 128, f 100; at depth 3 a pixel is 0.03
    for cx, cy in ((0, 40), (127, 80), (50, 0), (90, 127), (0, 0), (127, 127)):
        X, Y = (cx - 64) * 0.03, (cy - 64) * 0.03
        s.append([[X - 0.2, Y - 0.2, 3.0], [X - 0.2, Y + 0.25, 3.0], [X + 0.25, Y - 0.2, 3.0]])
    s = np.array(s).reshape(-1, 3)
    v, t = join((P, g), (Q, q), (big, bt), (s, np.arange(len(s)).reshape(-1, 3)[:, [0, 2, 1]]))
    C1, C2 = np.array([0.0, 0.5, 4.0]), np.array([0.5, 3.0, -2.0])
    R1, R2 = look_at(C1, np.array([1.0, 0.5, 8.5]), 0.0), look_at(C2, np.array([0.0, 0.0, 4.0]), 0.1)
    Ks = [pix(), np.array([[80.0, 0, 50], [0, 80, 40], [0, 0, 1]]), np.array([[90.0, 0, 61], [0, 90, 47], [0, 0, 1]])]
    return _case(_images([(128, 128), (80, 100), (94, 122)], seed=9), Ks, [np.eye(3), R1, R2],
                 [np.zeros(3), -R1 @ C1, -R2 @ C2], v, t, lam=0.5)


def many_views(maxViewAngleDeg=75.0):
    """Rule 3: a bumpy pixel grid seen by 15 cameras at lambda 0: 11 oblique ones, of which 5 and 10 come twice
    (images 5 and 6, 11 and 12: equal q, the image-ascending tie), then the pixel camera twice (images 13 and 14),
    the best view of most faces.  So faces have more than 8 passing images, their 8th and 9th can tie, the best 8
    are not the first 8 found, and a tie for the best view decides the label."""
    rng = np.random.default_rng(10)
    v, t = pixel_grid(20, 20, 10, 10, 8, cx=60.0, cy=60.0, jitter=0.25, seed=10)
    v[:, 2] += rng.uniform(-3.0, 3.0, len(v))
    offs = [(rng.uniform(-60, 60), rng.uniform(-60, 60), -rng.uniform(150, 220)) for _ in range(11)]
    Ks, Rs, ts = (list(x) for x in oblique([0.0, 0.0, 100.0], 96, 80, offs, seed=11))
    imgs = _images([(80, 96)] * 11 + [(120, 120)], seed=12)
    Ks.append(pix(cx=60.0, cy=60.0)), Rs.append(np.eye(3)), ts.append(np.zeros(3))
    for k in (11, 10, 5):                           # camera and image k again at k + 1
        for a in (Ks, Rs, ts, imgs):
            a.insert(k + 1, a[k].copy())
    return _case(imgs, Ks, Rs, ts, v, t, lam=0.0, maxViewAngleDeg=maxViewAngleDeg)


def depth_ratio(depthTol=0.01):
    """Rule 3's depth test: a front strip at depth 100 over part of a back grid whose depth runs from 98.4 to 103.2
    across the image (the same pixels), so the back grid's samples under the strip sit at depth ratios on both sides
    of 1 + depthTol."""
    f, ft = pixel_grid(20, 20, 8, 2, 10)
    b, bt = pixel_grid(20, 20, 8, 8, 10)
    b = b * (0.984 + 0.048 * (b[:, 0] + 44.0) / 80.0)[:, None]
    v, t = join((f, ft), (b, bt))
    Ks, Rs, ts = _with(pix(), oblique([-4.0, -4.0, 100.0], 120, 100, [(-40, 15, -200), (45, -25, -190)], seed=13))
    return _case(_images([(120, 120), (100, 120), (100, 120)], seed=14), Ks, Rs, ts, v, t, lam=0.5, depthTol=depthTol)


def image_groups(shapes, cap):
    """The call's image groups: consecutive images while their buffers (8 bytes per pixel) fit cap, one at least."""
    groups, acc = 1, 0
    for a, (h, w) in enumerate(shapes):
        b = 8 * h * w
        if a > 0 and acc + b > cap:
            groups, acc = groups + 1, 0
        acc += b
    return groups


MIXED_SHAPES = [(2, 2), (5, 3), (29, 37), (50, 63), (9, 4095), (119, 161), (119, 161), (61, 45), (3, 7)]


def mixed_sizes():
    """Rule 3 over images of every size (2 x 2 to 4095 wide, widths not multiples of 4) and over image groups: images
    5 and 6 are one camera and image twice.  groups: a cap that puts images 0 to 3 in one group, image 4 (9 x 4095,
    larger than the cap) alone, splits the pair 5 | 6 and puts 6, 7 and 8 together; a cap 1 byte lower, which moves
    the boundary to 6 | 7; and 1 byte (an image per group)."""
    rng = np.random.default_rng(15)
    v, t = pixel_grid(20, 20, 16, 16, 5, jitter=0.2, seed=15)
    v[:, 2] += rng.uniform(-2.0, 2.0, len(v))
    target = np.array([-4.0, -4.0, 100.0])
    Ks, Rs, ts = [], [], []
    for k, (H, W) in enumerate(MIXED_SHAPES):
        if k == 6:
            Ks.append(Ks[5]), Rs.append(Rs[5]), ts.append(ts[5])
            continue
        C = target + np.array([rng.uniform(-30, 30), rng.uniform(-30, 30), -200.0])
        R = look_at(C, target, rng.uniform(-0.2, 0.2))
        f = max(W, H) * 1.3 if max(W, H) < 1000 else 300.0
        Ks.append(np.array([[f, 0, (W - 1) / 2 + 0.3], [0, f, (H - 1) / 2 - 0.2], [0, 0, 1.0]]))
        Rs.append(R)
        ts.append(-R @ C)
    imgs = _images(MIXED_SHAPES, seed=16)
    imgs[6] = imgs[5].copy()
    per = [8 * h * w for h, w in MIXED_SHAPES]
    cap = sum(per[:4]) + per[4] // 2
    return _case(imgs, Ks, Rs, ts, v, t, lam=0.5, atlasWidth=4096) | dict(groups=[cap, per[5] + per[7] - 1, 1])


def labelling(n=100, **kw):
    """Rule 4: a jittered bumpy n x n pixel grid (2 n^2 faces; 20 000 at n = 100, enough for 4 colours) seen by the
    pixel camera and 3 oblique ones, every 7th face turned away from every camera (unseen faces between seen ones)."""
    rng = np.random.default_rng(17)
    c = 20.0 + n
    v, t = pixel_grid(20, 20, n, n, 2, cx=c, cy=c, jitter=0.2, seed=17)
    v[:, 2] += rng.uniform(-0.8, 0.8, len(v))
    t[::7] = t[::7][:, [0, 2, 1]]
    d = 2.5 * n
    Ks, Rs, ts = _with(pix(cx=c, cy=c), oblique([0.0, 0.0, 100.0], 256, 224, [(-0.4 * d, 0.15 * d, -d),
                                                                                 (0.45 * d, -0.1 * d, -d),
                                                                                 (0.05 * d, 0.5 * d, -d)], seed=18))
    imgs = _images([(2 * n + 40, 2 * n + 40)] + [(224, 256)] * 3, seed=19)
    return _case(imgs, Ks, Rs, ts, v, t, **({"lam": 0.5} | kw))


def big_chart(n=224):
    """Rule 5: one chart of 2 n^2 >= 10^5 faces (n = 224: 100 352), faces and vertex ids in random order, seen by the
    pixel camera alone."""
    c = 20.0 + n
    v, t = pixel_grid(20, 20, n, n, 2, f=400.0, cx=c, cy=c)
    v, t = _relabel(v, t, seed=20)
    return _case(_images([(2 * n + 40, 2 * n + 40)], seed=21), [pix(400.0, c, c)], [np.eye(3)], [np.zeros(3)], v, t,
                 lam=0.5)


def deep_strip(n=3000):
    """Rule 5: a strip of 2n faces, one cell high, with face ids reversed along it, seen by the pixel camera: one
    chart whose union-find links run the whole strip."""
    c = 20.0 + n / 2
    v, t = pixel_grid(20, 20, n, 1, 1, f=2000.0, cx=c, cy=20.5)
    t = t.reshape(2, n, 3).transpose(1, 0, 2).reshape(-1, 3)[::-1]
    return _case(_images([(41, n + 40)], seed=22), [pix(2000.0, c, 20.5)], [np.eye(3)], [np.zeros(3)], v, t,
                 lam=0.5, atlasWidth=4096)


def single_charts():
    """Rule 5: lambda 0 on a grid with random depth jitter as large as its cells, seen from the left and from the
    right, so neighbouring faces often have different best views: many one-face charts."""
    rng = np.random.default_rng(23)
    v, t = pixel_grid(20, 20, 20, 20, 4, cx=60.0, cy=60.0)
    v[:, 2] += rng.uniform(-5.0, 5.0, len(v))
    Ks, Rs, ts = oblique([0.0, 0.0, 100.0], 120, 100, [(-90, 0, -150), (90, 0, -150)], seed=24)
    return _case(_images([(100, 120)] * 2, seed=25), Ks, Rs, ts, v, t, lam=0.0)


def atlas(padding=0):
    """Rules 5 and 6 on a 100 x 120 image of the pixel camera with atlasWidth 100, the widest image: a grid spanning
    every column (corners at u = 0 and u = W - 1 exactly; a chart as wide as the atlas), and two separate grids
    below it, 60 and 40 pixels wide, which fill their shelf exactly (cx + w == atlasWidth).  With padding 16 the
    rectangles are clamped at x = 0 and x = W - 1."""
    K = dict(cx=50.0, cy=60.0)
    top = pixel_grid(0, 2, 11, 3, 9, **K)           # u 0 .. 99, v 2 .. 29
    a = pixel_grid(40, 50, 6, 2, 9, **K)            # u 40 .. 94, and a face out to 99
    a = (np.concatenate([a[0], _at_pixels(np.array([99.0]), np.array([50.0]), 100.0, 50.0, 60.0, 1.0)]),
         np.concatenate([a[1], [[6, 13, len(a[0])]]]))
    b = pixel_grid(0, 50, 4, 2, 9, **K)             # u 0 .. 36, and a face out to 39
    b = (np.concatenate([b[0], _at_pixels(np.array([39.0]), np.array([50.0]), 100.0, 50.0, 60.0, 1.0)]),
         np.concatenate([b[1], [[4, 9, len(b[0])]]]))
    v, t = join(top, a, b)
    return _case(_images([(120, 100)], seed=26), [pix(100.0, 50.0, 60.0)], [np.eye(3)], [np.zeros(3)], v, t, lam=0.5,
                 padding=padding, atlasWidth=100)


def unseen():
    """Rule 6 with no face seen: a grid behind the camera and one turned away from it (C = 0, no atlas rows)."""
    v1, t1 = pixel_grid(20, 20, 4, 4, 10, depth=-1.0)
    v2, t2 = pixel_grid(20, 20, 4, 4, 10)
    v, t = join((v1, t1), (v2, t2[:, [0, 2, 1]]))
    return _case(_images([(80, 80)], seed=27), [pix()], [np.eye(3)], [np.zeros(3)], v, t, lam=0.5)


SCALE_FACES = (1 << 21) + 2048 + 7


def scale(T=SCALE_FACES, patches=96):
    """Past the launch shape's grid cap: T > 2^21 faces, so the per-face loops and the raster loop stride, and the
    energy total has several 256-tile groups.  Most faces are isolated triangles behind every camera; `patches`
    jittered 3 x 3-cell grids (18 faces each) are spread through the index range and seen by 4 images."""
    rng = np.random.default_rng(28)
    vis = []
    for p in range(patches):
        v, t = pixel_grid(20 + 24 * (p % 12), 20 + 24 * (p // 12), 3, 3, 6, cx=170.0, cy=120.0, jitter=0.2,
                          seed=100 + p)
        v[:, 2] += rng.uniform(-2.0, 2.0, len(v))
        vis.append((v, t))
    vv, vt = join(*vis)
    hidden = T - len(vt)
    tri = np.array([[0.0, 0, 0], [1.0, 0, 0], [0, 1.0, 0]])
    hv = (tri[None] + rng.uniform(-50, 50, (hidden, 1, 3)) * np.array([1.0, 1.0, 0.0])
          + np.array([0, 0, -200.0])).reshape(-1, 3)
    v, t = join((vv, vt), (hv, np.arange(3 * hidden).reshape(-1, 3)))
    pos = np.sort(rng.choice(T, len(vt), replace=False))    # where the visible faces go
    order = np.empty(T, np.int64)
    order[pos] = np.arange(len(vt))
    order[np.setdiff1d(np.arange(T), pos)] = len(vt) + np.arange(hidden)
    Ks, Rs, ts = _with(pix(cx=170.0, cy=120.0), oblique([0.0, 0.0, 100.0], 320, 240, [(-60, 20, -250),
                                                                                        (55, -15, -260),
                                                                                        (10, 60, -240)], seed=29))
    return _case(_images([(240, 340)] + [(240, 320)] * 3, seed=30), Ks, Rs, ts, v, t[order], lam=0.5)
