"""Cases for cs_texture_mesh_bp (rule 4b; tests/test_texture_bp_*.py): a triangle strip whose face graph is a path, the
island that ICM keeps and BP removes, and case-level inputs (candidates and adjacency, no images) for random paths."""
import numpy as np

import texture_cases as tc
import texture_oracle as to


def strip(n=40, seed=60):
    """A strip of 2n faces, one cell high, with face ids reversed along it (deep_strip's layout), seen by the pixel
    camera and two oblique ones: a path graph on which BP is exact."""
    c = 20.0 + 4 * n / 2
    v, t = tc.pixel_grid(20, 20, n, 1, 4, f=400.0, cx=c, cy=22.0)
    t = t.reshape(2, n, 3).transpose(1, 0, 2).reshape(-1, 3)[::-1]
    v[:, 2] += np.random.default_rng(seed).uniform(-0.5, 0.5, len(v)) * 4
    Ks, Rs, ts = tc._with(tc.pix(400.0, c, 22.0), tc.oblique([0.0, 0.0, 400.0], 256, 64,
                                                               [(-120.0, 10.0, -400.0), (130.0, -10.0, -400.0)],
                                                               seed=seed + 1))
    imgs = tc._images([(44, 4 * n + 40), (64, 256), (64, 256)], seed=seed + 2)
    return tc._case(imgs, Ks, Rs, ts, v, t, lam=0.5, dataTerm=1, outlierK=0.0, atlasWidth=1024)


def path_order(nbr):
    """The faces of a path graph from one end to the other."""
    deg = (np.asarray(nbr) >= 0).sum(1)
    f, prev, out = int(np.flatnonzero(deg == 1)[0]), -1, []
    while f >= 0:
        out.append(f)
        nxt = [int(g) for g in nbr[f] if g >= 0 and g != prev]
        prev, f = f, (nxt[0] if nxt else -1)
    return out


ISLAND = (3, 6)            # the run of faces, in path order, that prefers the second view
ISLAND_DELTA = 0.3         # the target D of the first view on the run


def island(seed=62):
    """Rule 4b's reason: a 10-face strip seen by two copies of the pixel camera.  The first image is noise; the second
    is the same noise scaled per face (by the depth buffer's owner of each pixel), by 1 / (1 - 0.3) over the run of 3
    faces in the middle and by 0.6 elsewhere.  Under GMI q is about area (g + 1), so the outer faces prefer view 0
    (D(1) about 0.4) and the run prefers view 1 with D(0) about 0.3: under lambda 0.5 the start labelling has two
    seams (E = 1.0), no single flip lowers E, and labelling the run 0 gives E about 0.9."""
    v, t = tc.pixel_grid(8, 8, 5, 1, 16, cx=48.0, cy=16.0)
    K = tc.pix(100.0, 48.0, 16.0)
    W, H = 96, 32
    buf = to.depth_buffer(K, np.eye(3), np.zeros(3), W, H, v, t)
    owner = (buf & np.uint64(0xFFFFFFFF)).astype(np.int64)
    owner[buf == to.EMPTY] = -1
    order = path_order(to.adjacency(t))
    gain = np.full(len(t), 0.6)
    gain[order[ISLAND[0]:ISLAND[1]]] = 1.0 / (1.0 - ISLAND_DELTA)
    base = np.random.default_rng(seed).uniform(0, 255, (H, W))
    scaled = base * np.where(owner >= 0, gain[np.maximum(owner, 0)], 1.0)
    return tc._case([base, scaled], [K, K], [np.eye(3)] * 2, [np.zeros(3)] * 2, v, t, lam=0.5, dataTerm=1,
                    outlierK=0.0) | dict(order=order)


def random_path(n, rng):
    """Case-level inputs of a path of n faces: faces (i, i + 1, i + 2), so face i shares edge (i + 1, i + 2) with face
    i + 1 and no other; 1 to 5 candidates per face from 6 views, q in (0.2, 1].  Returns (tris, nbr, col, cands)."""
    tris = np.stack([np.arange(n), np.arange(n) + 1, np.arange(n) + 2], 1)
    nbr = to.adjacency(tris)
    col, _ = to.colouring(nbr)
    cands = []
    for _ in range(n):
        k = int(rng.integers(1, 6))
        views = rng.choice(6, k, replace=False)
        cands.append(to.best_candidates([(float(rng.uniform(0.2, 1.0)), int(a)) for a in views]))
    return tris, nbr, col, cands


def viterbi(cands, lam):
    """The exact minimum of rule 4's E on a path (faces in order, each adjacent to the next): a labelling."""
    n = len(cands)
    D = [[1.0 - q / c[0][0] for q, _ in c] for c in cands]
    cost, back = list(D[0]), []
    for i in range(1, n):
        prev = [a for _, a in cands[i - 1]]
        cur = [a for _, a in cands[i]]
        nc, bk = [], []
        for r, a in enumerate(cur):
            best = min(range(len(prev)), key=lambda s: cost[s] + (lam if prev[s] != a else 0.0))
            nc.append(cost[best] + (lam if prev[best] != a else 0.0) + D[i][r])
            bk.append(best)
        cost, back = nc, back + [bk]
    r = int(np.argmin(cost))
    out = [r]
    for bk in reversed(back):
        r = bk[r]
        out.append(r)
    out.reverse()
    return np.array([cands[i][r][1] for i, r in enumerate(out)], np.int64)


CASES = {"strip": strip, "island": island}
