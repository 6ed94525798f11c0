"""Open surfaces for the screened Poisson mesher's tests: a wavy height field over [-1, 1]^2 with upward normals, seen
from one side only, and the distance of points to it."""
import numpy as np


def sheet_height(x, y):
    return 0.15 * np.sin(2 * x) * np.cos(1.5 * y)


def sheet(n, seed=0):
    """An open height field z = 0.15 sin 2x cos 1.5y over [-1, 1]^2 with upward unit normals."""
    rng = np.random.default_rng(seed)
    x, y = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    z = sheet_height(x, y)
    nrm = np.stack([-0.3 * np.cos(2 * x) * np.cos(1.5 * y), 0.225 * np.sin(2 * x) * np.sin(1.5 * y), np.ones(n)], 1)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return np.stack([x, y, z], 1).astype(np.float32), nrm.astype(np.float32)


def sheet_distance(P, samples=201, steps=20):
    """Distance of points P [n, 3] to the sheet's surface: from the nearest of a sample of the surface, Gauss-Newton on
    the foot point (x, y), kept inside [-1, 1]^2."""
    from scipy.spatial import cKDTree
    P = np.asarray(P, np.float64)
    u = np.linspace(-1, 1, samples)
    X, Y = np.meshgrid(u, u)
    S = np.stack([X.ravel(), Y.ravel(), sheet_height(X, Y).ravel()], 1)
    xy = S[cKDTree(S).query(P)[1], :2].copy()
    for _ in range(steps):
        x, y = xy[:, 0], xy[:, 1]
        hx, hy = 0.3 * np.cos(2 * x) * np.cos(1.5 * y), -0.225 * np.sin(2 * x) * np.sin(1.5 * y)
        r = np.stack([x - P[:, 0], y - P[:, 1], sheet_height(x, y) - P[:, 2]], 1)
        J = np.zeros((len(P), 3, 2))
        J[:, 0, 0] = J[:, 1, 1] = 1.0
        J[:, 2, 0], J[:, 2, 1] = hx, hy
        JtJ = np.einsum("nki,nkj->nij", J, J)
        xy = np.clip(xy - np.linalg.solve(JtJ, np.einsum("nki,nk->ni", J, r)[..., None])[..., 0], -1, 1)
    foot = np.stack([xy[:, 0], xy[:, 1], sheet_height(xy[:, 0], xy[:, 1])], 1)
    return np.linalg.norm(P - foot, axis=1)
