"""Float64 restatement of cs_poisson_mesh_screened (include/cudasift_b200.h): the Neumann graph Laplacian as a
scipy.sparse matrix, the edge-divergence right-hand side, the point weights B and omega, the exact coarse screening and
its diagonals, the V-cycle on L_l + diag(s_l) and its explicit matrix, MGPCG, the iso-value and the whole call.  The
grid, the splat, the interpolation and the extraction are tests/mesh_oracle.py's."""
import itertools

import numpy as np
import scipy.sparse as sp

import mesh_oracle as mo

NU, NU_COARSE = mo.NU, mo.NU_COARSE


# ---- operator, right-hand side, screening ---------------------------------------------------------------------------
def _path(m):
    """The graph Laplacian of a path of m nodes."""
    d = np.full(m, 2.0)
    d[0] = d[-1] = 1.0
    return sp.diags([-np.ones(m - 1), d, -np.ones(m - 1)], [-1, 0, 1])


def laplacian(n):
    """L on all (n + 1)^3 nodes of a level with n cells (x fastest): deg_q on the diagonal, -1 per in-grid neighbour."""
    T, I = _path(n + 1), sp.identity(n + 1)
    return (sp.kron(sp.kron(I, I), T) + sp.kron(sp.kron(I, T), I) + sp.kron(sp.kron(T, I), I)).tocsr()


def degree(n):
    """deg_q (z, y, x): the number of in-grid neighbours."""
    e = np.full(n + 1, 2.0)
    e[0] = e[-1] = 1.0
    return e[:, None, None] + e[None, :, None] + e[None, None, :]


def rhs(V, h):
    """b (float32, (z, y, x)): the divergence of the edge field (h / 2)(V_a(q) + V_a(q + e_a)) over the in-grid edges,
    in the header's order (per axis the central difference, or the one-sided sum at a face, then (h/2)((x + y) + z))."""
    V = V.astype(np.float64)
    d = []
    for a, ax in enumerate((2, 1, 0)):                  # V[a] is indexed (z, y, x): axis a of the grid is array axis ax
        Va = np.moveaxis(V[a], ax, 0)
        t = np.empty_like(Va)
        t[1:-1] = Va[2:] - Va[:-2]
        t[0] = Va[0] + Va[1]
        t[-1] = -(Va[-2] + Va[-1])
        d.append(np.moveaxis(t, 0, ax))
    return (h / 2 * ((d[0] + d[1]) + d[2])).astype(np.float32)


def weights(g, n):
    """B as a sparse [P, (n + 1)^3] matrix: point p's weights prod (1 - |g_a - q_a|) at the corners of its cell
    clamp(floor(g), 0, n - 1)."""
    g = np.asarray(g, np.float64)
    n1 = n + 1
    c = np.clip(np.floor(g).astype(np.int64), 0, n - 1)
    rows, cols, vals = [], [], []
    for bz, by, bx in itertools.product((0, 1), repeat=3):
        q = c + np.array([bx, by, bz])
        rows.append(np.arange(len(g)))
        cols.append((q[:, 2] * n1 + q[:, 1]) * n1 + q[:, 0])
        vals.append(np.prod(1.0 - np.abs(g - q), axis=1))
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                         shape=(len(g), n1 ** 3))


def omega(alpha, D, g, N):
    """alpha / the mean density at the points (mesh_oracle's interpolation, as info_out[5])."""
    return alpha / float(mo.interpolate(D, g, N).mean())


def level_sizes(N):
    out, n = [], N
    while n >= 4:
        out.append(n)
        n //= 2
    return out


def diagonals(g, N, w):
    """s_l (z, y, x) for every level: (w / 2^l) sum_p (B^l_p(Q))^2 at the level-l coordinates g / 2^l."""
    out = []
    for l, n in enumerate(level_sizes(N)):
        B = weights(np.asarray(g) / 2 ** l, n)
        out.append((w / 2 ** l * np.asarray(B.multiply(B).sum(0)).reshape(-1)).reshape((n + 1,) * 3))
    return out


def prolongation(nc):
    """P from a level of nc cells to one of 2 nc (trilinear, every node) as a sparse matrix."""
    m = 2 * nc + 1
    rows, cols, vals = [], [], []
    for i in range(m):
        cs = [i // 2] if i % 2 == 0 else [i // 2, i // 2 + 1]
        rows += [i] * len(cs)
        cols += cs
        vals += [1.0 / len(cs)] * len(cs)
    P1 = sp.csr_matrix((vals, (rows, cols)), shape=(m, nc + 1))
    return sp.kron(sp.kron(P1, P1), P1).tocsr()


def system(xyz, normal, depth, scale, alpha):
    """(A, b (float32, (z, y, x)), omega, sorted g, N, o, h, D, the levels' diagonals)."""
    g, nh, _, N, o, h, ok, _ = mo.sorted_points(xyz, normal, None, depth, scale)
    assert ok
    V, D, _ = mo.splat(g, nh, None, N)
    b = rhs(V, h)
    w = omega(alpha, D, g, N)
    B = weights(g, N)
    A = (laplacian(N) + w * (B.T @ B)).tocsr()
    return A, b, w, g, N, o, h, D, diagonals(g, N, w)


# ---- V-cycle and MGPCG ----------------------------------------------------------------------------------------------
def _nbr(x):
    y = np.zeros_like(x)
    for ax in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[ax], hi[ax] = slice(0, -1), slice(1, None)
        y[tuple(lo)] += x[tuple(hi)]
        y[tuple(hi)] += x[tuple(lo)]
    return y


def _sweep(x, f, dg, colour):
    n = x.shape[0] - 1
    k, j, i = np.ogrid[:n + 1, :n + 1, :n + 1]
    mask = (i + j + k) % 2 == colour
    x[mask] = ((f + _nbr(x)) / dg)[mask]


def _pairs(x, f, dg, pairs, red_first):
    for _ in range(pairs):
        _sweep(x, f, dg, 0 if red_first else 1)
        _sweep(x, f, dg, 1 if red_first else 0)


def v_cycle(f, s, l=0):
    """The header's V-cycle from x = 0 on level l (f full (z, y, x); s: the diagonals of every level)."""
    n = f.shape[0] - 1
    dg = degree(n) + s[l]
    x = np.zeros_like(f, dtype=np.float64)
    if l == len(s) - 1:
        _pairs(x, f, dg, NU_COARSE, True)
        _pairs(x, f, dg, NU_COARSE, False)
        return x
    _pairs(x, f, dg, NU, True)
    t = f - (dg * x - _nbr(x))
    P = prolongation(n // 2)
    fc = (0.5 * (P.T @ t.reshape(-1))).reshape((n // 2 + 1,) * 3)
    x += (P @ v_cycle(fc, s, l + 1).reshape(-1)).reshape(x.shape)
    _pairs(x, f, dg, NU, False)
    return x


def v_cycle_matrix(s):
    """The V-cycle on level 0 as an explicit matrix."""
    n = s[0].shape[0] - 1
    m = (n + 1) ** 3
    out = np.zeros((m, m))
    for c in range(m):
        e = np.zeros(m)
        e[c] = 1.0
        out[:, c] = v_cycle(e.reshape((n + 1,) * 3), s).reshape(-1)
    return out


def mgpcg(A, b, s, tol, max_iter):
    """The header's MGPCG in float64 on A with the V-cycle on s: (chi (z, y, x), iterations, |r| / |b|)."""
    shape = b.shape
    b = b.astype(np.float64).reshape(-1)
    x = np.zeros_like(b)
    r = b.copy()
    bb = float(b @ b)
    rr = bb
    k = 0
    if rr <= tol * tol * bb:
        return x.reshape(shape), 0, 0.0
    z = v_cycle(r.reshape(shape), s).reshape(-1)
    p = z.copy()
    rz = float(r @ z)
    while True:
        q = A @ p
        pq = float(p @ q)
        if not pq > 0:
            break
        alpha = rz / pq
        x += alpha * p
        r -= alpha * q
        rr = float(r @ r)
        k += 1
        if rr <= tol * tol * bb or k >= max_iter:
            break
        z = v_cycle(r.reshape(shape), s).reshape(-1)
        rzn = float(r @ z)
        p = z + rzn / rz * p
        rz = rzn
    return x.reshape(shape), k, np.sqrt(rr / bb) if bb > 0 else 0.0


# ---- the whole call -------------------------------------------------------------------------------------------------
def mesh(xyz, normal, intensity=None, depth=6, scale=1.1, alpha=4.0, trim=0.0, chi=None, tau=None, tol=1e-10):
    """The whole call in float64 with a tight MGPCG solve (or a given chi and tau): a dict with the mesh, chi, b, D,
    tau, dbar, omega, o, h, the iterations to tol."""
    g, nh, I, N, o, h, ok, used = mo.sorted_points(xyz, normal, intensity, depth, scale)
    assert ok
    V, D, S = mo.splat(g, nh, I, N)
    b = rhs(V, h)
    w = omega(alpha, D, g, N)
    B = weights(g, N)
    A = (laplacian(N) + w * (B.T @ B)).tocsr()
    s = diagonals(g, N, w)
    iters = None
    if chi is None:
        chi, iters, _ = mgpcg(A, b, s, tol, 1000)
    t = float(mo.interpolate(chi, g, N).mean()) if tau is None else tau
    dbar = float(mo.interpolate(D, g, N).mean())
    out = mo.extract(chi, t, o, h, D, S, trim, dbar)
    out.update(chi=chi, b=b, D=D, S=S, tau=t, dbar=dbar, omega=w, o=o, h=h, N=N, g=g, A=A, s=s, iters=iters)
    return out


def on_faces(verts, o, h, N):
    """Whether each vertex lies on a face of the grid's box (to float rounding of the vertex position)."""
    q = (np.asarray(verts, np.float64) - np.asarray(o)) / h
    tol = 1e-4
    return ((np.abs(q) < tol) | (np.abs(q - N) < tol)).any(1)


def boundary_edge_vertices(tris):
    """The vertex pairs of the directed edges whose reverse does not appear."""
    e = mo.directed_edges(tris)
    key = e[:, 0] * (e.max() + 1) + e[:, 1]
    rkey = e[:, 1] * (e.max() + 1) + e[:, 0]
    return e[~np.isin(rkey, key)]
