"""Float64 restatement of cs_poisson_mesh (include/cudasift_b200.h): used points, grid, the splat, the right-hand side,
the operator as a scipy.sparse matrix, a tight solve, the V-cycle and MGPCG, the iso-value, marching tetrahedra with the
header's order and orientation rules, trimming, compaction and vertex intensity, plus mesh topology helpers."""
import itertools

import numpy as np
import scipy.sparse as sp
import scipy.sparse.csgraph as csg
import scipy.sparse.linalg as spla

DIRS = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1)]
PERMS = list(itertools.permutations(range(3)))          # lexicographic
NU, NU_COARSE = 2, 8


# ---- grid and splat -------------------------------------------------------------------------------------------------
def grid(xyz, normal, depth, scale):
    """(used mask, unit normals [used], N, o [3], h, ok)."""
    X = np.asarray(xyz, np.float32).astype(np.float64)
    Nr = np.asarray(normal, np.float32).astype(np.float64)
    N = 1 << depth
    with np.errstate(invalid="ignore", over="ignore"):
        ln = np.sqrt((Nr ** 2).sum(1))
        used = np.isfinite(X).all(1) & np.isfinite(Nr).all(1) & (ln > 0)
    if not used.any():
        return used, None, N, np.zeros(3), 0.0, False
    lo, hi = X[used].min(0), X[used].max(0)
    E = float((hi - lo).max())
    L = max(scale, N / (N - 8)) * E
    h = L / N
    o = (lo + hi) / 2 - L / 2
    return used, Nr[used] / ln[used, None], N, o, h, E > 0


def sorted_points(xyz, normal, intensity, depth, scale):
    """The used points in the header's sorted order: (g [U, 3], n^ [U, 3], I [U] or None, N, o, h, ok, used mask)."""
    used, nh, N, o, h, ok = grid(xyz, normal, depth, scale)
    if not ok:
        return None, None, None, N, o, h, ok, used
    X = np.asarray(xyz, np.float32).astype(np.float64)[used]
    g = (X - o) / h
    c = np.clip(np.floor(g).astype(np.int64), 0, N - 1)
    key = (c[:, 2] * N + c[:, 1]) * N + c[:, 0]
    order = np.argsort(key, kind="stable")
    I = None if intensity is None else np.asarray(intensity, np.float32).astype(np.float64)[used][order]
    return g[order], nh[order], I, N, o, h, ok, used


def splat(g, nh, I, N):
    """V [3, n1, n1, n1], D, S (or None) as float32 arrays indexed (z, y, x), summed in float64."""
    n1 = N + 1
    V = np.zeros((3, n1 ** 3))
    D = np.zeros(n1 ** 3)
    S = np.zeros(n1 ** 3) if I is not None else None
    c = np.clip(np.floor(g).astype(np.int64), 0, N - 1)
    for bz, by, bx in itertools.product((0, 1), repeat=3):
        q = c + np.array([bx, by, bz])
        w = np.prod(1.0 - np.abs(g - q), axis=1)
        idx = (q[:, 2] * n1 + q[:, 1]) * n1 + q[:, 0]
        for a in range(3):
            np.add.at(V[a], idx, w * nh[:, a])
        np.add.at(D, idx, w)
        if S is not None:
            np.add.at(S, idx, w * I)
    sh = (n1, n1, n1)
    return (V.reshape((3,) + sh).astype(np.float32), D.reshape(sh).astype(np.float32),
            None if S is None else S.reshape(sh).astype(np.float32))


def rhs(V, h):
    """b (float32, (z, y, x)): (h / 2) sum_a (V_a(q + e_a) - V_a(q - e_a)) at interior nodes, 0 on the boundary."""
    V = V.astype(np.float64)
    b = np.zeros(V.shape[1:])
    dx = V[0][1:-1, 1:-1, 2:] - V[0][1:-1, 1:-1, :-2]
    dy = V[1][1:-1, 2:, 1:-1] - V[1][1:-1, :-2, 1:-1]
    dz = V[2][2:, 1:-1, 1:-1] - V[2][:-2, 1:-1, 1:-1]
    b[1:-1, 1:-1, 1:-1] = h / 2 * ((dx + dy) + dz)
    return b.astype(np.float32)


# ---- operator and solves --------------------------------------------------------------------------------------------
def operator(n):
    """A on the (n - 1)^3 interior nodes of a level with n cells (x fastest): 6 on the diagonal, -1 per neighbour."""
    m = n - 1
    T = sp.diags([-np.ones(m - 1), np.zeros(m), -np.ones(m - 1)], [-1, 0, 1])
    I = sp.identity(m)
    return (6 * sp.kron(sp.kron(I, I), I) + sp.kron(sp.kron(I, I), T) + sp.kron(sp.kron(I, T), I)
            + sp.kron(sp.kron(T, I), I)).tocsr()


def interior(a):
    return a[1:-1, 1:-1, 1:-1].reshape(-1)


def embed(x, n):
    out = np.zeros((n + 1,) * 3)
    out[1:-1, 1:-1, 1:-1] = x.reshape((n - 1,) * 3)
    return out


def solve(b, n, rtol=1e-13):
    """A chi = b on the interior by CG to rtol (float64); chi (z, y, x) with a zero boundary."""
    A = operator(n)
    bi = interior(b).astype(np.float64)
    x, info = spla.cg(A, bi, rtol=rtol, atol=0.0, maxiter=20000)
    assert info == 0
    return embed(x, n)


def _apply(x):
    """A x on a full (z, y, x) array, 0 on the boundary."""
    y = np.zeros_like(x)
    c = x[1:-1, 1:-1, 1:-1]
    y[1:-1, 1:-1, 1:-1] = 6 * c - (x[1:-1, 1:-1, :-2] + x[1:-1, 1:-1, 2:] + x[1:-1, :-2, 1:-1] + x[1:-1, 2:, 1:-1]
                                   + x[:-2, 1:-1, 1:-1] + x[2:, 1:-1, 1:-1])
    return y


def _sweep(x, f, colour):
    n = x.shape[0] - 1
    k, j, i = np.meshgrid(*(np.arange(n + 1),) * 3, indexing="ij")
    mask = ((i + j + k) % 2 == colour)
    mask[0, :, :] = mask[-1, :, :] = mask[:, 0, :] = mask[:, -1, :] = mask[:, :, 0] = mask[:, :, -1] = False
    nb = np.zeros_like(x)
    nb[1:-1, 1:-1, 1:-1] = (x[1:-1, 1:-1, :-2] + x[1:-1, 1:-1, 2:] + x[1:-1, :-2, 1:-1] + x[1:-1, 2:, 1:-1]
                            + x[:-2, 1:-1, 1:-1] + x[2:, 1:-1, 1:-1])
    x[mask] = (f[mask] + nb[mask]) / 6.0


def _pairs(x, f, pairs, red_first):
    for _ in range(pairs):
        _sweep(x, f, 0 if red_first else 1)
        _sweep(x, f, 1 if red_first else 0)


def restrict(t):
    """(1/2) P^T t on the coarse interior (0 on the coarse boundary)."""
    n = t.shape[0] - 1
    nc = n // 2
    out = np.zeros((nc + 1,) * 3)
    for dz, dy, dx in itertools.product((-1, 0, 1), repeat=3):
        w = (0.5 if dx else 1.0) * (0.5 if dy else 1.0) * (0.5 if dz else 1.0)
        out[1:-1, 1:-1, 1:-1] += w * t[2 + dz:n - 1 + dz:2, 2 + dy:n - 1 + dy:2, 2 + dx:n - 1 + dx:2]
    return 0.5 * out


def _interp_axis(a, axis):
    nc = a.shape[axis] - 1
    shape = list(a.shape)
    shape[axis] = 2 * nc + 1
    out = np.zeros(shape)
    even, odd, lo, hi = ([slice(None)] * 3 for _ in range(4))
    even[axis], odd[axis], lo[axis], hi[axis] = slice(0, None, 2), slice(1, None, 2), slice(0, -1), slice(1, None)
    out[tuple(even)] = a
    out[tuple(odd)] = 0.5 * (a[tuple(lo)] + a[tuple(hi)])
    return out


def prolong(xc):
    """P xc on the fine grid (trilinear), zero on the fine boundary."""
    out = _interp_axis(_interp_axis(_interp_axis(xc, 2), 1), 0)
    out[0, :, :] = out[-1, :, :] = out[:, 0, :] = out[:, -1, :] = out[:, :, 0] = out[:, :, -1] = 0
    return out


def v_cycle(f):
    """The header's V-cycle from x = 0 on a level of n cells (f: full (z, y, x) array, boundary ignored)."""
    n = f.shape[0] - 1
    x = np.zeros_like(f, dtype=np.float64)
    if n <= 4:
        _pairs(x, f, NU_COARSE, True)
        _pairs(x, f, NU_COARSE, False)
        return x
    _pairs(x, f, NU, True)
    t = f - _apply(x)
    t[0, :, :] = t[-1, :, :] = t[:, 0, :] = t[:, -1, :] = t[:, :, 0] = t[:, :, -1] = 0
    x += prolong(v_cycle(restrict(t)))
    _pairs(x, f, NU, False)
    return x


def mgpcg(b, tol, max_iter):
    """The header's MGPCG in float64: (chi, iterations, recurrence |r| / |b|)."""
    b = b.astype(np.float64)
    x = np.zeros_like(b)
    r = b.copy()
    bb = float((b * b).sum())
    rr = bb
    k = 0
    if rr <= tol * tol * bb:
        return x, 0, 0.0
    z = v_cycle(r)
    p = z.copy()
    rz = float((r * z).sum())
    while True:
        q = _apply(p)
        pq = float((p * q).sum())
        if not pq > 0:
            break
        alpha = rz / pq
        x += alpha * p
        r -= alpha * q
        rr = float((r * r).sum())
        k += 1
        if rr <= tol * tol * bb or k >= max_iter:
            break
        z = v_cycle(r)
        rzn = float((r * z).sum())
        p = z + rzn / rz * p
        rz = rzn
    return x, k, np.sqrt(rr / bb) if bb > 0 else 0.0


def v_cycle_matrix(n):
    """The V-cycle on a level of n cells as an explicit matrix on the interior unknowns."""
    m = (n - 1) ** 3
    B = np.zeros((m, m))
    for c in range(m):
        e = np.zeros(m)
        e[c] = 1.0
        B[:, c] = interior(v_cycle(embed(e, n)))
    return B


def interpolate(F, g, N):
    """Trilinear interpolation of the node array F (z, y, x) at grid coordinates g [P, 3]."""
    c = np.clip(np.floor(g).astype(np.int64), 0, N - 1)
    t = g - c
    out = np.zeros(len(g))
    F = F.astype(np.float64)
    for bz, by, bx in itertools.product((0, 1), repeat=3):
        w = ((t[:, 0] if bx else 1 - t[:, 0]) * (t[:, 1] if by else 1 - t[:, 1]) * (t[:, 2] if bz else 1 - t[:, 2]))
        out += w * F[c[:, 2] + bz, c[:, 1] + by, c[:, 0] + bx]
    return out


# ---- extraction -----------------------------------------------------------------------------------------------------
def _tet_table():
    """For each tetrahedron (perm) and each inside pattern of its 4 chain corners (bit v: corner v inside): the list of
    triangles as 3 (corner a, corner b) bit-pattern pairs, with the header's order and orientation."""
    table = []
    for perm in PERMS:
        cor = [0, 1 << perm[0], (1 << perm[0]) | (1 << perm[1]), 7]
        pos = [np.array([(c >> a) & 1 for a in range(3)], float) for c in cor]
        rows = []
        for code in range(16):
            ins = [v for v in range(4) if (code >> v) & 1]
            outs = [v for v in range(4) if not (code >> v) & 1]
            if len(ins) in (0, 4):
                rows.append([])
                continue
            if len(ins) in (1, 3):
                a = ins[0] if len(ins) == 1 else outs[0]
                others = outs if len(ins) == 1 else ins
                cyc = [(a, o) for o in others]
            else:
                a, b = ins
                c, d = outs
                cyc = [(a, c), (a, d), (b, d), (b, c)]
            mids = [(pos[u] + pos[w]) / 2 for u, w in cyc]
            n = np.cross(mids[1] - mids[0], mids[2] - mids[0])
            towards = np.mean([pos[v] for v in outs], 0) - np.mean([pos[v] for v in ins], 0)
            if n @ towards < 0:
                cyc = [cyc[0]] + cyc[1:][::-1]
            tris = [cyc[:3]] if len(cyc) == 3 else [[cyc[0], cyc[1], cyc[2]], [cyc[0], cyc[2], cyc[3]]]
            rows.append([[(cor[u], cor[w]) for u, w in t] for t in tris])
        table.append((cor, rows))
    return table


TET_TABLE = _tet_table()
_DIR_OF = {1: 0, 2: 1, 4: 2, 3: 3, 5: 4, 6: 5, 7: 6}


def _edge_of(a, b):
    lo, hi = a & b, a | b
    return np.array([lo & 1, (lo >> 1) & 1, (lo >> 2) & 1]), _DIR_OF[hi & ~lo]


def extract(chi, tau, o=(0.0, 0.0, 0.0), h=1.0, D=None, S=None, trim=0.0, dbar=0.0):
    """Marching tetrahedra of the node array chi (z, y, x; any size) at tau.  Returns a dict: vertices [V, 3]
    (float32), triangles [T, 3], intensity [V] or None, the pre-trim counts, the kept-vertex edge ids, densities."""
    chi = np.asarray(chi, np.float32).astype(np.float64)
    nz, ny, nx = chi.shape
    inside = chi >= tau
    M = chi.size
    # crossing edges and vertex ids (ascending edge id = node-major, direction-minor)
    cross = np.zeros((nz, ny, nx, 7), bool)
    for d, (dx, dy, dz) in enumerate(DIRS):
        a = inside[:nz - dz, :ny - dy, :nx - dx]
        b = inside[dz:, dy:, dx:]
        cross[:nz - dz, :ny - dy, :nx - dx, d] = a != b
    flat = cross.reshape(M, 7)
    eid = np.nonzero(flat.reshape(-1))[0]
    vid = -np.ones(M * 7, np.int64)
    vid[eid] = np.arange(len(eid))
    node, d = eid // 7, eid % 7
    k, j, i = node // (ny * nx), (node // nx) % ny, node % nx
    delta = np.array(DIRS)[d]
    chia = chi.reshape(-1)[node]
    chib = chi[k + delta[:, 2], j + delta[:, 1], i + delta[:, 0]]
    t = (tau - chia) / (chib - chia)
    q = np.stack([i, j, k], 1).astype(np.float64)
    verts = (np.asarray(o, np.float64) + h * (q + t[:, None] * delta)).astype(np.float32)

    def lerp(F):
        F = F.astype(np.float64)
        a = F.reshape(-1)[node]
        return a + t * (F[k + delta[:, 2], j + delta[:, 1], i + delta[:, 0]] - a)

    dens = lerp(D) if D is not None else np.zeros(len(eid))
    # triangles in (cell, tet, k) order
    cz, cy, cx = np.meshgrid(np.arange(nz - 1), np.arange(ny - 1), np.arange(nx - 1), indexing="ij")
    cz, cy, cx = cz.reshape(-1), cy.reshape(-1), cx.reshape(-1)
    cell = (cz * (ny - 1) + cy) * (nx - 1) + cx
    keys, tris = [], []
    for ti, (cor, rows) in enumerate(TET_TABLE):
        code = np.zeros(len(cell), np.int64)
        for v, c in enumerate(cor):
            code |= inside[cz + ((c >> 2) & 1), cy + ((c >> 1) & 1), cx + (c & 1)].astype(np.int64) << v
        for cd in range(16):
            sel = np.nonzero(code == cd)[0]
            if len(sel) == 0:
                continue
            for kk, tri in enumerate(rows[cd]):
                ids = []
                for a, b in tri:
                    off, dd = _edge_of(a, b)
                    nidx = ((cz[sel] + off[2]) * ny + cy[sel] + off[1]) * nx + cx[sel] + off[0]
                    ids.append(vid[nidx * 7 + dd])
                tris.append(np.stack(ids, 1))
                keys.append(cell[sel] * 12 + ti * 2 + kk)
    if tris:
        keys = np.concatenate(keys)
        tris = np.concatenate(tris)[np.argsort(keys, kind="stable")]
    else:
        tris = np.zeros((0, 3), np.int64)
    assert (tris >= 0).all()
    V0, T0 = len(verts), len(tris)
    keep = np.ones(len(tris), bool)
    if D is not None:
        keep = ~(dens[tris] < trim * dbar).any(1)
    tris = tris[keep]
    ref = np.zeros(len(verts), bool)
    ref[tris.reshape(-1)] = True
    remap = np.cumsum(ref) - 1
    inten = None
    if S is not None:
        den = lerp(D)
        num = lerp(S)
        with np.errstate(invalid="ignore", divide="ignore"):
            inten = np.where(den != 0, num / np.where(den != 0, den, 1), 0.0).astype(np.float32)[ref]
    return dict(vertices=verts[ref], triangles=remap[tris].astype(np.int64), intensity=inten, pre=(V0, T0),
                edges=eid[ref], density=dens[ref], marginal=None)


def mesh(xyz, normal, intensity=None, depth=6, scale=1.1, trim=0.0, chi=None, tau=None):
    """The whole call in float64 with a tight solve (or a given chi and tau): a dict with the mesh, chi, b, D, tau,
    dbar, o, h."""
    g, nh, I, N, o, h, ok, used = sorted_points(xyz, normal, intensity, depth, scale)
    assert ok
    V, D, S = splat(g, nh, I, N)
    b = rhs(V, h)
    if chi is None:
        chi = solve(b, N)
    t = float(interpolate(chi, g, N).mean()) if tau is None else tau
    dbar = float(interpolate(D, g, N).mean())
    out = extract(chi, t, o, h, D, S, trim, dbar)
    out.update(chi=chi, b=b, D=D, S=S, tau=t, dbar=dbar, o=o, h=h, N=N, g=g)
    return out


# ---- topology -------------------------------------------------------------------------------------------------------
def directed_edges(tris):
    t = np.asarray(tris, np.int64)
    return np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])


def closed_and_oriented(tris):
    """Every directed edge appears exactly once and its reverse exactly once."""
    e = directed_edges(tris)
    if len(e) == 0:
        return True
    key = e[:, 0] * (e.max() + 1) + e[:, 1]
    rkey = e[:, 1] * (e.max() + 1) + e[:, 0]
    u, cnt = np.unique(key, return_counts=True)
    return bool((cnt == 1).all() and np.isin(rkey, u).all())


def boundary_edges(tris):
    """Directed edges whose reverse does not appear."""
    e = directed_edges(tris)
    key = e[:, 0] * (e.max() + 1) + e[:, 1]
    rkey = e[:, 1] * (e.max() + 1) + e[:, 0]
    return int((~np.isin(rkey, key)).sum())


def euler(tris):
    t = np.asarray(tris, np.int64)
    e = directed_edges(t)
    und = np.unique(np.sort(e, 1), axis=0)
    return len(np.unique(t)) - len(und) + len(t)


def components(tris, nv):
    t = np.asarray(tris, np.int64)
    e = directed_edges(t)
    G = sp.coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(nv, nv))
    n, lab = csg.connected_components(G, directed=False)
    return len(np.unique(lab[np.unique(t)]))
