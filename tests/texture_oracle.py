"""cs_texture_mesh restated in float64 (numpy element-wise operations, each rounded once, in the header's order): the
input check, the adjacency, the depth buffers, the candidates, the Jones-Plassmann colouring, the ICM sweeps, the energy
totals in coop.cuh's three-level order, the charts, the shelf packing, the texture coordinates and the atlas."""
import math

import numpy as np

MCAND = 8
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
TILE, THREADS = 2048, 256


def tie_of(f):
    m = (np.asarray(f, np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)
    return m ^ (m >> np.uint64(16))


def validate(verts, tris):
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    if len(t) == 0:
        return True
    if t.min() < 0 or t.max() >= len(verts):
        return False
    if ((t[:, 0] == t[:, 1]) | (t[:, 1] == t[:, 2]) | (t[:, 0] == t[:, 2])).any():
        return False
    return bool(np.isfinite(np.asarray(verts, np.float32)[np.unique(t)]).all())


def project(K, R, t, X):
    """(u, v, z) of the float64 points X [..., 3]: Y = R X + t, (u, v) = (K Y)_{0,1} / Y_z, in the header's order."""
    x, y, z = X[..., 0], X[..., 1], X[..., 2]
    Y = [((R[i, 0] * x + R[i, 1] * y) + R[i, 2] * z) + t[i] for i in range(3)]
    u = ((K[0, 0] * Y[0] + K[0, 1] * Y[1]) + K[0, 2] * Y[2]) / Y[2]
    v = ((K[1, 0] * Y[0] + K[1, 1] * Y[1]) + K[1, 2] * Y[2]) / Y[2]
    return u, v, Y[2]


def centre(R, t):
    return np.array([-((R[0, i] * t[0] + R[1, i] * t[1]) + R[2, i] * t[2]) for i in range(3)])


def area2(u, v):
    return (u[..., 1] - u[..., 0]) * (v[..., 2] - v[..., 0]) - (v[..., 1] - v[..., 0]) * (u[..., 2] - u[..., 0])


def adjacency(tris):
    """nbr [T, 3]: the face across edge k (corner k -> k + 1) of each face when exactly two faces hold the edge."""
    t = np.asarray(tris, np.int64)
    T = len(t)
    a, b = t, np.roll(t, -1, axis=1)
    key = (np.minimum(a, b) << 32) | np.maximum(a, b)
    key = key.reshape(-1)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    nbr = np.full(3 * T, -1, np.int64)
    for i in pair_starts(ks):
        c1, c2 = order[i], order[i + 1]
        nbr[c1], nbr[c2] = c2 // 3, c1 // 3
    return nbr.reshape(T, 3)


def pair_starts(ks):
    """The positions i of the sorted edge keys where a run of exactly two equal keys starts."""
    n = len(ks)
    return [i for i in range(n - 1)
            if not ((i > 0 and ks[i - 1] == ks[i]) or ks[i + 1] != ks[i] or (i + 2 < n and ks[i + 2] == ks[i]))]


def depth_buffer(K, R, t, W, H, verts, tris):
    """The keys (float(depth) bits << 32) | face of one image [H, W] (EMPTY where no face covers the pixel)."""
    buf = np.full(H * W, EMPTY, np.uint64)
    for f, pix, d in face_depths(K, R, t, W, H, verts, tris):
        combine(buf, pix, d, f)
    return buf.reshape(H, W)


def covers(w0, w1, w2, S):
    return (w0 >= 0) & (w1 >= 0) & (w2 >= 0) & (S > 0)


def combine(buf, pix, d, f):
    """The pixels pix of face f with their float64 depths d into the buffer: the depth rounded to float once, then the
    key's 64-bit minimum (the nearer float depth wins, ties go to the lower face)."""
    key = (d.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(f)
    np.minimum.at(buf, pix, key)


def face_depths(K, R, t, W, H, verts, tris):
    """Per rasterised face: (face, the flat indices y W + x of its covered pixels, their float64 depths)."""
    X = np.asarray(verts, np.float32).astype(np.float64)
    tr = np.asarray(tris, np.int64)
    u, v, z = project(K, R, t, X[tr])
    A = area2(u, v)
    with np.errstate(invalid="ignore"):
        ok = (z > 0).all(1) & (A != 0) & np.isfinite(A)
        xlo = np.maximum(0.0, np.ceil(np.minimum(np.minimum(u[:, 0], u[:, 1]), u[:, 2])))
        xhi = np.minimum(W - 1.0, np.floor(np.maximum(np.maximum(u[:, 0], u[:, 1]), u[:, 2])))
        ylo = np.maximum(0.0, np.ceil(np.minimum(np.minimum(v[:, 0], v[:, 1]), v[:, 2])))
        yhi = np.minimum(H - 1.0, np.floor(np.maximum(np.maximum(v[:, 0], v[:, 1]), v[:, 2])))
        ok &= (xlo <= xhi) & (ylo <= yhi)
    for f in np.nonzero(ok)[0]:
        s = 1.0 if A[f] > 0 else -1.0
        ys, xs = np.mgrid[int(ylo[f]):int(yhi[f]) + 1, int(xlo[f]):int(xhi[f]) + 1]
        ys, xs = ys.reshape(-1).astype(np.float64), xs.reshape(-1).astype(np.float64)
        w = []
        for k in range(3):
            a, b = k, (k + 1) % 3
            lo = tr[f, a] < tr[f, b]
            P, Q = (a, b) if lo else (b, a)
            du, dv = u[f, Q] - u[f, P], v[f, Q] - v[f, P]
            w.append((s if lo else -s) * (du * (ys - v[f, P]) - dv * (xs - u[f, P])))
        S = (w[0] + w[1]) + w[2]
        cov = covers(w[0], w[1], w[2], S)
        if not cov.any():
            continue
        w0, w1, w2, S = w[0][cov], w[1][cov], w[2][cov], S[cov]
        iz = ((w1 / z[f, 0] + w2 / z[f, 1]) + w0 / z[f, 2]) / S
        yield f, ys[cov].astype(np.int64) * W + xs[cov].astype(np.int64), 1.0 / iz


def candidates(cams, bufs, verts, tris, maxViewAngleDeg, depthTol):
    """Per face its (q, image) candidates, best first, at most MCAND; and the count of all (face, image) pairs that
    passed."""
    X = np.asarray(verts, np.float32).astype(np.float64)
    tr = np.asarray(tris, np.int64)
    T = len(tr)
    p0, p1, p2 = X[tr[:, 0]], X[tr[:, 1]], X[tr[:, 2]]
    e1, e2 = p1 - p0, p2 - p0
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    cen = ((p0 + p1) + p2) / 3.0
    dot = lambda a, b: (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]
    ln = np.sqrt(dot(n, n))
    cosLim = math.cos(maxViewAngleDeg * math.pi / 180.0)
    fid = np.arange(T, dtype=np.uint64)
    lists = [[] for _ in range(T)]
    total = 0
    for a, (K, R, t, W, H) in enumerate(cams):
        d = centre(R, t)[None, :] - cen
        dn = dot(n, d)
        ok = (dn > 0) & (dn >= cosLim * (ln * np.sqrt(dot(d, d))))
        uv = []
        for P in (p0, p1, p2, cen):
            u, v, z = project(K, R, t, P)
            with np.errstate(invalid="ignore"):
                inside = (z > 0) & (u >= 0) & (u <= W - 1.0) & (v >= 0) & (v <= H - 1.0)
            px = np.where(inside, np.floor(u + 0.5), 0).astype(np.int64)
            py = np.where(inside, np.floor(v + 0.5), 0).astype(np.int64)
            key = bufs[a][py, px]
            dep = (key >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
            with np.errstate(invalid="ignore"):
                vis = (key == EMPTY) | ((key & np.uint64(0xFFFFFFFF)) == fid) | (z <= dep * (1.0 + depthTol))
            ok &= inside & vis
            uv.append((u, v))
        U = np.stack([uv[0][0], uv[1][0], uv[2][0]], 1)
        V = np.stack([uv[0][1], uv[1][1], uv[2][1]], 1)
        q = 0.5 * np.abs(area2(U, V))
        ok &= q > 0
        for f in np.nonzero(ok)[0]:
            lists[f].append((float(q[f]), a))
        total += int(ok.sum())
    return [best_candidates(c) for c in lists], total


def best_candidates(c):
    """A face's (q, image) pairs in image order: its best MCAND by (q descending, image ascending)."""
    return sorted(c, key=lambda e: (-e[0], e[1]))[:MCAND]


def colouring(nbr):
    """Jones-Plassmann rounds with priority s(f); returns (colour per face, rounds)."""
    T = len(nbr)
    pr = tie_of(np.arange(T)).astype(np.int64)
    col = np.full(T, -1, np.int64)
    rounds = 0
    while True:
        new = col.copy()
        left = 0
        for f in np.nonzero(col < 0)[0]:
            wins, held = True, set()
            for g in nbr[f]:
                if g < 0:
                    continue
                if col[g] < 0:
                    wins = wins and pr[f] > pr[g]
                else:
                    held.add(int(col[g]))
            if wins:
                c = 0
                while c in held:
                    c += 1
                new[f] = c
            else:
                left += 1
        col = new
        rounds += 1
        if left == 0:
            return col, rounds


def _butterfly(v):
    v = np.array(v, np.float64).reshape(-1, 32)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, lane ^ o]
    return v[:, 0]


def _cta_partial(v):
    w = _butterfly(v)
    s = w[0]
    for x in w[1:]:
        s = s + x
    return s


def tree_total(e):
    """coop.cuh's three-level total of e: tiles of 2048 items, groups of 256 tile partials, the group partials."""
    e = np.asarray(e, np.float64)
    n = len(e)
    tiles = (n + TILE - 1) // TILE
    part = []
    for t in range(tiles):
        acc = np.zeros(THREADS)
        for m in range(TILE // THREADS):
            i = t * TILE + m * THREADS + np.arange(THREADS)
            acc = acc + np.where(i < n, e[np.minimum(i, n - 1)], 0.0)
        part.append(_cta_partial(acc))
    groups = (tiles + THREADS - 1) // THREADS
    grp = []
    for g in range(groups):
        i = g * THREADS + np.arange(THREADS)
        grp.append(_cta_partial(np.where(i < tiles, np.array(part + [0.0])[np.minimum(i, tiles)], 0.0)))
    acc = np.zeros(32)
    for i in range(0, groups, 32):
        chunk = np.zeros(32)
        k = min(32, groups - i)
        chunk[:k] = grp[i:i + k]
        acc = acc + chunk
    return float(_butterfly(acc)[0])


def energy(label, cands, nbr, lam):
    T = len(label)
    e = np.zeros(T)
    for f in range(T):
        l = label[f]
        if l < 0:
            continue
        c = cands[f]
        r = [a for _, a in c].index(l)
        dis = sum(1 for g in nbr[f] if g > f and label[g] >= 0 and label[g] != l)
        e[f] = (1.0 - c[r][0] / c[0][0]) + lam * float(dis)
    return tree_total(e)


def texture(images, Ks, Rs, ts, verts, tris, lam=0.5, maxViewAngleDeg=75.0, depthTol=0.01, padding=2,
            atlasWidth=1024, maxSweeps=100, maxAtlasRows=None, maxCharts=None, bufs=None):
    """The whole call.  images are float32 [H, W]; bufs (the depth buffers) may be passed in when already computed.
    Returns a dict: atlas [full rows, atlasWidth] (the prefix of maxAtlasRows rows when given), uv [T, 3, 2], labels,
    faceChart, charts [C, 8] (the prefix of maxCharts), info [2], stats [11], the colours, the depth buffers, the
    candidates and the chart count (the return value)."""
    X = np.asarray(verts, np.float32)
    tr = np.asarray(tris, np.int64).reshape(-1, 3)
    T = len(tr)
    cams = [(np.asarray(Ks[a], np.float64), np.asarray(Rs[a], np.float64), np.asarray(ts[a], np.float64),
             images[a].shape[1], images[a].shape[0]) for a in range(len(images))]
    if T == 0:
        return dict(ret=0, stats=[0] * 11, info=[0.0, 0.0])
    if not validate(X, tr):
        return dict(ret=0, stats=[T] + [0] * 9 + [2], info=[0.0, 0.0])
    nbr = adjacency(tr)
    if bufs is None:
        bufs = [depth_buffer(K, R, t, W, H, X, tr) for K, R, t, W, H in cams]
    cands, total = candidates(cams, bufs, X, tr, maxViewAngleDeg, depthTol)
    label = np.array([c[0][1] if c else -1 for c in cands], np.int64)
    unseen = int((label < 0).sum())
    col, rounds = colouring(nbr)
    colours = int(col.max()) + 1
    e0 = energy(label, cands, nbr, lam)
    sweeps = changed = 0
    while True:
        if sweeps == maxSweeps:
            status = 3
            break
        ch = 0
        for c in range(colours):
            for f in np.nonzero((col == c) & (label >= 0))[0]:
                cf = cands[f]
                local = lambda a_q: (1.0 - a_q[0] / cf[0][0]) + lam * float(
                    sum(1 for g in nbr[f] if g >= 0 and label[g] >= 0 and label[g] != a_q[1]))
                cur = label[f]
                best, bestE = cur, local(cf[[a for _, a in cf].index(cur)])
                for e in cf:
                    x = local(e)
                    if x < bestE:
                        best, bestE = e[1], x
                if best != cur:
                    label[f] = best
                    ch += 1
        sweeps += 1
        changed += ch
        if ch == 0:
            status = 0
            break
    e1 = energy(label, cands, nbr, lam)
    root = chart_roots(label, nbr)
    roots = [f for f in range(T) if label[f] >= 0 and root[f] == f]
    idx = {r: c for c, r in enumerate(roots)}
    C = len(roots)
    raw = [[int(label[r]), 1 << 40, 1 << 40, -(1 << 40), -(1 << 40), 0] for r in roots]
    Xd = X.astype(np.float64)
    faceChart = np.full(T, -1, np.int64)
    proj = {}
    for f in range(T):
        if label[f] < 0:
            continue
        c = idx[root[f]]
        faceChart[f] = c
        K, R, t, W, H = cams[label[f]]
        u, v, _ = project(K, R, t, Xd[tr[f]])
        proj[f] = (u, v)
        e = raw[c]
        e[1] = min(e[1], int(np.floor(u).min()))
        e[2] = min(e[2], int(np.floor(v).min()))
        e[3] = max(e[3], int(np.ceil(u).max()))
        e[4] = max(e[4], int(np.ceil(v).max()))
        e[5] += 1
    table = np.zeros((C, 8), np.int64)
    for c, e in enumerate(raw):
        x0, y0, x1, y1 = chart_rect(e, cams[e[0]][3], cams[e[0]][4], padding)
        table[c] = [e[0], x0, y0, x1 - x0 + 1, y1 - y0 + 1, 0, 0, e[5]]
    full = pack(table, atlasWidth)
    rows = full if maxAtlasRows is None else min(full, maxAtlasRows)
    atlas = np.zeros((full, atlasWidth), np.float32)
    for c in range(C):
        a, x0, y0, w, h, ox, oy = table[c, :7]
        atlas[oy:oy + h, ox:ox + w] = images[a][y0:y0 + h, x0:x0 + w]
    uv = np.full((T, 3, 2), np.nan, np.float32)
    for f, (u, v) in proj.items():
        e = table[faceChart[f]]
        uv[f, :, 0] = ((u - float(e[1])) + float(e[5])).astype(np.float32)
        uv[f, :, 1] = ((v - float(e[2])) + float(e[6])).astype(np.float32)
    stats = [T, unseen, total, colours, rounds, sweeps, changed, C, int(full), int(rows), status]
    return dict(ret=C, atlas=atlas[:rows], uv=uv, labels=label.astype(np.int32), faceChart=faceChart.astype(np.int32),
                charts=table[:C if maxCharts is None else min(C, maxCharts)].astype(np.int32), info=[e0, e1],
                stats=stats, colours=col, bufs=bufs, cands=cands, nbr=nbr, start=np.array(
                    [c[0][1] if c else -1 for c in cands], np.int64))


def chart_roots(label, nbr):
    """Rule 5's union-find: per face the root of its chart, the lowest face of the chart (every link from the higher
    root to the lower); unseen faces are their own roots."""
    T = len(label)
    parent = np.arange(T)

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x
    for f in range(T):
        for g in nbr[f]:
            if g > f and label[f] >= 0 and label[g] == label[f]:
                a, b = find(f), find(g)
                if a != b:
                    parent[max(a, b)] = min(a, b)
    return np.array([find(f) for f in range(T)])


def chart_rect(e, W, H, padding):
    """(x0, y0, x1, y1) of a chart's raw rectangle e {image, xmin, ymin, xmax, ymax, faces}, padded and clamped."""
    return max(0, e[1] - padding), max(0, e[2] - padding), min(W - 1, e[3] + padding), min(H - 1, e[4] + padding)


def pack(table, atlasWidth):
    """Rule 6's shelves over the chart table [C, 8] (ox, oy written in place); returns the full atlas height."""
    C = len(table)
    order = sorted(range(C), key=lambda c: (-table[c, 4], -table[c, 3], c))
    shelfY = shelfH = cx = 0
    for c in order:
        if cx + table[c, 3] > atlasWidth:
            shelfY += shelfH
            shelfH = cx = 0
        table[c, 5], table[c, 6] = cx, shelfY
        cx += table[c, 3]
        shelfH = max(shelfH, table[c, 4])
    return shelfY + shelfH
