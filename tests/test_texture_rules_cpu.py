"""The texturing cases of tests/texture_cases.py reach the rules they are built for, shown on the oracle without a GPU:
(a) each case's precondition (no hole in the occluder's buffer, more than 8 passing images with a tie at rank 8/9,
depth rounding that decides visibility, 4 colours, the sweep cap, clamped padding, an exactly filled shelf, more than
2^21 faces, ...); (b) each oracle mutation of a rule changes the output of at least one case, so a kernel with the
same slip would fail the GPU comparison in test_texture_rules_gpu.py."""
import numpy as np
import pytest

import texture_cases as tc
import texture_oracle as to

_memo = {}


def _case(key, make):
    if key not in _memo:
        _memo[key] = make()
    return _memo[key]


def _texture(c):
    return to.texture(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], **c["kw"])


def _ref(key, make):
    k = ("ref",) + (key,)
    if k not in _memo:
        _memo[k] = _texture(_case(key, make))
    return _memo[k]


def _cam(c, a):
    return c["Ks"][a], c["Rs"][a], c["ts"][a], c["imgs"][a].shape[1], c["imgs"][a].shape[0]


def _samples(c, a):
    """Per face the (u, v, z) of its 4 sample points (corners, centroid) in image a."""
    K, R, t, W, H = _cam(c, a)
    X = np.asarray(c["v"], np.float64)[np.asarray(c["t"], np.int64)]
    P = np.concatenate([X, ((X[:, 0] + X[:, 1]) + X[:, 2])[:, None] / 3.0], 1)
    return to.project(K, R, t, P)


def _depth(key):
    return (key >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)


# ---- (a) preconditions ----------------------------------------------------------------------------------------------
def test_topology_reaches_rule_1():
    c = tc.topology()
    t = np.asarray(c["t"], np.int64)
    a, b = t, np.roll(t, -1, axis=1)
    _, counts = np.unique(((np.minimum(a, b) << 32) | np.maximum(a, b)).reshape(-1), return_counts=True)
    assert {1, 2, 3, 4} <= set(counts.tolist())
    nbr = to.adjacency(t)
    assert any(g >= 0 and (nbr[f] == g).all() for f, g in enumerate(nbr[:, 0]))     # the repeated face
    assert np.isnan(c["v"]).any() and to.validate(c["v"], t)
    assert len(np.unique(t)) < len(c["v"])
    r = _ref("topology", tc.topology)
    assert r["stats"][10] == 0 and r["stats"][7] > 1 and r["stats"][1] < len(t)


@pytest.mark.parametrize("jitter", [0.0, 0.3])
def test_occluder_has_no_hole_and_hides_the_back_faces(jitter):
    c = tc.occluder(jitter)
    buf = to.depth_buffer(*_cam(c, 0)[:3], *_cam(c, 0)[3:], c["v"], c["t"])
    inside = buf[20:101, 20:101]
    assert (inside != to.EMPTY).all()
    assert (_depth(inside) == 100.0).all()
    r = _texture(c)
    back = np.arange(len(c["t"]) - 64, len(c["t"]))
    assert all(all(a != 0 for _, a in r["cands"][f]) for f in back)
    if not jitter:
        # every sample of every back face falls on a pixel of an occluder edge or vertex
        u, v, _ = _samples(c, 0)
        px, py = np.floor(u[back] + 0.5), np.floor(v[back] + 0.5)
        x, y = (px - 20) % 10, (py - 20) % 10
        assert ((x == 0) | (y == 0) | (x == y)).all()


def _full_lists(c, monkeypatch):
    got = []
    with monkeypatch.context() as m:
        m.setattr(to, "best_candidates", lambda l: got.append(sorted(l, key=lambda e: (-e[0], e[1]))) or
                  sorted(l, key=lambda e: (-e[0], e[1]))[:to.MCAND])
        _texture(c)
    return got


def test_many_views_pass_more_than_8_with_a_tie_at_rank_8(monkeypatch):
    c = _case("many_views", tc.many_views)
    lists = _full_lists(c, monkeypatch)
    assert len(c["imgs"]) >= 12
    assert max(len(l) for l in lists) > 8
    assert any(len(l) > 8 and l[7][0] == l[8][0] for l in lists)
    n90, n75, n4 = (_ref(k, m)["stats"][2] for k, m in (("many_views_90", lambda: tc.many_views(90.0)),
                                                       ("many_views", tc.many_views),
                                                       ("many_views_4", lambda: tc.many_views(4.0))))
    assert n90 > n75 > n4 > 0


def test_coplanar_copies_tie_after_rounding():
    """At depthTol 0 the copies cover the same pixels with float64 depths that differ in their last bits and round to
    the same float: the tie order (the lower face) and the rounding before the comparison decide the owner, and a
    copy whose sample falls on a pixel its twin owns is visible only when its z <= that float depth."""
    c = tc.coplanar()
    assert c["kw"]["depthTol"] == 0.0
    split = behind = 0
    for a in range(len(c["imgs"])):
        K, R, t, W, H = _cam(c, a)
        buf = np.full(H * W, to.EMPTY, np.uint64)
        d64 = {}
        for f, pix, d in to.face_depths(K, R, t, W, H, c["v"], c["t"]):
            to.combine(buf, pix, d, f)
            for p, x in zip(pix.tolist(), d.tolist()):
                d64.setdefault(p, []).append((x, f))
        for p, got in d64.items():
            if len(got) == 2:
                (x, f), (y, g) = got
                owner = int(buf[p] & np.uint64(0xFFFFFFFF))
                split += x != y and np.float32(x) == np.float32(y) and owner == min(f, g) and \
                    (x < y) != (f < g)
        u, v, z = _samples(c, a)
        ok = (z > 0) & (u >= 0) & (u <= W - 1) & (v >= 0) & (v <= H - 1)
        px, py = np.where(ok, np.floor(u + 0.5), 0).astype(int), np.where(ok, np.floor(v + 0.5), 0).astype(int)
        key = buf[py * W + px]
        other = ok & (key != to.EMPTY) & ((key & np.uint64(0xFFFFFFFF)) != np.arange(len(c["t"]))[:, None])
        behind += int((other & (z > _depth(key))).sum())
    assert split > 0 and behind > 0, (split, behind)


def test_raster_edges_reach_their_faces():
    c = tc.raster_edges()
    K, R, t, W, H = _cam(c, 0)
    X = np.asarray(c["v"], np.float64)[np.asarray(c["t"], np.int64)]
    u, v, z = to.project(K, R, t, X)
    A = to.area2(u, v)
    assert ((A == 0) & (z > 0).all(1)).any()                 # the grid through camera 0's centre
    _, _, z1 = to.project(*_cam(c, 1)[:3], X)
    assert ((z1 > 0).any(1) & (z1 <= 0).any(1)).any()        # faces across camera 1's Y_z = 0
    big = (u.min(1) < 0) & (u.max(1) > W - 1) & (v.min(1) < 0) & (v.max(1) > H - 1)
    assert big.any()
    straddle = ((u.min(1) < 0) | (u.max(1) > W - 1) | (v.min(1) < 0) | (v.max(1) > H - 1)) & ~big & (z > 0).all(1)
    buf = to.depth_buffer(K, R, t, W, H, c["v"], c["t"])
    owners = set((buf[buf != to.EMPTY] & np.uint64(0xFFFFFFFF)).astype(np.int64).tolist())
    assert sum(f in owners for f in np.flatnonzero(straddle)) >= 6


@pytest.mark.parametrize("tol", [0.0, 0.01, 1.0])
def test_depth_ratio_crosses_the_tolerance(tol):
    c = tc.depth_ratio(tol)
    K, R, t, W, H = _cam(c, 0)
    buf = to.depth_buffer(K, R, t, W, H, c["v"], c["t"])
    u, v, z = _samples(c, 0)
    back = np.arange(32, len(c["t"]))
    px, py = np.floor(u[back] + 0.5).astype(int), np.floor(v[back] + 0.5).astype(int)
    key = buf[py, px]
    front = (key & np.uint64(0xFFFFFFFF)) < 32
    ratio = z[back][front] / _depth(key[front])
    assert (ratio < 1.0).any() and ((1.0 < ratio) & (ratio <= 1.01)).any() and (ratio > 1.01).any()


def test_mixed_sizes_groups():
    c = tc.mixed_sizes()
    shapes = [im.shape for im in c["imgs"]]
    assert min(w for _, w in shapes) == 2 and max(w for _, w in shapes) == 4095
    assert any(w % 4 for _, w in shapes)
    assert [tc.image_groups(shapes, cap) for cap in c["groups"]] == [4, 5, len(shapes)]
    assert 8 * 9 * 4095 > c["groups"][0]
    assert np.array_equal(c["Ks"][5], c["Ks"][6]) and np.array_equal(c["imgs"][5], c["imgs"][6])


def test_labelling_reaches_rule_4():
    c = _case("labelling", tc.labelling)
    assert len(c["t"]) == 20000
    col, _ = to.colouring(to.adjacency(c["t"]))
    assert col.max() == 3
    r = _ref("labelling", tc.labelling)
    assert r["stats"][10] == 0 and r["stats"][5] > 2 and r["stats"][6] > 0
    seen = r["labels"] >= 0
    nbr = r["nbr"]
    assert any(not seen[f] and (nbr[f] >= 0).all() and seen[nbr[f]].all() for f in range(len(seen)))


def test_charts_reach_rule_5():
    r = _ref("deep_strip", tc.deep_strip)
    assert r["stats"][7] == 1 and r["charts"][0, 7] == 6000
    r = _ref("single_charts", tc.single_charts)
    assert (r["charts"][:, 7] == 1).sum() >= 10 and r["stats"][6] == 0


def test_atlas_reaches_rule_6():
    r = _ref("atlas0", tc.atlas)
    ch = r["charts"]
    assert (ch[:, 3] == 100).any()                            # a chart as wide as the atlas
    for oy in np.unique(ch[:, 6]):
        on = ch[ch[:, 6] == oy]
        assert on[:, 3].sum() == 100                          # both shelves filled exactly
    assert (ch[:, 6] > 0).sum() == 2
    r = _ref("atlas16", lambda: tc.atlas(16))
    ch = r["charts"]
    assert (ch[:, 1] == 0).sum() >= 2 and (ch[:, 1] + ch[:, 3] == 100).sum() >= 2
    assert (ch[:, 2] == 0).any()
    r = _ref("unseen", tc.unseen)
    assert r["ret"] == 0 and r["stats"][1] == r["stats"][0] and r["stats"][8] == 0 and r["atlas"].shape[0] == 0


def test_scale_spreads_visible_faces_over_groups():
    c = tc.scale()
    T = len(c["t"])
    assert T > 1 << 21
    X = np.asarray(c["v"], np.float64)[np.asarray(c["t"], np.int64)]
    front = np.flatnonzero((X[:, :, 2] > 0).all(1))
    assert len(np.unique(front // (to.TILE * to.THREADS))) >= 4 and 1000 < len(front) < 5000


# ---- (b) sensitivity ------------------------------------------------------------------------------------------------
def _strict_cover(w0, w1, w2, S):
    return (w0 > 0) & (w1 > 0) & (w2 > 0) & (S > 0)


def _ties_to_higher(buf, pix, d, f):
    dn = d.astype(np.float32).view(np.uint32).astype(np.uint64)
    old = buf[pix]
    do, fo = old >> np.uint64(32), old & np.uint64(0xFFFFFFFF)
    win = (old == to.EMPTY) | (dn < do) | ((dn == do) & (np.uint64(f) > fo))
    buf[pix[win]] = (dn[win] << np.uint64(32)) | np.uint64(f)


_d64 = {}


def _unrounded(buf, pix, d, f):
    side = _d64.setdefault(id(buf), (buf, np.full(len(buf), np.inf)))[1]
    old = buf[pix]
    win = (old == to.EMPTY) | (d < side[pix]) | ((d == side[pix]) & (np.uint64(f) < (old & np.uint64(0xFFFFFFFF))))
    side[pix[win]] = d[win]
    buf[pix[win]] = (d[win].astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(f)


def _three_face_edges(ks):
    n = len(ks)
    return [i for i in range(n - 1) if not (i > 0 and ks[i - 1] == ks[i]) and ks[i + 1] == ks[i]
            and not (i + 3 < n and ks[i + 3] == ks[i] and ks[i + 2] == ks[i])]


def _roots_high(label, nbr):
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
                    parent[min(a, b)] = max(a, b)
    return np.array([find(f) for f in range(T)])


def _pack_ge(table, atlasWidth):
    C = len(table)
    order = sorted(range(C), key=lambda c: (-table[c, 4], -table[c, 3], c))
    shelfY = shelfH = cx = 0
    for c in order:
        if cx + table[c, 3] >= atlasWidth:
            shelfY += shelfH
            shelfH = cx = 0
        table[c, 5], table[c, 6] = cx, shelfY
        cx += table[c, 3]
        shelfH = max(shelfH, table[c, 4])
    return shelfY + shelfH


def _left_to_right(e):
    s = 0.0
    for x in np.asarray(e, np.float64):
        s += x
    return s


MUTATIONS = {
    "cover_strict": ("covers", _strict_cover, ["occluder", "occluder_jittered"]),
    "depth_ties_to_higher_face": ("combine", _ties_to_higher, ["coplanar"]),
    "depth_compared_unrounded": ("combine", _unrounded, ["coplanar"]),
    "candidate_tie_image_descending": ("best_candidates", lambda c: sorted(c, key=lambda e: (-e[0], -e[1]))[:8],
                                       ["many_views"]),
    "first_8_candidates": ("best_candidates", lambda c: sorted(c[:8], key=lambda e: (-e[0], e[1])),
                           ["many_views"]),
    "three_face_edges_adjacent": ("pair_starts", _three_face_edges, ["topology"]),
    "chart_roots_highest": ("chart_roots", _roots_high, ["topology", "single_charts"]),
    "padding_clamp_at_W": ("chart_rect", lambda e, W, H, p: (max(0, e[1] - p), max(0, e[2] - p), min(W, e[3] + p),
                                                              min(H - 1, e[4] + p)), ["atlas16"]),
    "shelf_ge": ("pack", _pack_ge, ["atlas0"]),
    "energy_left_to_right": ("tree_total", _left_to_right, ["topology", "labelling"]),
}
MAKERS = {"occluder": tc.occluder, "occluder_jittered": lambda: tc.occluder(0.3), "coplanar": tc.coplanar,
          "many_views": tc.many_views, "topology": tc.topology, "single_charts": tc.single_charts,
          "atlas0": tc.atlas, "atlas16": lambda: tc.atlas(16), "labelling": tc.labelling}


def _outputs(r):
    return [np.asarray(r[k]).tobytes() for k in ("ret", "stats", "info", "labels", "faceChart", "charts", "uv",
                                                 "atlas")]


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_every_mutation_is_seen(mutation, monkeypatch):
    name, fn, cases = MUTATIONS[mutation]
    changed = []
    for key in cases:
        ref = _outputs(_ref(key, MAKERS[key]))
        with monkeypatch.context() as m:
            m.setattr(to, name, fn)
            _d64.clear()
            try:
                out = _outputs(_texture(_case(key, MAKERS[key])))
            except (ValueError, IndexError):         # a rectangle past the image: the copy cannot be made
                out = None
        if out != ref:
            changed.append(key)
    print("%s: changes %s" % (mutation, changed))
    assert changed, mutation
