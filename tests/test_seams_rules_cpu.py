"""The seam levelling cases of tests/seam_cases.py reach the rules they are built for, shown on the oracle without a
GPU:
(a) each case's precondition (touching and gapped charts and corner 0 on exclusive edges, every input failure, S at
an exact integer and in the thousands, samples on texel centres and clamped taps, 3- and 4-face edges, a (v, a, b) row
whose ends' order changes its float sum, an unknown with more incidences than one coop.cuh piece, row counts either
side of 256 and 2048, b = 0, A = 0 and A < 0, key ties between faces); (b) each one-line mutation of a rule in the
oracle changes, on at least one case, an output test_seams_rules_gpu.py compares bit for bit (the stats, the seam
energy's bits, the atlas given fixed corner offsets), so a kernel with the same slip would fail that comparison; the
order of the offset sum in the texel stage is the exception, seen by the oracle only; (c) the overlapping chart table
on which the oracle's first-chart rule and the device's row-index search part; (d) the vectorised oracle giving the
scalar one's bytes on every small case, and the scale case past 2048 x 256 unknowns and seam rows."""
import math

import numpy as np
import pytest

import seam_cases as sc
import seam_oracle as so
import texture_oracle as to

_memo = {}


def case(name):
    if name not in _memo:
        _memo[name] = sc.CASES[name]()
    return _memo[name]


def build(name):
    c = case(name)
    return so.build(c["v"], c["t"], c["labels"], c["uv"], c["charts"], c["atlas"], c["kw"].get("smoothness", 0.1))


def level(c):
    return so.level(c["v"], c["t"], c["labels"], c["uv"], c["charts"], c["atlas"], **c["kw"])


# ---- (a) preconditions ----------------------------------------------------------------------------------------------
def test_lookup_reaches_rule_1():
    c = case("lookup")
    ch = c["charts"]
    shelf0 = ch[ch[:, 6] == 0]
    assert len(shelf0) == 24 and (shelf0[1:, 5] == shelf0[:-1, 5] + shelf0[:-1, 3]).all()      # touching
    b = build("lookup")
    seen = c["labels"] >= 0
    x, y = np.floor(c["uv"][seen, 0, 0]), np.floor(c["uv"][seen, 0, 1])
    e = ch[b["faceChart"][seen]]
    assert ((c["uv"][seen, 0, 0] == e[:, 5]) & (x > 0)).sum() >= 20          # on the left chart's exclusive right edge
    assert ((c["uv"][seen, 0, 1] == 6.0)).sum() >= 10                        # on shelf 0's exclusive bottom edge
    assert ((x == e[:, 5] + e[:, 3] - 1)).sum() >= 20                        # in a chart's last column
    assert len(b["seam"]) > 0 and level(c)["stats"][7] == 0
    assert not seen.all() and np.isnan(c["uv"][~seen]).all()


@pytest.mark.parametrize("variant", [v for v in sc.INVALID if v != "overlap"])
def test_every_input_failure_gives_status_2(variant):
    c = case("invalid_" + variant)
    assert build("invalid_" + variant) is None
    assert level(c)["stats"] == [0] * 7 + [2]


def _record(monkeypatch, name, log):
    fn = getattr(so, name)
    monkeypatch.setattr(so, name, lambda *a: log.append((a, fn(*a))) or fn(*a))


def test_samples_reach_rule_3(monkeypatch):
    counts, reads, ends = [], [], []
    _record(monkeypatch, "sample_count", counts)
    _record(monkeypatch, "bilinear", reads)
    _record(monkeypatch, "end_order", ends)
    b = build("samples")
    c = case("samples")
    S = {(La, Lb): s for (La, Lb), s in counts}
    assert S[(0.0, 0.0)] == 1 and any(s > 1 and 0.0 in L for L, s in S.items())
    assert any(max(L) == 5.0 and s == 5 for L, s in S.items())               # ceil of an exact integer
    assert any(5.0 < max(L) < 5.001 and s == 6 for L, s in S.items())
    assert max(S.values()) == 2501
    on = [(x, y) for (_, e, x, y), _ in reads if x == math.floor(x) and y == math.floor(y)]
    assert len(on) >= 12                                                     # fx = fy = 0
    box = lambda e: (e[5], e[5] + e[3] - 1, e[6], e[6] + e[4] - 1)
    out = [(x, y) for (_, e, x, y), _ in reads
           if not (box(e)[0] <= x < box(e)[1] and box(e)[2] <= y < box(e)[3])]
    assert len(out) >= 10                                                    # taps clamped to the chart
    assert any(x < 0 for x, y in out)                                        # a side that leaves the atlas
    # edges held by 3 and 4 faces, and a two-face edge with one side unseen
    t = np.asarray(c["t"], np.int64)
    k = ((np.minimum(t, np.roll(t, -1, 1)) << 32) | np.maximum(t, np.roll(t, -1, 1))).reshape(-1)
    _, n = np.unique(k, return_counts=True)
    assert {3, 4} <= set(n.tolist())
    nbr = to.adjacency(t)
    lab = c["labels"]
    assert any(g >= 0 and (lab[f] < 0) != (lab[g] < 0) for f in range(len(t)) for g in nbr[f])
    # a row of at least 3 ends whose sum in another order gives other bits
    def total(parts):
        s = [0.0, 0.0, 0.0]
        for p in parts:
            s = [s[i] + p[i] for i in range(3)]
        return s
    assert any(len(p) >= 3 and total(p) != total(p[::-1]) for (p,), _ in ends)
    # a vertex on 8 labels, labels up to 2^31 - 2
    per_vertex = np.bincount([v for v, _ in b["keys"]])
    assert per_vertex.max() == 8 and max(l for _, l in b["keys"]) == 2 ** 31 - 2


def test_rows_and_solve_reach_rules_4_to_6():
    b = build("valence")
    inc = np.bincount(np.array([[i, j] for i, j, _, _ in b["seam"]] + list(b["smooth"])).reshape(-1))
    assert inc.max() > 11 * 256
    for name, (rows, unknowns) in sc.COUNTS.items():
        b = build("counts_" + name)
        assert len(b["seam"]) == rows and (unknowns is None or len(b["keys"]) == unknowns), name
    b = build("constant")
    _, rhs = so.system(b, 1e-3)
    assert len(b["seam"]) > 0 and not rhs.any()
    assert level(case("constant"))["stats"][5:] == [0, level(case("constant"))["stats"][6], 0]
    b = build("solve_tol_0")
    assert so.pcg(b, 1e-3, 0.0, 40)[1:] == (40, False)
    assert level(case("solve_max_iterations_0"))["stats"][5::2] == [0, 3]


def test_texels_reach_rule_7(monkeypatch):
    c = case("texels_pad2")
    U = c["uv"].astype(np.float64)
    A = to.area2(U[:, :, 0], U[:, :, 1])
    assert (A < 0).any() and (A == 0).sum() >= 2
    assert ((U[:, 0] == U[:, 1]).all(1) & (U[:, 1] == U[:, 2]).all(1)).any()
    wins = []
    monkeypatch.setattr(so, "key_wins", lambda k, old: wins.append((int(k), int(old))) or k < old)
    level(c)
    m = (1 << 32) - 1
    assert any(k >> 32 == o >> 32 and (k & m) != (o & m) and o != int(to.EMPTY) for k, o in wins)     # key ties
    assert any(k >> 32 == 0 and o >> 32 == 0 and (k & m) != (o & m) for k, o in wins)   # a centre on two faces
    outside = np.ones(c["atlas"].shape, bool)
    for e in c["charts"]:
        outside[e[6]:e[6] + e[4], e[5]:e[5] + e[3]] = False
    a = c["atlas"][outside]
    assert np.isnan(a).any() and (np.signbit(a) & (a == 0)).any()


# ---- (b) sensitivity ------------------------------------------------------------------------------------------------
def _three_face_edges(ks):
    n = len(ks)
    return [i for i in range(n - 1) if not (i > 0 and ks[i - 1] == ks[i]) and ks[i + 1] == ks[i]
            and not (i + 3 < n and ks[i + 3] == ks[i] and ks[i + 2] == ks[i])]


def _ties_to_higher(k, old):
    m = np.uint64(0xFFFFFFFF)
    return old == to.EMPTY or (k >> np.uint64(32)) < (old >> np.uint64(32)) or \
        ((k >> np.uint64(32)) == (old >> np.uint64(32)) and (k & m) > (old & m))


def _key_of_d2(d2, f):
    return (np.uint64(np.float32(d2).view(np.uint32)) << np.uint64(32)) | np.uint64(f)


def _smooth_per_edge(cu, seen):
    return sorted((min(cu[f, k], cu[f, (k + 1) % 3]), max(cu[f, k], cu[f, (k + 1) % 3]))
                  for f in np.nonzero(seen)[0] for k in range(3))


SMALL = ["lookup", "samples", "ends", "texels_pad0", "texels_pad2", "solve_smoothness_0"]
MUTATIONS = {
    "chart_right_edge_inclusive": ("holds", lambda e, x, y: e[5] <= x <= e[5] + e[3] and e[6] <= y < e[6] + e[4]),
    "taps_clamped_to_the_atlas": ("tap_box", lambda a, e: (0, a.shape[1] - 1, 0, a.shape[0] - 1)),
    "t_k_is_k_over_S": ("sample_t", lambda k, S: k / S),
    "S_without_max_1": ("sample_count", lambda La, Lb: int(math.ceil(max(La, Lb)))),
    "ends_in_reverse_key_order": ("end_order", lambda parts: parts[::-1]),
    "sides_by_face_id": ("sides", lambda f, g, lab: (min(f, g), max(f, g))),
    "three_face_edges_are_seams": ("pair_starts", _three_face_edges),
    "smoothness_rows_per_face_edge": ("smooth_rows", _smooth_per_edge),
    "texel_ties_to_the_higher_face": ("key_wins", _ties_to_higher),
    "segment_ties_to_the_higher_k": ("nearer", lambda d2, best: d2 <= best),
    "box_grown_by_padding": ("box_grow", lambda padding: float(padding)),
    "key_from_d2": ("texel_key", _key_of_d2),
}


def _ref(key):
    if ("ref", key) not in _memo:
        _memo[("ref", key)] = level(case(key))
    return _memo[("ref", key)]


def _gpu_channels(c, r, corner):
    """What test_seams_rules_gpu.py compares bit for bit: the stats but the CG count (compared within 1), the seam
    energy before levelling, and the atlas of the texel stage given fixed corner offsets (the unmutated oracle's)."""
    st = list(r["stats"])
    if "build" not in r:
        return [st]
    atlas, _ = so.texels(c["t"], c["labels"], c["uv"], c["charts"], r["build"]["faceChart"], c["atlas"], corner,
                         c["kw"].get("padding", 2), copy_all=not r["build"]["seam"])
    return [st[:5] + st[6:], np.float64(r["info"][0]).tobytes(), atlas.tobytes()]


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_every_mutation_is_seen(mutation, monkeypatch):
    """Each mutation changes, on some case, an output the GPU test compares bit for bit.  The mutated oracle must run
    to the end: a mutation is seen through its outputs, never through an exception."""
    name, fn = MUTATIONS[mutation]
    changed = []
    for key in SMALL:
        c, ref = case(key), _ref(key)
        want = _gpu_channels(c, ref, ref.get("corner"))
        with monkeypatch.context() as m:
            m.setattr(to if name == "pair_starts" else so, name, fn)
            got = _gpu_channels(c, level(c), ref.get("corner"))
        if got != want:
            changed.append(key)
    print("%s: changes %s" % (mutation, changed))
    assert changed, mutation


def test_offset_sum_order_is_seen_by_the_oracle_only(monkeypatch):
    """The offset sum (b_0 o_0 + b_1 o_1) + b_2 o_2 against b_0 o_0 + (b_1 o_1 + b_2 o_2): the two round alike on
    the corner offsets a solve gives, so the GPU comparison cannot tell them apart; the oracle's texel stage does, given
    the corner offsets (2^40, -2^40, 0.3) and (0.3, 2^40, -2^40) on every face, which cancel exactly in one order where
    the two big offsets' weights are equal (the bisector of a right-angled uv triangle)."""
    def stage(c, b):
        return [so.texels(c["t"], c["labels"], c["uv"], c["charts"], b["faceChart"], c["atlas"],
                          np.tile(np.float32(o), (len(c["t"]), 1)), c["kw"].get("padding", 2))[0].tobytes()
                for o in ((2.0 ** 40, -2.0 ** 40, 0.3), (0.3, 2.0 ** 40, -2.0 ** 40))]
    changed = []
    for key in ("texels_pad0", "texels_pad2"):
        c, b = case(key), build(key)
        want = stage(c, b)
        with monkeypatch.context() as m:
            m.setattr(so, "corner_sum", lambda bw, o: bw[0] * float(o[0]) + (bw[1] * float(o[1]) + bw[2] * float(o[2])))
            if stage(c, b) != want:
                changed.append(key)
    assert changed


# ---- (d) the vectorised oracle --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(sc.CASES))
def test_vectorised_oracle_gives_the_same_bytes(name):
    """build_np and texels_np against build and texels on every small case: the same dict and, given random corner
    offsets of 10^-3..10^3, the same atlas bytes and visited count."""
    c = case(name)
    args = (c["v"], c["t"], c["labels"], c["uv"], c["charts"], c["atlas"], c["kw"].get("smoothness", 0.1))
    a, b = so.build(*args), so.build_np(*args)
    assert (a is None) == (b is None)
    if a is None:
        return
    for k in a:
        x, y = a[k], b[k]
        if k == "seam":
            x, y = np.array(x, np.float64).tobytes(), np.array(y, np.float64).tobytes()
        assert np.array_equal(np.asarray(x), np.asarray(y)), k
    rng = np.random.default_rng(5)
    corner = (rng.choice([-1.0, 1.0], (len(c["t"]), 3)) * 10.0 ** rng.uniform(-3, 3, (len(c["t"]), 3)))
    corner = corner.astype(np.float32)
    for copy_all in (False, True):
        want = so.texels(c["t"], c["labels"], c["uv"], c["charts"], a["faceChart"], c["atlas"], corner,
                         c["kw"].get("padding", 2), copy_all)
        got = so.texels_np(c["t"], c["labels"], c["uv"], c["charts"], a["faceChart"], c["atlas"], corner,
                           c["kw"].get("padding", 2), copy_all, chunk=1000)
        assert got[1] == want[1] and got[0].tobytes() == want[0].tobytes()


def test_scale_passes_two_levels_of_totals():
    """The scale case's unknowns and seam rows both exceed 2048 x 256, so level 3 of every total runs."""
    c = sc.scale()
    b = so.build_np(c["v"], c["t"], c["labels"], c["uv"], c["charts"], c["atlas"])
    assert len(b["keys"]) > 2048 * 256 and len(b["seam"]) > 2048 * 256


# ---- (c) the chart table ------------------------------------------------------------------------------------------
def _device_chart(uv, label, charts, rows):
    """seams_check_kernel's search restated: the row index of the table (per row, charts by (ox, index)) and the last
    entry with ox <= x, which must hold x and have the label."""
    x, y = math.floor(float(uv[0, 0])), math.floor(float(uv[0, 1]))
    row = sorted((e[5], c) for c, e in enumerate(charts) if e[6] <= y < e[6] + e[4])
    at = [c for ox, c in row if ox <= x]
    if not at:
        return -1
    e = charts[at[-1]]
    return at[-1] if x < e[5] + e[3] and e[0] == label else -1


def test_overlapping_charts_part_the_rules():
    """Without the overlap check the oracle levels this table and the device's search fails a face (status 2)."""
    c = case("invalid_overlap")
    b = build("invalid_overlap")
    assert b is not None
    rows = c["atlas"].shape[0]
    dev = [_device_chart(c["uv"][f], c["labels"][f], c["charts"], rows) for f in np.flatnonzero(c["labels"] >= 0)]
    assert -1 in dev
    # on every valid case the two agree
    for name in ("lookup", "samples", "texels_pad2"):
        cc, bb = case(name), build(name)
        for f in np.flatnonzero(cc["labels"] >= 0):
            assert _device_chart(cc["uv"][f], cc["labels"][f], cc["charts"], rows) == bb["faceChart"][f]
