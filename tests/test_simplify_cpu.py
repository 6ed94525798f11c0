"""CPU checks of the simplifier's rules (tests/simplify_oracle.py) and of cs_simplify_mesh's argument checks: the
oracle's outputs stay oriented 2-manifolds with their Euler characteristic and boundary loops, frozen vertices and the
refused collapses hold on hand-made meshes, the quality stays near a sequential greedy decimator's, maxError bounds
every applied error, and the sweeps that chose f and the default boundaryWeight."""
import ctypes
import math
import os

import numpy as np
import pytest

import cudasift_b200 as cs
import mesh_oracle as mo
import mesh_screened_cases as msc
import simplify_cases as scs
import simplify_oracle as so
from test_arg_ranges_cpu import BASE, MSG, _buf, _layout, _share

CS_E_ARG = -2
QUALITY_MEAN_FACTOR = 1.5      # mean analytic distance against the greedy decimator's at the same target
QUALITY_WORST_FACTOR = 2.0     # worst analytic distance against the greedy decimator's


@pytest.fixture(scope="module")
def sphere():
    v, t, c, R = scs.sphere_mesh(16, 5.3)
    return v, t, lambda p: np.abs(np.linalg.norm(np.asarray(p, np.float64) - c, axis=1) - R)


@pytest.fixture(scope="module")
def torus():
    v, t, c, (R, r) = scs.torus_mesh(16, 4.6, 1.9)
    return v, t, lambda p: scs.torus_distance(p, c, R, r)


@pytest.fixture(scope="module")
def sheet():
    v, t, h = scs.sheet_mesh(depth=4)
    return v, t, lambda p: msc.sheet_distance(p) / h


def _areas(v, t):
    v = np.asarray(v, np.float64)
    return np.linalg.norm(np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]]), axis=1)


def _check_output(v, t, r, target):
    out = r["triangles"]
    assert r["stats"][8] == 0 and target - 1 <= len(out) <= target, r["stats"]
    assert so.manifold_apart_from(out, [])
    ia, oa = _areas(v, np.asarray(t)), _areas(r["vertices"], out)
    assert (oa[ia[r["tid"]] > 0] > 0).all()


@pytest.mark.parametrize("jitter", [0.0, 0.1])
def test_closed_meshes_keep_their_topology(jitter):
    for make, chi in ((lambda: scs.sphere_mesh(16, 5.3, jitter=jitter), 2),
                      (lambda: scs.torus_mesh(16, 4.6, 1.9, jitter=jitter), 0)):
        v, t = make()[:2]
        assert mo.closed_and_oriented(t) and mo.euler(t) == chi
        target = len(t) // 10
        r = so.simplify(v, t, target=target)
        _check_output(v, t, r, target)
        assert mo.closed_and_oriented(r["triangles"]) and mo.euler(r["triangles"]) == chi


def test_sheet_keeps_its_boundary_loops(sheet):
    v, t, _ = sheet
    loops = so.boundary_loops(t)
    target = len(t) // 10
    r = so.simplify(v, t, target=target)
    _check_output(v, t, r, target)
    assert so.boundary_loops(r["triangles"]) == loops
    assert mo.euler(r["triangles"]) == mo.euler(t)


def test_grid_keeps_its_boundary_and_plane():
    v, t = scs.grid(8, jitter=0.2)
    r = so.simplify(v, t, target=20)
    _check_output(v, t, r, 20)
    assert so.boundary_loops(r["triangles"]) == 1
    assert (r["vertices"][:, 2] == 0).all()


def test_bowtie_vertex_is_frozen_and_never_moves():
    v, t = scs.bowtie()
    r = so.simplify(v, t)
    assert r["stats"][1] == 1 and r["frozen"][0] and not r["frozen"][1:].any()
    assert np.array_equal(r["vertices"][0], v[0])


def test_tetrahedron_is_refused():
    v, t = scs.tetrahedron()
    r = so.simplify(v, t)
    assert r["stats"][8] == 1 and r["stats"][3] == 0 and len(r["triangles"]) == 4


def test_three_face_edge_freezes_its_ends():
    v, t, (a, b) = scs.three_faces()
    r = so.simplify(v, t, target=4)
    assert r["frozen"][a] and r["frozen"][b]
    for x in (a, b):
        assert any(np.array_equal(p, v[x]) for p in r["vertices"]), x


def test_flipped_face_freezes_its_corners():
    v, t, f = scs.flipped()
    r = so.simplify(v, t, target=4)
    assert all(r["frozen"][x] for x in f)
    for x in f:
        assert any(np.array_equal(p, v[x]) for p in r["vertices"]), x


def test_invalid_inputs():
    v, t = scs.grid(2)
    for bad in (lambda t: t.__setitem__((0, 0), -1), lambda t: t.__setitem__((0, 0), len(v)),
                lambda t: t.__setitem__((0, 1), t[0, 0])):
        tt = t.copy()
        bad(tt)
        assert so.simplify(v, tt)["stats"][8] == 2
    vv = v.copy()
    vv[t[0, 0], 2] = np.inf
    assert so.simplify(vv, t)["stats"][8] == 2


def test_quality_against_greedy(sphere, torus, sheet):
    for name, (v, t, dist) in (("sphere", sphere), ("torus", torus), ("sheet", sheet)):
        target = len(t) // 10
        r = so.simplify(v, t, target=target)
        gv, gt = so.greedy(v, t, target=target)
        d, g = dist(r["vertices"]), dist(gv)
        print("%s at 10%%: parallel mean %.4f worst %.4f, greedy mean %.4f worst %.4f, %d passes"
              % (name, d.mean(), d.max(), g.mean(), g.max(), r["stats"][2]))
        assert d.mean() <= QUALITY_MEAN_FACTOR * g.mean() and d.max() <= QUALITY_WORST_FACTOR * g.max()
        # to the input mesh: every output vertex near an input vertex
        from scipy.spatial import cKDTree
        near = cKDTree(np.asarray(v, np.float64)).query(r["vertices"])[0]
        gnear = cKDTree(np.asarray(v, np.float64)).query(gv)[0]
        assert near.mean() <= QUALITY_MEAN_FACTOR * gnear.mean() + 1e-9


def test_max_error_bounds_every_collapse(sphere):
    v, t, _ = sphere
    for bound in (0.01, 0.05):
        r = so.simplify(v, t, maxError=bound)
        assert r["stats"][8] == 1 and 0 < r["info"] <= bound and r["stats"][3] > 0
        assert mo.closed_and_oriented(r["triangles"]) and mo.euler(r["triangles"]) == 2


def test_f_sweep(sphere, torus, sheet):
    """Passes and the mean-distance ratio to the greedy decimator for f in {1/8, 1/4, 1/2, 1} at 10 % (f = 1/2 is the
    library's)."""
    for name, (v, t, dist) in (("sphere", sphere), ("torus", torus), ("sheet", sheet)):
        target = len(t) // 10
        g = dist(so.greedy(v, t, target=target)[0]).mean()
        row = []
        for shift in (3, 2, 1, 0):
            r = so.simplify(v, t, target=target, f_shift=shift)
            row.append("f=1/%d: %d passes, ratio %.3f" % (1 << shift, r["stats"][2], dist(r["vertices"]).mean() / g))
            assert r["stats"][8] == 0
        print("%s (%d triangles): %s" % (name, len(t), "; ".join(row)))


def test_boundary_weight_sweep(sheet):
    """The distance of the output boundary from the input boundary on the trimmed sheet at 10 % (1 is the default)."""
    v, t, _ = sheet
    from scipy.spatial import cKDTree

    def boundary_vertices(tris):
        d = mo.directed_edges(tris)
        s = set(map(tuple, d))
        return np.unique([a for a, b in d if (b, a) not in s])

    tin = np.asarray(t, np.int64)
    ref = cKDTree(np.asarray(v, np.float64)[boundary_vertices(tin)])
    out = []
    for bw in (0.0, 0.25, 1.0, 4.0, 16.0):
        r = so.simplify(v, t, target=len(t) // 10, boundaryWeight=bw)
        d = ref.query(r["vertices"][boundary_vertices(r["triangles"])].astype(np.float64))[0]
        out.append((bw, d.mean(), d.max()))
    print("boundaryWeight: " + "; ".join("%g: mean %.4f worst %.4f" % o for o in out))
    assert out[2][1] <= out[0][1]


def test_tie_order_is_a_bijection():
    """s(id) = m ^ (m >> 16), m = id 0x9E3779B1 mod 2^32: the xorshift is its own inverse and the odd multiplier has an
    inverse mod 2^32, so s is a bijection of the 32-bit ids and keys stay unique; checked through the inverse on ids
    across the whole range and exhaustively as distinct values over the first 3 * 2^20 ids."""
    inv = pow(0x9E3779B1, -1, 1 << 32)
    undo = lambda y: ((y ^ (y >> 16)) * inv) & 0xFFFFFFFF
    rng = np.random.default_rng(3)
    ids = [0, 1, 2, 3, (1 << 31) - 1, 1 << 31, (1 << 32) - 1] + [int(i) for i in rng.integers(0, 1 << 32, 20000)]
    for i in ids:
        s = so.tie_of(i)
        assert 0 <= s < (1 << 32) and undo(s) == i
    n = 3 << 20
    m = (np.arange(n, dtype=np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)
    s = m ^ (m >> np.uint64(16))
    assert len(np.unique(s)) == n and [so.tie_of(int(i)) for i in (5, 77, n - 1)] == [int(s[5]), int(s[77]), int(s[-1])]
    # equal errors: keys differ, and their order is not the ids' order
    keys = [so.key_of(0.0, i) for i in range(3000)]
    assert len(set(keys)) == 3000 and keys != sorted(keys)
    assert so.key_of(1.0, 0) > so.key_of(0.5, 2999) and so.key_of(math.inf, 0) > so.key_of(1e38, 2999)


def test_flat_grid_selects_many_edges_per_pass():
    """Every error of a flat grid is 0, so the tie order alone decides the selection: more than one edge per pass."""
    v, t = scs.grid(16)
    r = so.simplify(v, t, target=len(t) // 10, max_passes=1)
    assert r["stats"][2] == 1 and r["stats"][3] >= 10


# ---- library --------------------------------------------------------------------------------------------------------

def _call(verts=0x1000, vint=None, V=4, tris=0x2000, T=4, target=0, maxError=math.inf, bw=1.0, ov=0x10000, oi=None,
          maxV=4, ot=0x20000, maxT=4):
    return cs.lib().cs_simplify_mesh(verts, vint, V, tris, T, target, maxError, bw, ov, oi, maxV, ot, maxT, None, None,
                                     None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    assert msg.startswith("cs_simplify_mesh: invalid argument (CS_E_ARG)"), msg
    for w in words:
        assert w in msg, (w, msg)


def test_argument_checks():
    _rejects(_call(V=-1), "numVertices")
    _rejects(_call(V=(1 << 30) + 1), "numVertices")
    _rejects(_call(T=-1), "numTriangles")
    _rejects(_call(T=(1 << 29) + 1), "numTriangles")
    _rejects(_call(target=-1), "targetTriangles")
    _rejects(_call(maxError=-1.0), "maxError")
    _rejects(_call(maxError=float("nan")), "maxError")
    _rejects(_call(bw=-0.5), "boundaryWeight")
    _rejects(_call(bw=float("inf")), "boundaryWeight")
    _rejects(_call(maxV=-1), "maxOutVertices")
    _rejects(_call(maxT=-1), "maxOutTriangles")
    _rejects(_call(verts=None), "d_vertices")
    _rejects(_call(verts=0x1002), "d_vertices")
    _rejects(_call(tris=None), "d_triangles")
    _rejects(_call(tris=0x2001), "d_triangles")
    _rejects(_call(ov=None), "d_outVertices")
    _rejects(_call(ot=0x20002), "d_outTriangles")
    _rejects(_call(vint=0x3001, oi=0x4000), "d_vertexIntensity")
    _rejects(_call(vint=0x3000, oi=0x4002), "d_outIntensity")
    _rejects(_call(vint=0x3000), "d_vertexIntensity and d_outIntensity")
    _rejects(_call(oi=0x4000), "d_vertexIntensity and d_outIntensity")


def test_empty_mesh_makes_no_cuda_call():
    stats = np.full(9, -1, np.int64)
    r = cs.lib().cs_simplify_mesh(None, None, 0, None, 0, 0, math.inf, 1.0, None, None, 0, None, 0, None,
                                  stats.ctypes.data_as(ctypes.c_void_p), None)
    assert r == 0 and (stats == 0).all()


def _simplify_layout(rng):
    V, T, W, U = (int(rng.integers(1, 50)) for _ in range(4))
    with_i = bool(rng.integers(0, 2))
    sizes = {"d_vertices": 12 * V, "d_triangles": 12 * T, "d_outVertices": 12 * W, "d_outTriangles": 12 * U}
    if with_i:
        sizes.update({"d_vertexIntensity": 4 * V, "d_outIntensity": 4 * W})
    outs = {"d_outVertices", "d_outIntensity", "d_outTriangles"}

    def make(at):
        g = lambda x: at.get(x)
        return cs.lib().cs_simplify_mesh(g("d_vertices"), g("d_vertexIntensity"), V, g("d_triangles"), T, 0, math.inf,
                                         1.0, g("d_outVertices"), g("d_outIntensity"), W, g("d_outTriangles"), U,
                                         None, None, None)

    return sizes, (lambda a, b: a in outs or b in outs), make


def test_every_overlap_is_rejected_and_named():
    rng = np.random.default_rng(11)
    for _ in range(300):
        sizes, forbidden, make = _simplify_layout(rng)
        at = _layout(rng, sizes, forbidden)
        r = make({x: BASE + v for x, v in at.items()})
        msg = cs.lib().cs_last_error().decode()
        assert r == CS_E_ARG, (r, msg)
        m = MSG.match(msg)
        assert m, msg
        _, a, b = m.groups()
        assert a in sizes and b in sizes, (msg, sorted(sizes))
        assert forbidden(a, b) and _share((at[a], sizes[a]), (at[b], sizes[b])), (msg, at, sizes)
    assert not _buf.any()


def test_header_declares_the_call():
    hdr = open(os.path.join(os.path.dirname(cs.__file__), "..", "include", "cudasift_b200.h")).read()
    assert "int cs_simplify_mesh(" in hdr and "8 per pass" in hdr
    assert isinstance(cs.lib().cs_simplify_mesh, ctypes._CFuncPtr)
