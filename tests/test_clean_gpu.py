"""GPU checks of cs_clean_mesh (CleanMesh) against tests/clean_oracle.py: integer-equal triangle lists, bit-equal
vertices and intensities and equal info and stats on every hand-made case, with smoothing, with every stage off and on
PoissonMeshScreened's sheet meshes; repeat calls, truncation, statuses, launches, the depth-9 sphere with holes and
islands, and the chain PatchMatch -> geometric pass -> fusion -> PoissonMeshScreened -> CleanMesh -> SimplifyMesh ->
TextureMesh."""
import numpy as np
import pytest

import clean_cases as cc
import clean_oracle as co
import cudasift_b200 as cs
import mesh_cases as mc
import mesh_screened_cases as msc
import stereo_cases as sc

pytestmark = pytest.mark.gpu


def _equal(v, t, i, **kw):
    gv, gt, gi, info, stats, ms = cs.CleanMesh(v, t, i, **kw)
    ref = co.clean(v, t, i, **kw)
    assert list(stats) == ref["stats"]
    assert np.array_equal(gt, ref["triangles"])
    assert np.array_equal(gv.view(np.uint32), ref["vertices"].view(np.uint32))
    if i is not None:
        assert np.array_equal(gi.view(np.uint32), ref["intensity"].view(np.uint32))
    assert list(info) == list(ref["info"])
    return gv, gt, stats


@pytest.mark.parametrize("case", sorted(cc.CASES))
def test_oracle_equality(case):
    v, t, i = cc.CASES[case]()
    _, _, stats = _equal(v, t, i, **cc.SETTINGS.get(case, {}))
    print(case, list(stats))


@pytest.mark.parametrize("case", ["holes", "sphere_mess"])
def test_oracle_equality_smoothing(case):
    v, t, i = cc.CASES[case]()
    _equal(v, t, i, smoothIterations=5, **cc.SETTINGS.get(case, {}))


@pytest.mark.parametrize("case", sorted(cc.CASES))
def test_all_stages_off(case):
    v, t, i = cc.CASES[case]()
    _equal(v, t, i, **co.OFF)


@pytest.fixture(scope="module")
def sheets():
    x, n = msc.sheet(20000, seed=0)[:2]
    return {trim: cs.PoissonMeshScreened(x, n, depth=5, trim=trim)[:2] for trim in (0.5, 1.0)}


@pytest.mark.parametrize("trim", [0.5, 1.0])
def test_sheet_meshes(sheets, trim):
    v, t = sheets[trim]
    _, gt, stats = _equal(v, t, None)
    _equal(v, t, None, longEdgeFactor=3.0, minComponentFraction=0.1, maxHoleEdges=256, smoothIterations=2)
    assert co.components(gt).min() >= 50


def test_repeat_calls_same_bytes():
    v, t, i = cc.sphere_mess()
    a = cs.CleanMesh(v, t, i, longEdgeFactor=3.0, smoothIterations=3)
    b = cs.CleanMesh(v, t, i, longEdgeFactor=3.0, smoothIterations=3)
    for x, y in zip(a[:5], b[:5]):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_truncated_outputs_are_prefixes():
    v, t, i = cc.holes()
    full = co.clean(v, t, i, maxHoleEdges=40)
    V, T = len(v), len(t)
    buf = [cs.DeviceBuffer(12 * V), cs.DeviceBuffer(12 * T), cs.DeviceBuffer(4 * V)]
    ins = [cs.DeviceBuffer(12 * V), cs.DeviceBuffer(12 * T), cs.DeviceBuffer(4 * V)]
    try:
        for b, a in zip(ins, (v, t, i)):
            b.upload(np.ascontiguousarray(a))
        stats = np.zeros(19, np.int64)
        n = cs.lib().cs_clean_mesh(ins[0].ptr, ins[2].ptr, V, ins[1].ptr, T, 1, 20.0, 1, 50, 0.0, 40, 0, 0.5, -0.53,
                                   buf[0].ptr, buf[2].ptr, 100, buf[1].ptr, 1000, None, stats.ctypes.data, None)
        assert n == len(full["triangles"]) and stats[16] == 100 and stats[17] == 1000
        assert np.array_equal(buf[0].download(np.float32, 300).reshape(-1, 3), full["vertices"][:100])
        assert np.array_equal(buf[2].download(np.float32, 100), full["intensity"][:100])
        assert np.array_equal(buf[1].download(np.int32, 3000).reshape(-1, 3), full["triangles"][:1000])
    finally:
        for b in buf + ins:
            b.free()


def test_statuses():
    v, t, i = cc.holes()
    assert cs.CleanMesh(v, t)[4][18] == 0
    bad = t.copy()
    bad[5, 1] = len(v)
    out = cs.CleanMesh(v, bad)
    assert out[4][18] == 2 and len(out[1]) == 0 and len(out[0]) == 0
    nan = v.copy()
    nan[t[0, 0], 2] = np.nan
    assert cs.CleanMesh(nan, t)[4][18] == 2


def _radix_bits(n):
    b = 1
    while b < 31 and (1 << b) <= n:
        b += 1
    return b


@pytest.mark.parametrize("kw", [{}, dict(co.OFF), dict(longEdgeFactor=3.0, smoothIterations=4, minComponentFaces=0),
                                dict(removeDegenerate=False, removeNonManifold=False, maxHoleEdges=0)])
def test_launch_count(kw):
    v, t, i = cc.sphere_mess()
    p = dict(co.DEFAULTS, **kw)
    n = 1 + 1 + 1 + 3 + 2 + 4
    n += 3 if p["removeDegenerate"] else 0
    n += 4 if p["longEdgeFactor"] > 0 else 0
    n += 2 if p["removeNonManifold"] else 0
    n += 1 if p["minComponentFaces"] > 1 or p["minComponentFraction"] > 0 else 0
    n += 7 + _radix_bits(3 * len(t)) if p["maxHoleEdges"] else 0
    n += 2 + 2 * p["smoothIterations"] if p["smoothIterations"] else 0
    before = cs.lib().cs_launch_count()
    cs.CleanMesh(v, t, i, **kw)
    assert cs.lib().cs_launch_count() - before == n
    before = cs.lib().cs_launch_count()
    bad = t.copy()
    bad[0, 0] = -1
    cs.CleanMesh(v, bad, i, **kw)
    assert cs.lib().cs_launch_count() - before == 1


def test_depth9_sphere_with_holes_closes():
    x, n = mc.sphere(3_000_000, seed=4)
    v, t, _, _, _, _, _ = cs.PoissonMesh(x, n, depth=9)
    pv, pt = cc.punch(v, t, seed=1, rings=200, faces=200, islands=5)
    b0 = co.topology(pt)[0]
    gv, gt, _, _, stats, ms = cs.CleanMesh(pv, pt)
    b, nm, euler, oriented = co.topology(gt)
    print("depth 9 sphere: %d triangles with %d boundary edges -> %d triangles, %d zero-area faces dropped, "
          "%d loops filled (%d open), %d components dropped, %.1f ms" % (
              len(pt), b0, len(gt), stats[1], stats[10], stats[11], stats[7], ms))
    assert (b, nm, euler, oriented) == (0, 0, 2, True)
    assert stats[11] == 0 and stats[7] == 5 and len(gv) <= len(v)


def test_chain_on_library_outputs():
    Ks, Rs, ts, views = sc.render(8, 640, 480, seed=2, texels=96)
    images = [w[0] for w in views]
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(8)]) if b != a][:4], 3.0, 12.0) for a in range(8)]
    d, nr, c, _, _ = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs)
    dg, ng, cg, _, _ = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, d, nr)
    xyz, nrm, inten, _, _, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, dg, ng, cg)
    verts, tris, vint, _, _, _, _ = cs.PoissonMeshScreened(xyz, nrm, inten, depth=7, trim=1.0)
    cv, ct, ci, info, stats, ms = cs.CleanMesh(verts, tris, vint)
    sizes0, sizes = co.components(tris), co.components(ct)
    b0, b1 = co.topology(tris)[0], co.topology(ct)[0]
    print("chain: %d triangles, %d components (%d under 50), %d boundary edges -> %d triangles, %d components, "
          "%d boundary edges; loops %d filled %d open %d, %.1f ms" % (
              len(tris), len(sizes0), (sizes0 < 50).sum(), b0, len(ct), len(sizes), b1, stats[9], stats[10],
              stats[11], ms))
    assert stats[18] == 0 and sizes.min() >= 50
    ref = co.clean(verts, tris, vint)
    assert np.array_equal(ct, ref["triangles"]) and list(stats) == ref["stats"]
    # the loops left open are the output's boundary loops (filled loops share no vertex with them); each one of at
    # most maxHoleEdges (30) edges is one the ear rule refuses
    T64 = ct.astype(np.int64)
    loops, _ = co.boundary_loops(T64, np.ones(len(ct), bool))
    P = [tuple(float(c) for c in row) for row in cv.astype(np.float64)]
    edges = frozenset(co._edge_keys(T64, np.arange(len(ct)))[0].tolist())
    short = [lp for lp in loops if len(lp) <= 30]
    assert len(loops) == stats[11]
    assert all(co.ear_cut(P, [h[0] for h in lp], edges) is None for lp in short)
    print("chain: %d loops left open, %d of them with at most 30 edges (refused by the ear rule)" % (
        len(loops), len(short)))
    sv, st, si, _, sstats, _ = cs.SimplifyMesh(cv, ct, ci, targetTriangles=len(ct) // 4)
    uv0 = cs.TextureMesh(images, Ks, Rs, ts, *cs.SimplifyMesh(verts, tris, vint, targetTriangles=len(tris) // 4)[:2])
    uv1 = cs.TextureMesh(images, Ks, Rs, ts, sv, st)
    print("texture after SimplifyMesh to 1/4: uncleaned %d faces, %d unseen, %d charts; cleaned %d faces, %d unseen, "
          "%d charts" % (uv0[-2][0], uv0[-2][1], len(uv0[3]), uv1[-2][0], uv1[-2][1], len(uv1[3])))
    assert sstats[8] == 0 and uv1[-2][0] == len(st)
    # observed: the cleaned mesh leaves fewer faces unseen and makes fewer charts
    assert uv1[-2][1] <= uv0[-2][1] and len(uv1[3]) < len(uv0[3])
