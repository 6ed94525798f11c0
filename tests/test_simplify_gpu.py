"""GPU checks of cs_simplify_mesh (SimplifyMesh) against tests/simplify_oracle.py: integer-equal triangle lists,
bit-equal vertices and intensities and equal pass and collapse counts on the meshes PoissonMesh and PoissonMeshScreened
make (with and without jitter), topology and accuracy on larger meshes, determinism, truncation, statuses, launches,
the largest sphere, and the chain PatchMatch -> geometric pass -> fusion -> PoissonMeshScreened -> SimplifyMesh."""
import ctypes

import numpy as np
import pytest

import cudasift_b200 as cs
import mesh_cases as mc
import mesh_oracle as mo
import mesh_screened_cases as msc
import simplify_oracle as so
import stereo_cases as sc

pytestmark = pytest.mark.gpu

RADIUS_BOUND = 0.5         # |r - 1| / h of every simplified vertex of the depth-8 sphere at 10 %
CHAIN_SHARE_MARGIN = 0.02  # share of simplified vertices within 3 h of the scene against the input mesh's share


def _jitter(v, h, seed=3):
    rng = np.random.default_rng(seed)
    return (v.astype(np.float64) + rng.uniform(-0.05 * h, 0.05 * h, v.shape)).astype(np.float32)


@pytest.fixture(scope="module")
def meshes():
    out = {}
    x, n = mc.sphere(20000)
    inten = np.linspace(0, 1, len(x)).astype(np.float32)
    v, t, vi, info, _, _, _ = cs.PoissonMesh(x, n, inten, depth=5)
    out["sphere"] = (v, t, vi, info[3])
    x, n = mc.torus(20000)
    v, t, _, info, _, _, _ = cs.PoissonMesh(x, n, depth=5)
    out["torus"] = (v, t, None, info[3])
    x, n = msc.sheet(40000, seed=1)
    v, t, _, info, _, _, _ = cs.PoissonMeshScreened(x, n, depth=5, trim=0.5)
    out["sheet"] = (v, t, None, info[3])
    return out


@pytest.mark.parametrize("jitter", [False, True])
@pytest.mark.parametrize("case", ["sphere", "torus", "sheet"])
def test_oracle_equality(meshes, case, jitter):
    v, t, vi, h = meshes[case]
    if jitter:
        v = _jitter(v, h)
    target = len(t) // 10
    gv, gt, gi, info, stats, _ = cs.SimplifyMesh(v, t, vi, targetTriangles=target)
    ref = so.simplify(v, t, vi, target=target)
    print("%s%s: %d -> %d triangles, %d passes, %d collapses, %d frozen" % (
        case, " jittered" if jitter else "", len(t), len(gt), stats[2], stats[3], stats[1]))
    assert list(stats) == ref["stats"]
    assert np.array_equal(gt, ref["triangles"])
    assert np.array_equal(gv, ref["vertices"])
    assert info[0] == ref["info"]
    if vi is not None:
        assert np.array_equal(gi, ref["intensity"])
    assert stats[8] == 0 and target - 1 <= len(gt) <= target


def test_larger_mesh():
    x, n = mc.sphere(200000, seed=2)
    v, t, _, info, _, _, _ = cs.PoissonMesh(x, n, depth=8)
    target = len(t) // 10
    gv, gt, _, ginfo, stats, ms = cs.SimplifyMesh(v, t, targetTriangles=target)
    r = np.abs(np.linalg.norm(gv.astype(np.float64) - mc.CENTRE, axis=1) - 1.0) / info[3]
    print("depth 8 sphere: %d -> %d triangles, %d passes, %.1f ms, |r - 1| mean %.3f h worst %.3f h"
          % (len(t), len(gt), stats[2], ms, r.mean(), r.max()))
    assert stats[8] == 0 and target - 1 <= len(gt) <= target
    assert mo.closed_and_oriented(gt) and mo.euler(gt) == 2
    assert r.max() <= RADIUS_BOUND
    x, n = mc.torus(200000, seed=2)
    v, t, _, info, _, _, _ = cs.PoissonMesh(x, n, depth=8)
    gv, gt, _, _, stats, _ = cs.SimplifyMesh(v, t, targetTriangles=len(t) // 10)
    assert stats[8] == 0 and mo.closed_and_oriented(gt) and mo.euler(gt) == 0


def test_determinism_truncation_statuses_and_launches(meshes):
    v, t, vi, _ = meshes["sphere"]
    a = cs.SimplifyMesh(v, t, vi, targetTriangles=len(t) // 4)
    b = cs.SimplifyMesh(v, t, vi, targetTriangles=len(t) // 4)
    for x, y in zip(a[:5], b[:5]):
        assert np.array_equal(x, y)
    # truncated outputs: prefixes of the full lists, full counts reported
    bufs = [cs.DeviceBuffer(v.nbytes), cs.DeviceBuffer(t.nbytes), cs.DeviceBuffer(12 * 10), cs.DeviceBuffer(12 * 7)]
    try:
        bufs[0].upload(v)
        bufs[1].upload(np.ascontiguousarray(t, np.int32))
        stats = np.zeros(9, np.int64)
        T = cs.lib().cs_simplify_mesh(bufs[0].ptr, None, len(v), bufs[1].ptr, len(t), len(t) // 4, float("inf"), 1.0,
                                      bufs[2].ptr, None, 10, bufs[3].ptr, 7, None,
                                      stats.ctypes.data_as(ctypes.c_void_p), None)
        assert T == len(a[1]) and stats[6] == 10 and stats[7] == 7 and stats[4] == len(a[0])
        assert np.array_equal(bufs[2].download(np.float32, 30).reshape(10, 3), a[0][:10])
        assert np.array_equal(bufs[3].download(np.int32, 21).reshape(7, 3), a[1][:7])
    finally:
        for q in bufs:
            q.free()
    # status 0 with no pass, 1 (maxError), 2 (invalid input), 3 is the pass cap (not reachable on a small mesh)
    r = cs.SimplifyMesh(v, t, targetTriangles=len(t))
    assert r[4][8] == 0 and r[4][2] == 0 and len(r[1]) == len(t)
    before = cs.lib().cs_launch_count()
    r = cs.SimplifyMesh(v, t, maxError=1e-3)
    assert r[4][8] == 1 and r[3][0] <= 1e-3
    assert cs.lib().cs_launch_count() - before == 4 + 8 * r[4][2] + 4 + 4
    bad = t.copy()
    bad[5, 1] = bad[5, 0]
    before = cs.lib().cs_launch_count()
    r = cs.SimplifyMesh(v, bad)
    assert r[4][8] == 2 and len(r[1]) == 0 and cs.lib().cs_launch_count() - before == 1
    nan = v.copy()
    nan[t[0, 0], 1] = np.nan
    assert cs.SimplifyMesh(nan, t)[4][8] == 2


def test_largest_case():
    x, n = mc.sphere(3_000_000, seed=4)
    v, t, _, info, _, _, _ = cs.PoissonMesh(x, n, depth=9)
    target = len(t) // 10
    gv, gt, _, ginfo, stats, ms = cs.SimplifyMesh(v, t, targetTriangles=target)
    r = np.abs(np.linalg.norm(gv.astype(np.float64) - mc.CENTRE, axis=1) - 1.0) / info[3]
    print("depth 9 sphere: %d -> %d triangles, %d passes, %d collapses, %.1f ms, worst %.3f h"
          % (len(t), len(gt), stats[2], stats[3], ms, r.max()))
    assert stats[8] == 0 and target - 1 <= len(gt) <= target
    assert r.max() <= RADIUS_BOUND


def test_chain_on_library_outputs():
    Ks, Rs, ts, views = sc.render(8, 640, 480, seed=2, texels=96)
    images = [v[0] for v in views]
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(8)]) if b != a][:4], 3.0, 12.0) for a in range(8)]
    d, nr, c, _, _ = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs)
    dg, ng, cg, _, _ = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, d, nr)
    xyz, nrm, inten, _, total, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, dg, ng, cg)
    rects = sc.scene()
    verts, tris, vint, info, stats, _, _ = cs.PoissonMeshScreened(xyz, nrm, inten, depth=7, trim=0.5)
    gv, gt, gi, ginfo, gstats, ms = cs.SimplifyMesh(verts, tris, vint, targetTriangles=len(tris) // 10)
    near = lambda v: float(np.mean(mc.rect_distance(v.astype(np.float64), rects) <= 3 * info[3]))
    before, after = near(verts), near(gv)
    print("chain: %d triangles -> %d (status %d, %d passes, %d frozen, %.1f ms), within 3 h of the scene %.3f "
          "(input mesh %.3f)" % (len(tris), len(gt), gstats[8], gstats[2], gstats[1], ms, after, before))
    assert gstats[8] == 0 and len(gi) == len(gv) and np.isfinite(gi).all()
    assert after >= before - CHAIN_SHARE_MARGIN
