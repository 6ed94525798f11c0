"""GPU checks of cs_poisson_mesh_screened (PoissonMeshScreened) against tests/mesh_screened_oracle.py: the solve against
the oracle's system and MGPCG iteration count, the extraction replayed exactly from the GPU's chi and tau, the open
sheet, the closed sphere and torus, determinism, truncation, statuses, launches, the largest grid, and the dense chain
PatchMatch -> geometric pass -> fusion -> PoissonMeshScreened on the rendered scene, which the Dirichlet call cannot
mesh."""
import ctypes

import numpy as np
import pytest

import cudasift_b200 as cs
import mesh_cases as mc
import mesh_oracle as mo
import mesh_screened_cases as msc
import mesh_screened_oracle as so
import stereo_cases as sc
from test_mesh_screened_cpu import ALPHA, SHEET_MAX_BOUND, SHEET_MEAN_BOUND, SHEET_SEED

pytestmark = pytest.mark.gpu

RESIDUAL_ALLOWANCE = 2e-5  # float32 chi and A p against the float64 system
ITER_MARGIN = 1            # float32 vectors against the float64 oracle MGPCG
ULPS = 4                   # vertex positions: t from the same floats, float64 both sides, one rounding


def _ulp_close(a, b, ulps):
    return np.all(np.abs(a.astype(np.float64) - b) <= ulps * np.spacing(np.abs(b).astype(np.float32)))


@pytest.fixture(scope="module")
def runs():
    out = {}
    xs, ns = msc.sheet(40000, seed=SHEET_SEED)
    xp, npn = mc.sphere(20000)
    for name, (x, n) in (("sheet", (xs, ns)), ("sphere", (xp, npn))):
        for d in (5, 6):
            out[name, d] = (x, n), cs.PoissonMeshScreened(x, n, depth=d, pointWeight=ALPHA, returnChi=True)
    return out


@pytest.mark.parametrize("depth", [5, 6])
@pytest.mark.parametrize("case", ["sheet", "sphere"])
def test_solve_against_the_oracle_system(runs, case, depth):
    (x, n), (verts, tris, _, info, stats, chi, _) = runs[case, depth]
    assert stats[9] == 0, stats
    A, b, w, g, N, o, h, D, s = so.system(x, n, depth, 1.1, ALPHA)
    assert np.allclose(info[:3], o, rtol=0, atol=1e-12) and abs(info[3] - h) <= 1e-15
    assert abs(info[7] - w) <= 1e-6 * w
    bf = b.astype(np.float64).reshape(-1)
    res = np.linalg.norm(bf - A @ chi.astype(np.float64).reshape(-1)) / np.linalg.norm(bf)
    print("%s depth %d: residual %.3g (reported %.3g, recurrence below 1e-5), %d iterations"
          % (case, depth, res, info[6], stats[2]))
    assert res <= info[6] + RESIDUAL_ALLOWANCE
    assert res <= 1e-5 + RESIDUAL_ALLOWANCE
    k = so.mgpcg(A, b, s, 1e-5, 200)[1]
    assert abs(int(stats[2]) - k) <= ITER_MARGIN, (stats[2], k)


@pytest.mark.parametrize("case", ["sheet", "sphere"])
def test_extraction_replays_exactly(runs, case):
    (x, n), (verts, tris, _, info, stats, chi, _) = runs[case, 6]
    g, nh, _, N, o, h, ok, _ = mo.sorted_points(x, n, None, 6, 1.1)
    tau = float(mo.interpolate(chi, g, N).mean())
    assert abs(info[4] - tau) <= 1e-9 * np.abs(chi).max()
    assert abs(info[4]) <= 1e-4 * np.abs(chi).max()          # the mean of chi at the points is 0 up to rounding
    ref = so.mesh(x, n, depth=6, alpha=ALPHA)
    assert abs(info[4] - ref["tau"]) <= 1e-4 * np.abs(ref["chi"]).max()
    m = mo.extract(chi, info[4], info[:3], info[3])
    assert np.array_equal(tris, m["triangles"])
    assert _ulp_close(verts, m["vertices"].astype(np.float64), ULPS)
    assert stats[3] == m["pre"][0] and stats[4] == m["pre"][1]


def test_sheet(runs):
    (x, n), (verts, tris, _, info, stats, _, _) = runs["sheet", 5]
    assert stats[9] == 0 and mo.components(tris, len(verts)) == 1
    e = so.boundary_edge_vertices(tris)
    assert len(e) > 0 and so.on_faces(verts, info[:3], info[3], 32)[e].all()
    verts, tris, _, info, stats, _, _ = cs.PoissonMeshScreened(x, n, depth=5, pointWeight=ALPHA, trim=0.5)
    assert stats[9] == 0 and mo.components(tris, len(verts)) == 1
    d = msc.sheet_distance(verts) / info[3]
    print("sheet depth 5 trim 0.5: mean %.4f h, worst %.3f h" % (d.mean(), d.max()))
    assert d.mean() <= SHEET_MEAN_BOUND and d.max() <= SHEET_MAX_BOUND
    # the Dirichlet call on the same points: status 2
    assert cs.PoissonMesh(x, n, depth=5)[4][9] == 2


@pytest.mark.parametrize("case,euler", [("sphere", 2), ("torus", 0)])
def test_closed_shapes(case, euler):
    x, n = mc.sphere(20000) if case == "sphere" else mc.torus(20000)
    verts, tris, _, info, stats, _, _ = cs.PoissonMeshScreened(x, n, depth=6, pointWeight=ALPHA)
    assert stats[9] == 0
    assert mo.closed_and_oriented(tris) and mo.euler(tris) == euler
    v = verts.astype(np.float64)
    nrm = np.cross(v[tris[:, 1]] - v[tris[:, 0]], v[tris[:, 2]] - v[tris[:, 0]])
    c = v[tris].mean(1)
    if case == "sphere":
        out = c - mc.CENTRE
    else:
        p = c - mc.CENTRE
        ring = np.stack([p[:, 0], p[:, 1], np.zeros(len(p))], 1)
        out = p - ring / np.linalg.norm(ring, axis=1, keepdims=True)
    assert ((nrm * out).sum(1) > 0).mean() >= 0.99
    if case == "sphere":
        d = np.abs(np.linalg.norm(v - mc.CENTRE, axis=1) - 1.0) / info[3]
        vd, _, _, infod, _, _, _ = cs.PoissonMesh(x, n, depth=6)
        dd = np.abs(np.linalg.norm(vd.astype(np.float64) - mc.CENTRE, axis=1) - 1.0) / infod[3]
        print("sphere depth 6: screened mean %.4f h worst %.3f h, Dirichlet mean %.4f h worst %.3f h"
              % (d.mean(), d.max(), dd.mean(), dd.max()))
        assert d.mean() <= dd.mean() and d.max() <= dd.max() + 0.02


def test_determinism_intensities_and_truncation():
    x, n = msc.sheet(20000, seed=SHEET_SEED)
    inten = np.linspace(0, 1, len(x)).astype(np.float32)
    a = cs.PoissonMeshScreened(x, n, inten, depth=6, trim=0.5, returnChi=True)
    b = cs.PoissonMeshScreened(x, n, inten, depth=6, trim=0.5, returnChi=True)
    for u, v in zip(a[:6], b[:6]):
        assert np.array_equal(u, v)
    assert len(a[2]) == len(a[0]) and np.isfinite(a[2]).all()
    # truncated outputs: prefixes of the full lists, full counts reported
    verts, tris = a[0], a[1]
    P = len(x)
    bufs = [cs.DeviceBuffer(x.nbytes), cs.DeviceBuffer(n.nbytes), cs.DeviceBuffer(12 * 10), cs.DeviceBuffer(12 * 7)]
    try:
        bufs[0].upload(x)
        bufs[1].upload(n)
        info, stats = np.zeros(8), np.zeros(10, np.int64)
        T = cs.lib().cs_poisson_mesh_screened(bufs[0].ptr, bufs[1].ptr, None, P, 6, 1.1, ALPHA, 200, 1e-5, 0.5,
                                              bufs[2].ptr, None, 10, bufs[3].ptr, 7, None,
                                              info.ctypes.data_as(ctypes.c_void_p),
                                              stats.ctypes.data_as(ctypes.c_void_p), None)
        assert T == len(tris) and stats[7] == 10 and stats[8] == 7 and stats[5] == len(verts)
        assert np.array_equal(bufs[2].download(np.float32, 30).reshape(10, 3), verts[:10])
        assert np.array_equal(bufs[3].download(np.int32, 21).reshape(7, 3), tris[:7])
    finally:
        for q in bufs:
            q.free()


def test_statuses_and_launches():
    x, n = mc.sphere(5000)
    # status 1: no used point, or zero extent
    bad = np.full_like(x, np.nan)
    assert cs.PoissonMeshScreened(bad, n, depth=5)[4][9] == 1
    assert cs.PoissonMeshScreened(np.repeat(x[:1], 10, 0), n[:10], depth=5)[4][9] == 1
    # status 3: not converged in one iteration, still extracted
    verts, tris, _, info, stats, _, _ = cs.PoissonMeshScreened(x, n, depth=5, maxIterations=1)
    assert stats[9] == 3 and stats[2] == 1 and len(tris) > 0
    before = cs.lib().cs_launch_count()
    cs.PoissonMeshScreened(x, n, depth=5)
    assert cs.lib().cs_launch_count() - before == 10


def test_largest_grid():
    x, n = mc.sphere(3_000_000, seed=4)
    verts, tris, _, info, stats, _, ms = cs.PoissonMeshScreened(x, n, depth=9)
    print("depth 9, 3 M points: %d iterations, %d triangles, %.1f ms" % (stats[2], len(tris), ms))
    assert stats[9] == 0 and len(tris) > 0
    r = np.linalg.norm(verts.astype(np.float64) - mc.CENTRE, axis=1)
    assert np.abs(r - 1.0).max() <= 0.5 * info[3]


def test_chain_on_library_outputs():
    Ks, Rs, ts, views = sc.render(8, 640, 480, seed=2, texels=96)
    images = [v[0] for v in views]
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(8)]) if b != a][:4], 3.0, 12.0) for a in range(8)]
    d, nr, c, _, _ = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs)
    dg, ng, cg, _, _ = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, d, nr)
    xyz, nrm, inten, _, total, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, dg, ng, cg)
    rects = sc.scene()
    DEPTH, TRIM = 7, 0.5
    ref = so.mesh(xyz, nrm, inten, depth=DEPTH, alpha=ALPHA, trim=TRIM)
    verts, tris, vint, info, stats, _, _ = cs.PoissonMeshScreened(xyz, nrm, inten, depth=DEPTH, pointWeight=ALPHA,
                                                                  trim=TRIM)
    near = lambda v, h: float(np.mean(mc.rect_distance(v.astype(np.float64), rects) <= 3 * h))
    want, got = near(ref["vertices"], ref["h"]), near(verts, info[3])
    print("chain: %d fused points, status %d, %d iterations (oracle %d to 1e-10), %d triangles, within 3 h of the "
          "scene %.3f (oracle %.3f)" % (total, stats[9], stats[2], ref["iters"], len(tris), got, want))
    assert stats[9] == 0 and len(tris) > 0
    assert got >= want - 0.02
