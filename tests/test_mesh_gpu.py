"""GPU checks of cs_poisson_mesh (PoissonMesh) against tests/mesh_oracle.py: the solve against the oracle's system and
MGPCG iteration count, the extraction replayed exactly from the GPU's chi and tau, topology and geometry on a sphere,
torus and hollow shell, trimming on a hemisphere, intensities, determinism, truncation, statuses, the largest grid,
launches, and the dense chain PatchMatch -> geometric pass -> fusion -> PoissonMesh on the rendered scene."""
import ctypes

import numpy as np
import pytest

import cudasift_b200 as cs
import mesh_cases as mc
import mesh_oracle as mo
import stereo_cases as sc

pytestmark = pytest.mark.gpu

B_ALLOWANCE = 2e-6        # relative difference of the GPU's float b and the oracle's (each rounds V and b to float)
ITER_MARGIN = 1           # float32 vectors against the float64 oracle MGPCG
ULPS = 4                  # vertex positions: t from the same floats, float64 both sides, one rounding
MARGINAL_SHARE = 0.01     # trimmed triangles whose density is within 1e-6 relative of the threshold


def _ulp_close(a, b, ulps):
    return np.all(np.abs(a.astype(np.float64) - b) <= ulps * np.spacing(np.abs(b).astype(np.float32)))


@pytest.fixture(scope="module")
def sphere_runs():
    x, n = mc.sphere(20000)
    return {d: cs.PoissonMesh(x, n, depth=d, returnChi=True) for d in (5, 6)}, (x, n)


@pytest.mark.parametrize("depth", [5, 6])
def test_solve_against_the_oracle_system(sphere_runs, depth):
    runs, (x, n) = sphere_runs
    verts, tris, _, info, stats, chi, _ = runs[depth]
    assert stats[9] == 0, stats
    g, nh, _, N, o, h, ok, _ = mo.sorted_points(x, n, None, depth, 1.1)
    assert np.allclose(info[:3], o, rtol=0, atol=1e-12) and abs(info[3] - h) <= 1e-15
    V, D, _ = mo.splat(g, nh, None, N)
    b = mo.rhs(V, h)
    A = mo.operator(N)
    bi = mo.interior(b).astype(np.float64)
    res = np.linalg.norm(bi - A @ mo.interior(chi).astype(np.float64)) / np.linalg.norm(bi)
    assert info[6] <= 1e-5
    assert res <= info[6] + B_ALLOWANCE, (res, info[6])
    _, k, _ = mo.mgpcg(b.astype(np.float64), 1e-5, 200)
    assert abs(int(stats[2]) - k) <= ITER_MARGIN, (stats[2], k)
    print("depth %d: %d CG iterations (oracle %d), residual %.2e" % (depth, stats[2], k, info[6]))


@pytest.mark.parametrize("depth", [5, 6])
def test_extraction_replayed_exactly(sphere_runs, depth):
    runs, _ = sphere_runs
    verts, tris, _, info, stats, chi, _ = runs[depth]
    m = mo.extract(chi, info[4], info[:3], info[3])
    assert m["pre"] == (stats[3], stats[4]) and len(verts) == stats[5] and len(tris) == stats[6]
    assert np.array_equal(tris, m["triangles"])
    assert _ulp_close(verts, m["vertices"].astype(np.float64), ULPS)
    # tau is the mean of chi at the points
    x, n = sphere_runs[1]
    g, *_ = mo.sorted_points(x, n, None, depth, 1.1)
    assert abs(mo.interpolate(chi, g, 1 << depth).mean() - info[4]) <= 1e-9 * abs(info[4])


def _geometry(P, nrm, depth, surface, trim=0.0):
    """GPU mesh and the oracle's bound (its worst vertex distance x 1.5 + h / 4) at the same settings."""
    ref = mo.mesh(P, nrm, depth=depth, trim=trim)
    bound = 1.5 * surface(ref["vertices"].astype(np.float64)).max() + ref["h"] / 4
    out = cs.PoissonMesh(P, nrm, depth=depth, trim=trim)
    return out, bound


def _outward(verts, tris, grad):
    v = verts.astype(np.float64)
    nrm = np.cross(v[tris[:, 1]] - v[tris[:, 0]], v[tris[:, 2]] - v[tris[:, 0]])
    c = v[tris].mean(1)
    return float(((nrm * grad(c)).sum(1) > 0).mean())


def test_sphere_and_torus_topology_and_geometry():
    x, n = mc.sphere(60000, seed=3)
    sph = lambda v: np.abs(np.linalg.norm(v - mc.CENTRE, axis=1) - 1.0)
    (verts, tris, _, info, stats, _, _), bound = _geometry(x, n, 7, sph)
    assert stats[9] == 0
    assert mo.closed_and_oriented(tris) and mo.euler(tris) == 2 and mo.components(tris, len(verts)) == 1
    assert sph(verts.astype(np.float64)).max() <= bound
    assert _outward(verts, tris, lambda c: c - mc.CENTRE) >= 0.99

    x, n = mc.torus(80000, seed=4)

    def tor(v):
        d = v - mc.CENTRE
        return np.abs(np.sqrt((np.hypot(d[:, 0], d[:, 1]) - 1.0) ** 2 + d[:, 2] ** 2) - 0.4)

    def tgrad(c):
        d = c - mc.CENTRE
        rho = np.hypot(d[:, 0], d[:, 1])
        ring = np.stack([d[:, 0] / rho, d[:, 1] / rho, np.zeros_like(rho)], 1)
        return d - ring

    (verts, tris, _, info, stats, _, _), bound = _geometry(x, n, 7, tor)
    assert stats[9] == 0
    assert mo.closed_and_oriented(tris) and mo.euler(tris) == 0 and mo.components(tris, len(verts)) == 1
    assert tor(verts.astype(np.float64)).max() <= bound
    assert _outward(verts, tris, tgrad) >= 0.99


def test_nested_shell_gives_two_components():
    x, n = mc.shell(60000)
    verts, tris, _, info, stats, _, _ = cs.PoissonMesh(x, n, depth=7)
    assert stats[9] == 0
    assert mo.closed_and_oriented(tris) and mo.components(tris, len(verts)) == 2


def test_trimming_opens_the_hemisphere():
    x, n = mc.hemisphere(30000)
    verts, tris, _, info, stats, _, _ = cs.PoissonMesh(x, n, depth=6)
    assert mo.closed_and_oriented(tris)
    TRIM = 0.1
    tv, tt, _, tinfo, tstats, chi, _ = cs.PoissonMesh(x, n, depth=6, trim=TRIM, returnChi=True)
    assert tstats[3] == stats[3] and tstats[4] == stats[4]          # the same mesh before trimming
    assert len(tt) < len(tris) and mo.boundary_edges(tt) > 0
    h = tinfo[3]
    r = np.linalg.norm(tv - mc.CENTRE, axis=1)
    assert np.abs(r - 1.0).max() <= 1.5 * h and (tv[:, 2] >= mc.CENTRE[2] - 3 * h).all()
    # trimming against the oracle from the GPU's chi, tau and mean density
    g, nh, _, N, o, hh, _, _ = mo.sorted_points(x, n, None, 6, 1.1)
    _, D, _ = mo.splat(g, nh, None, N)
    m = mo.extract(chi, tinfo[4], tinfo[:3], h, D, None, TRIM, tinfo[5])
    if not np.array_equal(tt, m["triangles"]):
        full = mo.extract(chi, tinfo[4], tinfo[:3], h, D, None, 0.0, tinfo[5])
        dens = full["density"][full["triangles"]]
        marginal = (np.abs(dens - TRIM * tinfo[5]) <= 1e-6 * TRIM * tinfo[5]).any(1)
        assert marginal.mean() <= MARGINAL_SHARE
        assert abs(len(tt) - len(m["triangles"])) <= marginal.sum()


def test_intensity_and_null_intensity_geometry():
    x, n = mc.sphere(40000, seed=5)
    a, c0 = np.array([0.5, -0.25, 0.75]), 2.0
    I = (x.astype(np.float64) @ a + c0).astype(np.float32)
    v1, t1, vi, info, _, _, _ = cs.PoissonMesh(x, n, I, depth=6)
    v0, t0, none, _, _, _, _ = cs.PoissonMesh(x, n, None, depth=6)
    assert none is None
    assert np.array_equal(v0, v1) and np.array_equal(t0, t1)
    want = v1.astype(np.float64) @ a + c0
    assert np.abs(vi - want).max() <= 1.5 * info[3] * np.linalg.norm(a)


def _raw(x, n, depth, maxV, maxT):
    P = len(x)
    bufs = [cs.DeviceBuffer(max(x.nbytes, 4)), cs.DeviceBuffer(max(n.nbytes, 4)), cs.DeviceBuffer(12 * maxV + 4),
            cs.DeviceBuffer(12 * maxT + 4)]
    try:
        if P:
            bufs[0].upload(np.ascontiguousarray(x, np.float32))
            bufs[1].upload(np.ascontiguousarray(n, np.float32))
        info, stats = np.zeros(7), np.zeros(10, np.int64)
        l0 = cs.lib().cs_launch_count()
        T = cs.lib().cs_poisson_mesh(bufs[0].ptr, bufs[1].ptr, None, P, depth, 1.1, 200, 1e-5, 0.0, bufs[2].ptr, None,
                                     maxV, bufs[3].ptr, maxT, None, info.ctypes.data, stats.ctypes.data, None)
        launches = cs.lib().cs_launch_count() - l0
        assert T >= 0, cs.lib().cs_last_error()
        v = bufs[2].download(np.float32, 3 * maxV).reshape(-1, 3)
        t = bufs[3].download(np.int32, 3 * maxT).reshape(-1, 3)
    finally:
        for b in bufs:
            b.free()
    return T, v, t, info, stats, launches


def test_determinism_truncation_statuses_and_launches():
    x, n = mc.sphere(20000, seed=6)
    a = cs.PoissonMesh(x, n, depth=6, returnChi=True)
    b = cs.PoissonMesh(x, n, depth=6, returnChi=True)
    for u, w in zip(a[:6], b[:6]):
        assert (u is None and w is None) or u.tobytes() == w.tobytes()
    V, T = len(a[0]), len(a[1])
    T2, v, t, info, stats, launches = _raw(x, n, 6, V // 3, T // 2)
    assert launches == 10
    assert T2 == T and stats[7] == V // 3 and stats[8] == T // 2 and stats[5] == V and stats[6] == T
    assert np.array_equal(v, a[0][:V // 3]) and np.array_equal(t, a[1][:T // 2])
    assert (t >= V // 3).any()                                    # a written triangle may name an unwritten vertex
    # status 1: no points, all points refused, all points at one place
    for xs, ns in ((x[:0], n[:0]), (x[:10], np.zeros((10, 3), np.float32)), (np.repeat(x[:1], 5, 0), n[:5])):
        T3, _, _, _, st, launches = _raw(xs, ns, 4, 4, 4)
        assert T3 == 0 and st[9] == 1 and launches == 10, st
    # status 2: inward normals
    T4, _, _, info4, st4, _ = _raw(x, -n, 5, 4, 4)
    assert T4 == 0 and st4[9] == 2 and info4[4] <= 0
    # status 3: one iteration cannot reach the tolerance; the mesh is still extracted
    out = cs.PoissonMesh(x, n, depth=6, maxIterations=1, tol=1e-9)
    assert out[4][9] == 3 and out[4][2] == 1 and len(out[1]) > 0


def test_depth_9_with_millions_of_points():
    x, n = mc.sphere(3_000_000, seed=8)
    verts, tris, _, info, stats, _, ms = cs.PoissonMesh(x, n, depth=9)
    print("depth 9, 3M points: %d vertices, %d triangles, %d iterations, residual %.2e, %.1f ms"
          % (len(verts), len(tris), stats[2], info[6], ms))
    assert stats[9] == 0 and stats[0] == 3_000_000
    assert mo.closed_and_oriented(tris) and mo.euler(tris) == 2
    assert np.abs(np.linalg.norm(verts - mc.CENTRE, axis=1) - 1.0).max() <= 2 * info[3]


def test_chain_on_library_outputs():
    Ks, Rs, ts, views = sc.render(8, 640, 480, seed=2, texels=96)
    images = [v[0] for v in views]
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(8)]) if b != a][:4], 3.0, 12.0) for a in range(8)]
    d, nr, c, _, _ = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs)
    dg, ng, cg, _, _ = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, d, nr)
    xyz, nrm, inten, _, total, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, dg, ng, cg)
    rects = sc.scene()
    DEPTH, TRIM = 7, 0.5
    ref = mo.mesh(xyz, nrm, inten, depth=DEPTH, trim=TRIM)
    verts, tris, vint, info, stats, _, _ = cs.PoissonMesh(xyz, nrm, inten, depth=DEPTH, trim=TRIM)
    print("chain: %d fused points, tau %.4g (oracle %.4g), status %d, %d triangles"
          % (total, info[4], ref["tau"], stats[9], len(tris)))
    assert stats[0] == len(xyz) and total == len(xyz)
    # the iso-value's sign decides the status, so it must agree with the float64 solve
    assert abs(info[4] - ref["tau"]) <= 1e-3 * np.abs(ref["chi"]).max()
    if ref["tau"] <= 0:
        # an open scene seen from one side: chi at the points is below the boundary's 0 (status 2, no mesh)
        assert stats[9] == 2 and len(tris) == 0
        return
    near = lambda v, h: float(np.mean(mc.rect_distance(v.astype(np.float64), rects) <= 3 * h))
    want, got = near(ref["vertices"], ref["h"]), near(verts, info[3])
    print("within 3 h of the scene %.3f (oracle %.3f)" % (got, want))
    assert stats[9] == 0 and len(tris) > 0
    assert got >= want - 0.02
