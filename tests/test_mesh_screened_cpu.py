"""CPU checks of screened Poisson meshing with a Neumann boundary (cs_poisson_mesh_screened) on its float64 restatement
(tests/mesh_screened_oracle.py): the Dirichlet call's kernels are unchanged instruction for instruction, the
right-hand side sums to 0 and is the Dirichlet one inside, the coarse screening is exact, the V-cycle is a symmetric
positive-definite preconditioner, MGPCG converges in few iterations, an open sheet the Dirichlet call cannot mesh gets
one accurate component, closed shapes stay closed, and every documented CS_E_ARG is returned naming its argument."""
import ctypes
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import mesh_cases as mc
import mesh_oracle as mo
import mesh_screened_cases as msc
import mesh_screened_oracle as so
from cudasift_b200 import build
from test_arg_ranges_cpu import BASE, MSG, _buf, _layout, _share
from test_bundle_intrinsics_cpu import _sass

CS_E_ARG = -2
ALPHA = 4.0
MAX_ITERATIONS = 20            # MGPCG to 1e-5, depths 5 and 6, alpha 1, 4, 16 (10 to 17 observed)
CONTRACTION_BOUND = 0.6        # spectral radius of I - B A for the V-cycle B on the sheet at N = 8 (0.500 observed)
SHEET_MEAN_BOUND = 0.05        # mean vertex distance / h to the sheet at depth 5, trim 0.5
SHEET_MAX_BOUND = 0.5          # worst vertex distance / h
SHEET_SEED = 1                 # a sample of the sheet on which the Dirichlet call gives status 2

# sha256 of the normalised `cuobjdump -sass` of mesh.o's kernels before the screened call was added, from nvcc 12.9
# (V12.9.86) with the library's flags.
SASS = {"mesh_box_kernel": "84538b006ef3e84bd73f400e08634aa1ecaba7a6b93bbe9b3349d56bb691af2a",
        "mesh_keys_kernel": "02697cd888d913f7a5656134db6ec67968ce9fca546d9af62e37f5fb09244f49",
        "mesh_points_kernel": "bc8c955ffe431927aa84c91b12536f5b93b5a9dc1040ae296c7f4172f9d72c92",
        "mesh_splat_kernel": "68b00060a8db226301d5afd3ea3dfd0551f2c7a8b92af48120cf7afb83ffc362",
        "mesh_rhs_kernel": "f89da014c6a7b99a85b029d6601df72f1bd8ce2e0d5ee93c48ba34ef5583f664",
        "mesh_solve_kernel": "a36e5c108e7e35d74773413282e8e54c28e1143af7515986e4a9e00d02952742",
        "mesh_count_kernel": "3df31bc79c6effa52308a8ac9e4fa9ef1dab13c29bb9af8531b99b53814e6f94",
        "mesh_kept_kernel": "52825fcad2bf0c60b366cde6b2d2b3b895f318e66a17785a85ea5f143dbf6345",
        "mesh_vertices_kernel": "23adbba18fb1e25f39a163a7516dc556f8ceea8c7d1428c4d81ee1f9dd3a7c5a",
        "mesh_triangles_kernel": "76c56667a21cf59078815d9211e504b4cccd471f8cbfd518d0b9a5bc3e5a7c89"}


def test_dirichlet_kernels_are_unchanged():
    nvcc = build.nvcc_path()
    if nvcc is None or "V12.9.86" not in subprocess.run([nvcc, "--version"], stdout=subprocess.PIPE,
                                                        text=True).stdout:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    build.build_library()
    fs = _sass(os.path.join(build.OBJDIR, "mesh.o"))
    for name, digest in SASS.items():
        key = [f for f in fs if re.search(r"\d+%sE" % name, f)]
        assert len(key) == 1, (name, sorted(fs))
        assert hashlib.sha256("\n".join(fs[key[0]]).encode()).hexdigest() == digest, name
    assert any(re.search(r"\d+mesh_screened_solve_kernelE", f) for f in fs)


# ---- the system -----------------------------------------------------------------------------------------------------

def _points(case, depth):
    x, n = msc.sheet(40000) if case == "sheet" else mc.sphere(20000)
    g, nh, _, N, o, h, ok, _ = mo.sorted_points(x, n, None, depth, 1.1)
    V, D, _ = mo.splat(g, nh, None, N)
    return x, n, g, N, h, V, D


@pytest.mark.parametrize("case", ["sheet", "sphere"])
def test_rhs_sums_to_zero_and_is_the_dirichlet_one_inside(case):
    _, _, _, N, h, V, _ = _points(case, 5)
    b = so.rhs(V, h)
    # the exact sum of the float64 values before rounding is 0; after rounding each to float, within their spacing
    assert abs(b.astype(np.float64).sum()) <= np.spacing(np.abs(b)).astype(np.float64).sum()
    assert np.array_equal(b[1:-1, 1:-1, 1:-1], mo.rhs(V, h)[1:-1, 1:-1, 1:-1])


def test_laplacian_is_neumann():
    L = so.laplacian(6)
    assert np.abs(L @ np.ones(7 ** 3)).max() == 0
    d = L.diagonal().reshape(7, 7, 7)
    assert d.min() == 3 and d.max() == 6 and np.array_equal(d, so.degree(6))


def test_coarse_screening_is_exact():
    rng = np.random.default_rng(3)
    N, w = 16, 2.7
    g = rng.uniform(0, N, (500, 3))
    g[:5] = [[0, 0, 0], [N, N, N], [N, 3.5, 0], [2, 4, 6], [N - 1e-9, 1e-9, 8]]   # faces and corners
    B0, B1 = so.weights(g, N), so.weights(g / 2, N // 2)
    P = so.prolongation(N // 2)
    lhs = 0.5 * (P.T @ (w * (B0.T @ B0)) @ P).toarray()
    rhs = (w / 2 * (B1.T @ B1)).toarray()
    assert np.abs(lhs - rhs).max() <= 1e-12 * np.abs(rhs).max()
    s = so.diagonals(g, N, w)
    assert np.allclose(s[1].reshape(-1), np.diag(rhs), rtol=1e-13, atol=0)
    assert np.allclose(np.asarray(B0.sum(1)).ravel(), 1.0, rtol=0, atol=1e-13)


def test_v_cycle_is_spd_and_contracts():
    x, _ = msc.sheet(3000)
    N = 8                                                                 # levels of 8 and 4 cells
    g = (x.astype(np.float64) + [1.2, 1.2, 1.2]) * (N / 2.4)             # the sheet inside the box, open to its faces
    w = ALPHA / 3000 * 8                                                  # about alpha / mean density
    A = (so.laplacian(N) + w * (so.weights(g, N).T @ so.weights(g, N))).toarray()
    s = so.diagonals(g, N, w)
    B = so.v_cycle_matrix(s)
    assert np.abs(B - B.T).max() <= 1e-12 * np.abs(B).max()
    assert np.linalg.eigvalsh((B + B.T) / 2).min() > 0
    rho = np.abs(np.linalg.eigvals(np.eye(len(B)) - B @ A)).max()
    print("V-cycle contraction on A at N = 8: %.3f" % rho)
    assert rho < CONTRACTION_BOUND


@pytest.mark.parametrize("depth", [5, 6])
@pytest.mark.parametrize("case", ["sheet", "sphere"])
def test_mgpcg_iterations(case, depth):
    x, n = msc.sheet(40000) if case == "sheet" else mc.sphere(20000)
    its = []
    for alpha in (1.0, 4.0, 16.0):
        A, b, w, g, N, o, h, D, s = so.system(x, n, depth, 1.1, alpha)
        chi, k, rel = so.mgpcg(A, b, s, 1e-5, 200)
        assert rel <= 1e-5
        its.append(k)
    print("%s depth %d: iterations %s for alpha 1, 4, 16" % (case, depth, its))
    assert max(its) <= MAX_ITERATIONS, its


# ---- meshes ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def sheet5():
    x, n = msc.sheet(40000, seed=SHEET_SEED)
    return x, n, so.mesh(x, n, depth=5, alpha=ALPHA), so.mesh(x, n, depth=5, alpha=ALPHA, trim=0.5)


def test_sheet_dirichlet_has_no_mesh(sheet5):
    """With chi = 0 on the boundary, chi at a one-sided sheet's points is 0 up to noise: its sign depends on the sample
    (seeds 0 to 3 give tau from -1.6e-3 to 3.6e-3 at depth 5), and on this one it gives status 2."""
    x, n, _, _ = sheet5
    m = mo.mesh(x, n, depth=5)
    assert m["tau"] <= 0 and abs(m["tau"]) <= 1e-2 * np.abs(m["chi"]).max()


def test_sheet_screened_is_one_component_ending_on_the_faces(sheet5):
    x, n, m, _ = sheet5
    t = m["triangles"]
    assert len(t) > 0 and mo.components(t, len(m["vertices"])) == 1
    e = so.boundary_edge_vertices(t)
    assert len(e) > 0
    face = so.on_faces(m["vertices"], m["o"], m["h"], m["N"])
    assert face[e].all()
    assert abs(m["tau"]) <= 1e-6 * np.abs(m["chi"]).max()


def test_sheet_screened_trimmed_is_accurate(sheet5):
    x, n, _, m = sheet5
    assert len(m["triangles"]) > 0 and mo.components(m["triangles"], len(m["vertices"])) == 1
    d = msc.sheet_distance(m["vertices"]) / m["h"]
    print("sheet depth 5 trim 0.5: mean %.4f h, worst %.3f h" % (d.mean(), d.max()))
    assert d.mean() <= SHEET_MEAN_BOUND and d.max() <= SHEET_MAX_BOUND


@pytest.mark.parametrize("case,euler", [("sphere", 2), ("torus", 0)])
def test_closed_shapes_stay_closed(case, euler):
    x, n = mc.sphere(20000) if case == "sphere" else mc.torus(20000)
    m = so.mesh(x, n, depth=5, alpha=ALPHA)
    t = m["triangles"]
    assert mo.closed_and_oriented(t) and mo.euler(t) == euler
    assert mo.components(t, len(m["vertices"])) == 1


def test_alpha_sweep():
    """The fidelity and iteration count of alpha on the sheet at depth 5 (the default is 4)."""
    x, n = msc.sheet(40000)
    rows = []
    for alpha in (0.25, 1.0, 4.0, 16.0, 64.0):
        m = so.mesh(x, n, depth=5, alpha=alpha, trim=0.5)
        A, b, w, g, N, o, h, D, s = so.system(x, n, 5, 1.1, alpha)
        k = so.mgpcg(A, b, s, 1e-5, 200)[1]
        d = msc.sheet_distance(m["vertices"]) / m["h"]
        rows.append((alpha, k, d.mean(), d.max()))
        print("alpha %5.2f: %2d iterations, mean %.4f h, worst %.3f h" % rows[-1])
    assert all(r[2] <= SHEET_MEAN_BOUND for r in rows if r[0] >= 1)


# ---- arguments ------------------------------------------------------------------------------------------------------

def _call(xyz=0x1000, nrm=0x2000, inten=None, P=4, depth=4, scale=1.1, alpha=4.0, it=10, tol=1e-5, trim=0.0,
          verts=0x10000, vint=None, maxV=4, tris=0x20000, maxT=4, chi=None):
    return cs.lib().cs_poisson_mesh_screened(xyz, nrm, inten, P, depth, scale, alpha, it, tol, trim, verts, vint, maxV,
                                             tris, maxT, chi, None, None, None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    assert msg.startswith("cs_poisson_mesh_screened: invalid argument (CS_E_ARG)"), msg
    for w in words:
        assert w in msg, (w, msg)


def test_argument_checks():
    for a in (0.0, -1.0, 1000.5, float("nan"), float("inf")):
        _rejects(_call(alpha=a), "pointWeight")
    _rejects(_call(P=-1), "numPoints")
    _rejects(_call(P=(1 << 30) + 1), "numPoints")
    _rejects(_call(depth=3), "depth")
    _rejects(_call(depth=10), "depth")
    _rejects(_call(scale=0.99), "scale")
    _rejects(_call(scale=4.5), "scale")
    _rejects(_call(scale=float("nan")), "scale")
    _rejects(_call(it=0), "maxIterations")
    _rejects(_call(it=1001), "maxIterations")
    _rejects(_call(tol=0.0), "tol")
    _rejects(_call(tol=1.0), "tol")
    _rejects(_call(tol=float("nan")), "tol")
    _rejects(_call(trim=-0.1), "trim")
    _rejects(_call(trim=float("inf")), "trim")
    _rejects(_call(maxV=-1), "maxVertices")
    _rejects(_call(maxT=-1), "maxTriangles")
    _rejects(_call(xyz=None), "d_xyz")
    _rejects(_call(xyz=0x1002), "d_xyz")
    _rejects(_call(nrm=None), "d_normal")
    _rejects(_call(verts=None), "d_vertices")
    _rejects(_call(tris=0x20001), "d_triangles")
    _rejects(_call(inten=0x3001, vint=0x4000), "d_intensity")
    _rejects(_call(inten=0x3000, vint=0x4002), "d_vertexIntensity")
    _rejects(_call(chi=0x5002), "d_chi")
    _rejects(_call(inten=0x3000), "d_intensity and d_vertexIntensity")
    _rejects(_call(vint=0x4000), "d_intensity and d_vertexIntensity")


def test_every_overlap_is_rejected_and_named():
    rng = np.random.default_rng(11)
    for _ in range(300):
        P, V, T = int(rng.integers(1, 50)), int(rng.integers(1, 50)), int(rng.integers(1, 50))
        with_i, with_chi = bool(rng.integers(0, 2)), bool(rng.integers(0, 2))
        sizes = {"d_xyz": 12 * P, "d_normal": 12 * P, "d_vertices": 12 * V, "d_triangles": 12 * T}
        if with_i:
            sizes.update({"d_intensity": 4 * P, "d_vertexIntensity": 4 * V})
        if with_chi:
            sizes["d_chi"] = 4 * 17 ** 3
        outs = {"d_vertices", "d_triangles", "d_vertexIntensity", "d_chi"}
        forbidden = lambda a, b: a in outs or b in outs
        at = _layout(rng, sizes, forbidden)
        g = lambda x: BASE + at[x] if x in at else None
        r = cs.lib().cs_poisson_mesh_screened(g("d_xyz"), g("d_normal"), g("d_intensity"), P, 4, 1.1, ALPHA, 10, 1e-5,
                                              0.0, g("d_vertices"), g("d_vertexIntensity"), V, g("d_triangles"), T,
                                              g("d_chi"), None, None, None)
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
    assert "int cs_poisson_mesh_screened(" in hdr and "10 kernel launches" in hdr and "pointWeight" in hdr
    assert isinstance(cs.lib().cs_poisson_mesh_screened, ctypes._CFuncPtr)
