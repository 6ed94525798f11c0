"""CPU checks of the Poisson mesher's rules (tests/mesh_oracle.py) and of cs_poisson_mesh's argument checks: the
extraction is closed and oriented on every corner pattern and on random fields, the Euler characteristic is right on
analytic fields, the oracle's solve and mesh are accurate on a sphere, and the V-cycle is a symmetric positive-definite
preconditioner that contracts."""
import ctypes
import itertools

import numpy as np
import pytest

import cudasift_b200 as cs
import mesh_cases as mc
import mesh_oracle as mo
from test_arg_ranges_cpu import BASE, MSG, _buf, _layout, _share

CS_E_ARG = -2
SPHERE_RADIUS_BOUND = 0.5      # |r - R| / h of every oracle vertex on the depth-6 sphere (0.36 observed)
CONTRACTION_BOUND = 0.2        # spectral radius of I - B A for the V-cycle B at N = 8 (0.134 observed)


def _padded(core):
    """core values in the interior of a grid one node larger on every side, padded with outside nodes (0 < tau)."""
    out = np.zeros(tuple(s + 2 for s in core.shape), np.float32)
    out[1:-1, 1:-1, 1:-1] = core
    return out


def test_every_corner_pattern_gives_a_closed_oriented_mesh():
    rng = np.random.default_rng(0)
    for pattern in range(256):
        core = np.zeros((2, 2, 2), np.float32)
        for c in range(8):
            core[(c >> 2) & 1, (c >> 1) & 1, c & 1] = rng.uniform(0.6, 1.5) if (pattern >> c) & 1 else rng.uniform(0, 0.4)
        m = mo.extract(_padded(core), 0.5)
        tris = m["triangles"]
        assert (len(tris) == 0) == (pattern == 0), pattern
        assert mo.closed_and_oriented(tris), pattern


def test_random_fields_give_closed_oriented_meshes():
    rng = np.random.default_rng(1)
    for trial in range(40):
        core = rng.uniform(0, 1, tuple(int(v) for v in rng.integers(2, 7, 3))).astype(np.float32)
        m = mo.extract(_padded(core), 0.5)
        assert mo.closed_and_oriented(m["triangles"]), trial
        assert len(m["vertices"]) == m["pre"][0]                 # trim 0 keeps every vertex


def test_orientation_points_outward_and_ties_keep_topology():
    f = mc.sphere_field(24, 8.3)
    m = mo.extract(f, 0.0)
    v, t = m["vertices"].astype(np.float64), m["triangles"]
    n = np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]])
    c = v[t].mean(1) - (24 / 2 + 0.137)
    assert ((n * c).sum(1) > 0).mean() >= 0.99
    q = np.round(f * 2) / 2                                        # many nodes exactly at tau: t = 0 ties
    m = mo.extract(q, 0.0)
    assert mo.closed_and_oriented(m["triangles"])


@pytest.mark.parametrize("field,chi", [("sphere", 2), ("torus", 0)])
def test_euler_characteristic_on_analytic_fields(field, chi):
    f = mc.sphere_field(32, 11.2) if field == "sphere" else mc.torus_field(32, 9.3, 3.4)
    m = mo.extract(f, 0.0)
    t = m["triangles"]
    assert mo.closed_and_oriented(t)
    assert mo.euler(t) == chi
    assert mo.components(t, len(m["vertices"])) == 1


def test_oracle_solve_and_sphere_mesh():
    x, n = mc.sphere(20000)
    m = mo.mesh(x, n, depth=6)
    A = mo.operator(64)
    b = mo.interior(m["b"]).astype(np.float64)
    assert np.linalg.norm(A @ mo.interior(m["chi"]) - b) <= 1e-10 * np.linalg.norm(b)
    assert m["tau"] > 0
    r = np.linalg.norm(m["vertices"] - mc.CENTRE, axis=1)
    assert np.abs(r - 1.0).max() <= SPHERE_RADIUS_BOUND * m["h"]
    t = m["triangles"]
    assert mo.closed_and_oriented(t) and mo.euler(t) == 2


def test_v_cycle_is_spd_and_contracts():
    B = mo.v_cycle_matrix(8)
    A = mo.operator(8).toarray()
    assert np.abs(B - B.T).max() <= 1e-12 * np.abs(B).max()
    assert np.linalg.eigvalsh((B + B.T) / 2).min() > 0
    assert np.abs(np.linalg.eigvals(np.eye(len(A)) - B @ A)).max() < CONTRACTION_BOUND


def test_mgpcg_iterations_do_not_grow_with_n():
    its = []
    for depth in (4, 5, 6):
        x, n = mc.sphere(8000)
        g, nh, _, N, o, h, ok, _ = mo.sorted_points(x, n, None, depth, 1.1)
        V, D, _ = mo.splat(g, nh, None, N)
        its.append(mo.mgpcg(mo.rhs(V, h), 1e-5, 200)[1])
    assert max(its) <= min(its) + 3, its


# ---- arguments ------------------------------------------------------------------------------------------------------

def _call(xyz=0x1000, nrm=0x2000, inten=None, P=4, depth=4, scale=1.1, it=10, tol=1e-5, trim=0.0, verts=0x10000,
          vint=None, maxV=4, tris=0x20000, maxT=4, chi=None):
    return cs.lib().cs_poisson_mesh(xyz, nrm, inten, P, depth, scale, it, tol, trim, verts, vint, maxV, tris, maxT, chi,
                                    None, None, None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    assert msg.startswith("cs_poisson_mesh: invalid argument (CS_E_ARG)"), msg
    for w in words:
        assert w in msg, (w, msg)


def test_argument_checks():
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


def _mesh_layout(rng):
    P, V, T, depth = int(rng.integers(1, 50)), int(rng.integers(1, 50)), int(rng.integers(1, 50)), 4
    with_i = bool(rng.integers(0, 2))
    with_chi = bool(rng.integers(0, 2))
    sizes = {"d_xyz": 12 * P, "d_normal": 12 * P, "d_vertices": 12 * V, "d_triangles": 12 * T}
    if with_i:
        sizes.update({"d_intensity": 4 * P, "d_vertexIntensity": 4 * V})
    if with_chi:
        sizes["d_chi"] = 4 * 17 ** 3
    outs = {"d_vertices", "d_triangles", "d_vertexIntensity", "d_chi"}

    def make(at):
        g = lambda x: at.get(x)
        return cs.lib().cs_poisson_mesh(g("d_xyz"), g("d_normal"), g("d_intensity"), P, depth, 1.1, 10, 1e-5, 0.0,
                                        g("d_vertices"), g("d_vertexIntensity"), V, g("d_triangles"), T, g("d_chi"),
                                        None, None, None)

    return sizes, (lambda a, b: a in outs or b in outs), make


def test_every_mesh_overlap_is_rejected_and_named():
    rng = np.random.default_rng(7)
    for _ in range(300):
        sizes, forbidden, make = _mesh_layout(rng)
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
    import os
    hdr = open(os.path.join(os.path.dirname(cs.__file__), "..", "include", "cudasift_b200.h")).read()
    assert "int cs_poisson_mesh(" in hdr and "10 kernel launches" in hdr
    assert isinstance(cs.lib().cs_poisson_mesh, ctypes._CFuncPtr)
