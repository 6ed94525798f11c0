"""CPU checks of cs_clean_mesh's rules on tests/clean_oracle.py: one case per rule, rule mutations the checks must
see, the topology of a filled sphere, all stages off, the argument checks through the built library (no GPU call is
made) and the header."""
import ctypes
import math
import os

import numpy as np
import pytest

import clean_cases as cc
import clean_oracle as co
import cudasift_b200 as cs

CS_E_ARG = -2


def _run(name, mutation=None, **kw):
    v, t, i = cc.CASES[name]()
    return v, t, co.clean(v, t, i, mutation=mutation, **dict(cc.SETTINGS.get(name, {}), **kw))


def test_degenerate_faces():
    v, t, r = _run("zero_area")
    assert r["stats"][1] == 2 and r["stats"][2] == 0
    assert not any(set(f) in ({0, 11, 22}, {12, 13, len(v) - 1}) for f in map(set, r["triangles"].tolist()))
    assert len(r["vertices"]) == len(v) - 1           # the coincident copy is used by the dropped face only


def test_enclosed_zero_area_face_stays():
    v, t, r = _run("enclosed_slivers")
    assert r["stats"][1] == 0 and np.array_equal(r["triangles"], t)
    assert co.topology(r["triangles"]) == co.topology(t)
    # dropped, it would leave a flat slit of 3 edges that no allowed ear closes
    _, _, m = _run("enclosed_slivers", mutation="drop_enclosed")
    assert m["stats"][1] == 1 and m["stats"][9:12] == [2, 0, 2]
    assert co.topology(m["triangles"])[0] == co.topology(t)[0] + 3


def test_duplicates_keep_lowest():
    v, t, r = _run("duplicates")
    assert r["stats"][2] == 3
    assert np.array_equal(r["triangles"][0], t[0])    # the reversed copy in front stays, the original goes
    assert len(r["triangles"]) == len(t) - 3


def test_long_edge_fan_and_islands():
    v, t, r = _run("sphere_mess")
    s = r["stats"]
    assert s[3] == 6 and s[5] == 24 and s[7] == 3 and s[6] == 4
    assert r["info"][2] == r["info"][0] + 3.0 * r["info"][1]
    assert np.abs(np.linalg.norm(r["vertices"], axis=1) - 1).max() < 1e-5     # only the sphere is left


def test_fin_drops_the_highest_face():
    v, t, r = _run("fin")
    assert r["stats"][4] == 1
    assert np.array_equal(r["triangles"], t[:-1])
    assert co.topology(r["triangles"])[1] == 0


def test_holes_filled_up_to_max_edges():
    v, t, i = cc.holes()
    for m, filled, open_ in ((40, 4, 1), (30, 3, 2), (8, 3, 2), (4, 2, 3), (3, 1, 4)):
        r = co.clean(v, t, i, maxHoleEdges=m)
        assert r["stats"][9:12] == [5, filled, open_], (m, r["stats"])
    r = co.clean(v, t, i, maxHoleEdges=40)
    assert r["stats"][13] == 1 + 2 + 6 + 38
    assert co.topology(r["triangles"]) == (120, 0, 1, True)


def test_bowtie_rim_stays_open():
    v, t, r = _run("bowtie")
    s = r["stats"]
    assert s[8] == 1 and s[10] == 0 and s[12] == 8
    assert len(r["triangles"]) == len(t)


def test_filled_sphere_is_closed_and_oriented():
    v, t, r = _run("sphere_mess")
    assert r["stats"][10] == 2
    assert co.topology(r["triangles"]) == (0, 0, 2, True)


def test_all_stages_off_keeps_the_input():
    v, t, i = cc.sphere_mess()
    r = co.clean(v, t, i, **co.OFF)
    used = np.unique(t)
    remap = np.full(len(v), -1)
    remap[used] = np.arange(len(used))
    assert np.array_equal(r["triangles"], remap[t])
    assert np.array_equal(r["vertices"], v[used]) and np.array_equal(r["intensity"], i[used])
    assert r["stats"][1:6] == [0] * 5 and r["stats"][9:14] == [0] * 5


def test_smoothing_keeps_boundary_and_flatness():
    v, t, i = cc.holes()
    r0 = co.clean(v, t, i, maxHoleEdges=8)
    r = co.clean(v, t, i, maxHoleEdges=8, smoothIterations=3)
    assert np.array_equal(r["triangles"], r0["triangles"])
    assert (r["vertices"][:, 2] == 0).all()
    b = np.unique(np.asarray(co.boundary_loops(r0["triangles"].astype(np.int64),
                                                np.ones(len(r0["triangles"]), bool))[0][0])[:, 0])
    assert np.array_equal(r["vertices"][b], r0["vertices"][b])
    assert not np.array_equal(r["vertices"], r0["vertices"])


def test_unused_vertices_dropped():
    v, t, r = _run("sphere_mess")
    assert len(r["vertices"]) == len(np.unique(r["triangles"]))
    assert r["stats"][14] < len(v)


@pytest.mark.parametrize("mutation,case", [("keep_highest", "duplicates"), ("ear_tie_last", "holes"),
                                           ("fill_reversed", "holes"), ("fill_reversed", "sphere_mess")])
def test_mutations_change_an_output(mutation, case):
    _, _, r = _run(case)
    _, _, m = _run(case, mutation=mutation)
    assert not np.array_equal(r["triangles"], m["triangles"])
    if mutation == "fill_reversed":
        assert not co.topology(m["triangles"])[3]      # the orientation check sees it


def test_sheet_meshes():
    for trim, (v, t) in cc.sheet_meshes().items():
        r = co.clean(v, t)
        s = r["stats"]
        sizes = co.components(r["triangles"])
        print("sheet trim %.1f: %d faces, %d components, %d loops (%d filled), %d non-manifold vertices -> %d faces, "
              "smallest component %d" % (trim, s[0], s[6], s[9], s[10], s[8], s[15], sizes.min()))
        assert sizes.min() >= 50
        assert co.topology(r["triangles"])[1] == 0


# ---- argument checks and header -------------------------------------------------------------------------------------
def _call(V=4, T=4, verts=0x1000, tris=0x2000, outv=0x3000, outt=0x4000, deg=1, lef=20.0, nm=1, mcf=50, mcfr=0.0,
          hole=30, it=0, lam=0.5, mu=-0.53):
    return cs.lib().cs_clean_mesh(verts, None, V, tris, T, deg, lef, nm, mcf, mcfr, hole, it, lam, mu, outv, None, V,
                                  outt, T, None, None, None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    assert msg.startswith("cs_clean_mesh: invalid argument (CS_E_ARG)"), msg
    for w in words:
        assert w in msg, (w, msg)


def test_argument_checks():
    _rejects(_call(T=-1), "numTriangles")
    _rejects(_call(T=(1 << 26) + 1), "numTriangles")
    _rejects(_call(V=-1), "numVertices")
    for d in (-1, 2):
        _rejects(_call(deg=d), "removeDegenerate")
        _rejects(_call(nm=d), "removeNonManifold")
    for x in (-0.5, math.inf, math.nan):
        _rejects(_call(lef=x), "longEdgeFactor")
    _rejects(_call(mcf=-1), "minComponentFaces")
    for x in (-0.1, 1.5, math.nan):
        _rejects(_call(mcfr=x), "minComponentFraction")
    for h in (-1, 1, 2, 257):
        _rejects(_call(hole=h), "maxHoleEdges")
    for n in (-1, 1001):
        _rejects(_call(it=n), "smoothIterations")
    for x in (0.0, 1.5, math.nan):
        _rejects(_call(lam=x), "lambda")
    for x in (0.0, -1.5, 0.5, math.nan):
        _rejects(_call(mu=x), "mu")
    _rejects(_call(verts=0), "d_vertices")
    _rejects(_call(verts=0x1002), "d_vertices")
    _rejects(_call(tris=0), "d_triangles")
    _rejects(_call(outv=0), "d_outVertices")
    _rejects(_call(outt=0x2004), "overlap")


def test_empty_mesh_makes_no_call():
    stats = np.full(19, -1, np.int64)
    assert cs.lib().cs_clean_mesh(None, None, 0, None, 0, 1, 20.0, 1, 50, 0.0, 30, 0, 0.5, -0.53, None, None, 0,
                                  None, 0, None, stats.ctypes.data_as(ctypes.c_void_p), None) == 0
    assert (stats == 0).all()


def test_header_declares_the_call():
    hdr = open(os.path.join(os.path.dirname(cs.__file__), "..", "include", "cudasift_b200.h")).read()
    assert "int cs_clean_mesh(" in hdr and "292 bytes per triangle" in hdr
    f = cs.lib().cs_clean_mesh
    assert len(f.argtypes) == 22 and f.argtypes[6] is ctypes.c_double and f.argtypes[12] is ctypes.c_double
