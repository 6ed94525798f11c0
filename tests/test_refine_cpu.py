"""CPU checks of cs_mesh_refine's rules on tests/refine_oracle.py: each case of refine_cases reaches its rule, and a
mutation of each rule changes some case's output; the gradient checks (the thin-plate gradient against central
differences of E_s, the photometric gradient against central differences of E_photo at h = 1e-6 l0 wherever no pixel
changes state); on the small jittered scene the oracle lowers E and the RMS distance of the free vertices to their
true planes, which fixes RMS_FACTOR for the GPU test; the argument checks; and the header."""
import ctypes
import math
import os

import numpy as np
import pytest

import cudasift_b200 as cs
import refine_cases as rc
import refine_oracle as ro
from test_texture_cpu import IMG, KS, RS, TS

CS_E_ARG = -2
# The call's defaults (RefineMesh's), used by the oracle and GPU tests.
DEFAULTS = dict(windowRadius=4, smoothness=0.2, step=0.1, maxIterations=100, depthTol=0.01)
# The oracle's run in test_jittered_scene_improves lowers the RMS plane distance of the free vertices by this factor
# or more; the GPU test at 640 x 480 asserts the same factor.
RMS_FACTOR = 0.71


def _cams(c):
    return [(np.asarray(c["Ks"][a], np.float64), np.asarray(c["Rs"][a], np.float64), np.asarray(c["ts"][a], np.float64),
             c["imgs"][a].shape[1], c["imgs"][a].shape[0]) for a in range(len(c["imgs"]))]


def _eval(c, X, topo, P0=None, bufs=None, smoothness=0.1):
    kw = DEFAULTS | c["kw"]
    return ro.evaluate(c["imgs"], _cams(c), X, np.asarray(c["t"], np.int64), [tuple(p) for p in c["pairs"]], topo,
                       kw["windowRadius"], kw["depthTol"], smoothness, P0=P0, bufs=bufs)


def _refine(c, **over):
    kw = DEFAULTS | c["kw"] | over
    return ro.refine(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], c["pairs"], **kw)


# ---- each case reaches its rule -------------------------------------------------------------------------------------
def test_fixed_vertices():
    c = rc.fixed_vertices()
    topo = ro.topology(len(c["v"]), c["t"], c["v"].astype(np.float64))
    t = np.asarray(c["t"])
    used = np.zeros(len(c["v"]), bool)
    used[t.reshape(-1)] = True
    assert (~used).sum() == 2 and not topo["free"][~used].any()
    assert not topo["free"][23] and not topo["free"][24]          # the fin's edge has three faces
    assert not topo["free"][0] and topo["free"][12]               # a grid corner (boundary) and an interior vertex
    r = _refine(c, maxIterations=4)
    moved = (r["vertices"] != c["v"]).any(1)
    assert moved.any() and not moved[~topo["free"]].any()


def test_occluder_unmaps_pixels():
    c = rc.occluder()
    topo = ro.topology(len(c["v"]), c["t"], c["v"].astype(np.float64))
    e = _eval(c, c["v"].astype(np.float64), topo)
    keyed = (e["bufs"][0].reshape(-1) != ro.EMPTY).sum()
    loose = dict(c, kw=dict(depthTol=1.0))
    e1 = _eval(loose, c["v"].astype(np.float64), topo)
    assert e["pairs"][0]["mapped"].sum() < e1["pairs"][0]["mapped"].sum() <= keyed


def test_windows_cut_by_border_and_holes():
    c = rc.windows_cut()
    topo = ro.topology(len(c["v"]), c["t"], c["v"].astype(np.float64))
    e = _eval(c, c["v"].astype(np.float64), topo)
    p = e["pairs"][0]
    H, W = c["imgs"][0].shape
    m, s = p["mapped"].reshape(H, W), p["scoredMask"].reshape(H, W)
    edge = np.zeros_like(m)
    edge[:3], edge[-3:], edge[:, :3], edge[:, -3:] = True, True, True, True
    assert (m & edge).any() and not (s & edge).any()             # mapped at the border, never scored there
    assert ((m & ~s) & ~edge).any() and p["scored"] > 0           # windows cut by the holes


def test_flat_texture_hits_the_floor(monkeypatch):
    c = rc.flat()
    a = _refine(c, maxIterations=4)
    monkeypatch.setattr(ro, "FLOOR", 0.25)
    b = _refine(c, maxIterations=4)
    assert a["info"] != b["info"]


def test_repeated_pair_counts_twice():
    c = rc.repeated()
    topo = ro.topology(len(c["v"]), c["t"], c["v"].astype(np.float64))
    e = _eval(c, c["v"].astype(np.float64), topo)
    assert e["pairs"][0]["scored"] == e["pairs"][2]["scored"] and e["scored"] == 2 * e["pairs"][0]["scored"] + \
        e["pairs"][1]["scored"]


def test_line_search_rejects_and_halves():
    trace = []
    c = rc.rejects()
    kw = DEFAULTS | c["kw"] | dict(maxIterations=8)
    r = ro.refine(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], c["pairs"], trace=trace, **kw)
    assert any(not ok for _, ok in trace) and r["stats"][4] > r["stats"][5] + 1
    E = lambda i: i[0] + kw["smoothness"] * i[1]
    assert E(r["info"][2:]) <= E(r["info"][:2])


@pytest.mark.parametrize("mutation", ["cap", "floor", "free"])
def test_mutations_change_an_output(monkeypatch, mutation):
    c = rc.repeated()
    a = _refine(c, maxIterations=4)
    if mutation == "cap":
        monkeypatch.setattr(ro, "CAP", 1.0)
        c = rc.rejects()
        a = _refine(c, maxIterations=4)
        monkeypatch.setattr(ro, "CAP", 0.5)
    elif mutation == "floor":
        monkeypatch.setattr(ro, "FLOOR", 400.0)
    else:
        real = ro.topology

        def loose(V, tris, X):
            t = real(V, tris, X)
            used = np.zeros(V, bool)
            used[np.asarray(tris).reshape(-1)] = True
            return t | dict(free=used, F=int(used.sum()))
        monkeypatch.setattr(ro, "topology", loose)
    b = _refine(c, maxIterations=4)
    assert a["info"] != b["info"] or a["vertices"].tobytes() != b["vertices"].tobytes()


# ---- gradient checks ------------------------------------------------------------------------------------------------
def test_thin_plate_gradient():
    c = rc.repeated()
    X = c["v"].astype(np.float64)
    topo = ro.topology(len(X), c["t"], X)
    base = _eval(dict(c, pairs=np.zeros((0, 2), np.int32)), X, topo, P0=1, smoothness=1.0)
    h = 1e-6 * topo["l0"]
    rng = np.random.default_rng(1)
    for v in np.nonzero(topo["free"])[0]:
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        ev = lambda s: _eval(dict(c, pairs=np.zeros((0, 2), np.int32)), X + s * h * np.outer(np.arange(len(X)) == v, d),
                             topo, P0=1, smoothness=1.0)["es"]
        fd = (ev(1) - ev(-1)) / (2 * h)
        assert abs(fd - base["G"][v] @ d) <= 1e-5 * np.abs(base["G"]).max(), (v, fd, base["G"][v] @ d)


@pytest.mark.parametrize("name", ["repeated", "windows_cut", "occluder"])
def test_photometric_gradient(name):
    c = rc.CASES[name]()
    X = c["v"].astype(np.float64)
    topo = ro.topology(len(X), c["t"], X)
    base = _eval(c, X, topo, smoothness=0.0)
    h = 1e-6 * topo["l0"]
    nrm = np.zeros_like(X)
    P = X[np.asarray(c["t"], np.int64)]
    np.add.at(nrm, np.asarray(c["t"]).reshape(-1), np.repeat(ro.normals(P), 3, axis=0))
    checked = 0
    scale = np.abs(base["G"]).max()
    for v in np.nonzero(topo["free"])[0][::3]:
        d = nrm[v] / np.linalg.norm(nrm[v])
        Xp, Xm = X.copy(), X.copy()
        Xp[v] += h * d
        Xm[v] -= h * d
        ep = _eval(c, Xp, topo, P0=base["P0"], bufs=base["bufs"], smoothness=0.0)
        em = _eval(c, Xm, topo, P0=base["P0"], bufs=base["bufs"], smoothness=0.0)
        if not all((a["mapped"] == b["mapped"]).all() and (a["scoredMask"] == b["scoredMask"]).all()
                   for a, b in zip(ep["pairs"], em["pairs"])):
            continue
        fd = (ep["ep"] - em["ep"]) / (2 * h)
        assert abs(fd - base["G"][v] @ d) <= 1e-4 * scale, (v, fd, base["G"][v] @ d)
        checked += 1
    assert checked >= 10


# ---- the jittered scene ---------------------------------------------------------------------------------------------
def test_jittered_scene_improves():
    c = rc.scene()
    r = _refine(c, maxIterations=12)
    free = r["topo"]["free"]
    before = rc.plane_rms(c["v"], c["rect"], c["rects"], free)
    after = rc.plane_rms(r["vertices"], c["rect"], c["rects"], free)
    E = lambda i: i[0] + DEFAULTS["smoothness"] * i[1]
    print("scene: info %s stats %s rms %.6f -> %.6f (%.4f)" % (r["info"], r["stats"], before, after, after / before))
    assert E(r["info"][2:]) < E(r["info"][:2]) and r["stats"][5] > 0
    assert after <= RMS_FACTOR * before


# ---- argument checks and header -------------------------------------------------------------------------------------
PAIRS = np.array([[0, 1], [1, 0]], np.int32)


def _call(pairs=PAIRS, n=2, T=4, V=4, verts=0x1000, tris=0x2000, out=0x3000, rho=2, smooth=0.1, step=0.05, its=10,
          tol=0.01):
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    return cs.lib().cs_mesh_refine(IMG, 2, p(KS), p(RS), p(TS), verts, V, tris, T,
                                   p(pairs) if pairs is not None else None, n, rho, smooth, step, its, tol, out, None,
                                   None, None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    assert msg.startswith("cs_mesh_refine: invalid argument (CS_E_ARG)"), msg
    for w in words:
        assert w in msg, (w, msg)


def test_argument_checks():
    _rejects(_call(V=-1), "numVertices")
    _rejects(_call(T=-1), "numTriangles")
    _rejects(_call(T=(1 << 28) + 1), "numTriangles")
    _rejects(_call(n=-1), "numPairs")
    _rejects(_call(pairs=None), "pairs")
    for bad in ([0, 2], [-1, 0], [1, 1]):
        _rejects(_call(pairs=np.array([[0, 1], bad], np.int32)), "pairs[1]")
    for rho in (0, 6):
        _rejects(_call(rho=rho), "windowRadius")
    for s in (-0.1, math.inf, math.nan):
        _rejects(_call(smooth=s), "smoothness")
    for s in (0.0, -0.1, 1.5, math.nan):
        _rejects(_call(step=s), "step")
    for its in (-1, 1001):
        _rejects(_call(its=its), "maxIterations")
    for tol in (-0.1, 1.5, math.nan):
        _rejects(_call(tol=tol), "depthTol")
    _rejects(_call(verts=0x1002), "d_vertices")
    _rejects(_call(verts=0), "d_vertices")
    _rejects(_call(out=0), "d_outVertices")
    _rejects(_call(tris=0x2001), "d_triangles")
    _rejects(_call(out=0x1010), "overlap")
    _rejects(_call(out=0x100010), "overlap")


def test_header_declares_the_call():
    hdr = open(os.path.join(os.path.dirname(cs.__file__), "..", "include", "cudasift_b200.h")).read()
    assert "int cs_mesh_refine(" in hdr
    assert "evaluations (5 numPairs + 5) + evaluations - 1" in hdr and "240 bytes per face" in hdr
    f = cs.lib().cs_mesh_refine
    assert len(f.argtypes) == 20 and f.argtypes[12] is ctypes.c_double and f.argtypes[14] is ctypes.c_int
