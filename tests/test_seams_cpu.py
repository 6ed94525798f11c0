"""CPU checks of seam levelling (tests/seam_oracle.py) and of cs_level_texture_seams's argument checks: the system is
symmetric positive definite, the exact solution never raises the seam energy, per-view constant offsets are recovered
up to a common shift, a sweep of smoothness and regularization that fixed the defaults, every CS_E_ARG case with the
overlap sweeps (buffers and chart rectangles), every chart table the texturing oracle writes passing the chart
checks, and texture.o's kernels unchanged by the helpers it now shares with seams.cu."""
import ctypes
import hashlib
import math
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import seam_oracle as so
import texture_cases as tc
import texture_oracle as to
from cudasift_b200 import build
from test_arg_ranges_cpu import BASE, MSG, _buf, _layout, _share
from test_bundle_intrinsics_cpu import _sass

CS_E_ARG = -2


@pytest.fixture(scope="module")
def scene():
    imgs, Ks, Rs, ts, _ = tc.scene_views()
    v, t = tc.scene_mesh()
    r = to.texture(imgs, Ks, Rs, ts, v, t, lam=0.5)
    return imgs, Ks, Rs, ts, v, t, r


def _shifted(imgs, Ks, Rs, ts, v, t, r, offsets):
    q = to.texture([im + np.float32(o) for im, o in zip(imgs, offsets)], Ks, Rs, ts, v, t, lam=0.5, bufs=r["bufs"])
    assert np.array_equal(q["labels"], r["labels"])
    return q


def test_system_is_spd_and_levelling_never_raises_the_energy(scene):
    imgs, Ks, Rs, ts, v, t, r = scene
    rng = np.random.default_rng(4)
    q = _shifted(imgs, Ks, Rs, ts, v, t, r, rng.uniform(-20, 20, len(imgs)))
    for smooth, reg in ((0.1, 1e-3), (1.0, 1e-2), (0.01, 1e-4)):
        b = so.build(v, t, q["labels"], q["uv"], q["charts"], q["atlas"], smooth)
        A, rhs = so.system(b, reg)
        D = A.toarray()
        assert np.array_equal(D, D.T) and np.linalg.eigvalsh(D).min() > 0
        g = so.solve_exact(b, reg)
        assert so.energy(b, g) <= so.energy(b)


def test_constant_offsets_are_recovered(scene):
    """Views that differ by a constant per image: at every seam vertex g(v, a) - g(v, b) recovers c_b - c_a."""
    imgs, Ks, Rs, ts, v, t, r = scene
    c = np.array([0.0, 12.0, -7.0, 25.0, -15.0, 5.0])
    # the unperturbed scene's own seam targets are the baseline; the shifted scene adds c_b - c_a to every target
    b0 = so.build(v, t, r["labels"], r["uv"], r["charts"], r["atlas"], 0.0)
    q = _shifted(imgs, Ks, Rs, ts, v, t, r, c)
    b1 = so.build(v, t, q["labels"], q["uv"], q["charts"], q["atlas"], 0.0)
    g0, g1 = so.solve_exact(b0, 1e-9), so.solve_exact(b1, 1e-9)
    dg = g1 - g0
    keys = b1["keys"]
    for i, j, _, _ in b1["seam"]:
        (va, la), (vb, lb) = keys[i], keys[j]
        assert va == vb
        assert abs((dg[i] - dg[j]) - (c[lb] - c[la])) < 1e-3, (keys[i], keys[j])


def test_sweep_of_smoothness_and_regularization(scene):
    """Seam energy after / before and the median |offset| on the scene with per-view gain and offset.  The defaults
    (smoothness 0.1, regularization 1e-3) keep the energy ratio near its floor while the offsets stay bounded."""
    imgs, Ks, Rs, ts, v, t, r = scene
    rng = np.random.default_rng(1)
    gain, off = 1 + rng.uniform(-0.2, 0.2, len(imgs)), rng.uniform(-20, 20, len(imgs))
    q = to.texture([(im * g + o).astype(np.float32) for im, g, o in zip(imgs, gain, off)], Ks, Rs, ts, v, t, lam=0.5,
                   bufs=r["bufs"])
    rows = {}
    for smooth in (0.01, 0.1, 1.0):
        b = so.build(v, t, q["labels"], q["uv"], q["charts"], q["atlas"], smooth)
        e0 = so.energy(b)
        for reg in (1e-4, 1e-3, 1e-2, 1e-1):
            g = so.solve_exact(b, reg)
            rows[(smooth, reg)] = (so.energy(b, g) / e0, float(np.median(np.abs(g))))
            print("smoothness %-5g regularization %-6g energy ratio %.4f median |g| %.2f"
                  % (smooth, reg, *rows[(smooth, reg)]))
    ratio, size = rows[(0.1, 1e-3)]
    assert ratio <= 0.02 and size < 20
    assert ratio <= 1.5 * min(x for x, _ in rows.values())


# ---- library --------------------------------------------------------------------------------------------------------
CHARTS = np.array([[0, 0, 0, 10, 4, 0, 0, 3], [1, 0, 0, 12, 3, 10, 0, 2]], np.int32)


def _call(verts=0x1000, V=4, tris=0x2000, T=4, view=0x3000, uv=0x4000, charts=CHARTS, nc=2, atlas=0x10000, rows=4,
          width=32, pad=2, smooth=0.1, reg=1e-3, its=1000, tol=1e-4, out=0x20000, corner=0x30000):
    p = charts.ctypes.data_as(ctypes.c_void_p) if charts is not None else None
    return cs.lib().cs_level_texture_seams(verts, V, tris, T, view, uv, p, nc, atlas, rows, width, pad, smooth, reg,
                                           its, tol, out, corner, None, None, None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    assert msg.startswith("cs_level_texture_seams: invalid argument (CS_E_ARG)"), msg
    for w in words:
        assert w in msg, (w, msg)


def test_argument_checks():
    _rejects(_call(V=-1), "numVertices")
    _rejects(_call(V=(1 << 30) + 1), "numVertices")
    _rejects(_call(T=-1), "numTriangles")
    _rejects(_call(T=(1 << 29) + 1), "numTriangles")
    _rejects(_call(rows=-1), "atlasRows")
    for width in (0, 32769):
        _rejects(_call(width=width), "atlasWidth")
    for pad in (-1, 17):
        _rejects(_call(pad=pad), "padding")
    for smooth in (-0.1, math.inf, math.nan):
        _rejects(_call(smooth=smooth), "smoothness")
    for reg in (0.0, -1.0, math.inf, math.nan):
        _rejects(_call(reg=reg), "regularization")
    for its in (-1, 100001):
        _rejects(_call(its=its), "maxIterations")
    for tol in (-0.1, 1.0, math.nan):
        _rejects(_call(tol=tol), "tol")
    _rejects(_call(nc=-1), "numCharts")
    _rejects(_call(charts=None), "charts")
    for k, bad in ((0, -1), (3, 0), (4, 0), (5, -1), (6, -1), (5, 21), (6, 2)):
        c = CHARTS.copy()
        c[1, k] = bad
        _rejects(_call(charts=c), "charts[1]")
    _rejects(_call(verts=None), "d_vertices")
    _rejects(_call(verts=0x1002), "d_vertices")
    _rejects(_call(tris=None), "d_triangles")
    _rejects(_call(tris=0x2001), "d_triangles")
    _rejects(_call(view=None), "d_faceView")
    _rejects(_call(view=0x3001), "d_faceView")
    _rejects(_call(uv=None), "d_uv")
    _rejects(_call(uv=0x4002), "d_uv")
    _rejects(_call(corner=None), "d_cornerOffset")
    _rejects(_call(corner=0x30002), "d_cornerOffset")
    _rejects(_call(atlas=None), "d_atlas")
    _rejects(_call(atlas=0x10001), "d_atlas")
    _rejects(_call(out=None), "d_outAtlas")
    _rejects(_call(out=0x20002), "d_outAtlas")
    # charts whose rectangles share a texel, named by both indices: nested, partial, the same ox, the same oy, and
    # three charts of which only the last overlaps the first
    for rects, pair in (([(0, 0, 20, 4), (5, 1, 3, 2)], (0, 1)),
                        ([(0, 0, 10, 4), (9, 3, 5, 1)], (0, 1)),
                        ([(4, 0, 6, 2), (4, 1, 2, 3)], (0, 1)),
                        ([(0, 2, 4, 1), (3, 2, 8, 2)], (0, 1)),
                        ([(2, 0, 6, 2), (0, 2, 3, 2), (0, 1, 3, 1)], (0, 2)),
                        ([(0, 0, 32, 4), (31, 3, 1, 1)], (0, 1))):
        c = np.array([[l, 0, 0, w, h, ox, oy, 1] for l, (ox, oy, w, h) in enumerate(rects)], np.int32)
        _rejects(_call(charts=c, nc=len(c)), "charts[%d] and charts[%d] must not overlap" % pair)
    # rectangles that only touch (a shared edge or corner) pass the sweep; the call then stops at the overlapping
    # buffers
    c = np.array([[0, 0, 0, 4, 2, 0, 0, 1], [0, 0, 0, 4, 2, 4, 0, 1], [1, 0, 0, 4, 2, 0, 2, 1],
                  [2, 0, 0, 4, 2, 4, 2, 1], [3, 0, 0, 24, 4, 8, 0, 1]], np.int32)
    _rejects(_call(charts=c, nc=len(c), out=0x10000), "d_outAtlas and d_atlas overlap")
    # accepted edges of the ranges reach the overlap sweep only
    _rejects(_call(out=0x10000), "overlap")


@pytest.mark.parametrize("make", ["topology", "occluder", "coplanar", "single_charts", "atlas", "atlas16",
                                  "deep_strip", "raster_edges", "depth_ratio", "labelling"])
def test_texturing_chart_tables_pass_the_overlap_check(make):
    """Every chart table the texturing oracle writes for texture_cases' inputs passes the chart checks: the call stops
    at its overlapping output buffers instead."""
    c = tc.atlas(16) if make == "atlas16" else getattr(tc, make)()
    r = to.texture(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], **c["kw"])
    ch = np.ascontiguousarray(r["charts"], np.int32)
    rows, width = r["atlas"].shape
    assert len(ch) > 0
    res = _call(charts=ch, nc=len(ch), rows=rows, width=width, out=0x10000)
    msg = cs.lib().cs_last_error().decode()
    assert res == CS_E_ARG and "charts[" not in msg and msg.endswith("overlap"), msg


def _seams_layout(rng):
    V, T, rows = (int(rng.integers(1, 40)) for _ in range(3))
    sizes = {"d_vertices": 12 * V, "d_triangles": 12 * T, "d_faceView": 4 * T, "d_uv": 24 * T,
             "d_atlas": 4 * rows * 32, "d_outAtlas": 4 * rows * 32, "d_cornerOffset": 12 * T}
    outs = {"d_outAtlas", "d_cornerOffset"}

    def make(at):
        g = lambda x: at.get(x)
        return _call(verts=g("d_vertices"), V=V, tris=g("d_triangles"), T=T, view=g("d_faceView"), uv=g("d_uv"),
                     charts=np.zeros((0, 8), np.int32), nc=0, atlas=g("d_atlas"), rows=rows, width=32,
                     out=g("d_outAtlas"), corner=g("d_cornerOffset"))

    return sizes, (lambda a, b: a in outs or b in outs), make


def test_every_overlap_is_rejected_and_named():
    rng = np.random.default_rng(13)
    for _ in range(300):
        sizes, forbidden, make = _seams_layout(rng)
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
    assert "int cs_level_texture_seams(" in hdr
    assert "13 whatever the data" in hdr and "1061 bytes per face" in hdr
    assert isinstance(cs.lib().cs_level_texture_seams, ctypes._CFuncPtr)


# ---- texture.o's kernels are the parent's, instruction for instruction ----
# sha256 of the normalised `cuobjdump -sass` of texture.o's kernels before the edge keys, the adjacency and the
# lower-vertex edge rule moved to trimesh.cuh, from nvcc 12.9 (V12.9.86) with the library's flags.
SASS = {"texture_edges_kernel": "ba956c9310058fa060b0683c3d661aad9445f7acf385375609d0e25b7fc21b9f",
        "texture_adjacency_kernel": "8f726078a9b346a70856d8a4cdb45b550239704a3ef03b88c038ee35535e2ae1",
        "texture_raster_kernel": "d653af2e9debf71e764f5ee318c76de835746ede802289c6068d859d403dabb3",
        "texture_candidate_kernel": "83c146cd81f8a46f45da35300bc6ef6eb16926f1145a5a5b04d276f72de4e947",
        "texture_label_init_kernel": "3efd41d86beb6bc1530c93278541d2ae9833347d977f55f539d5038ada0d8158",
        "texture_colour_kernel": "d6f5141a78da49dbe933145ab0e30c88d60b211b5a9fcb99a0807b49dd103685",
        "texture_energy_kernel": "1257226c137fed944c2443cbe5c0d4f922549c23a9edbedc708df727bc0a9b8f",
        "texture_total_kernel": "98b240333790d9ccdfe2e6584a71858ee292c6cca1938c4e4bce8bece9c61242",
        "texture_icm_kernel": "1b3c0119abbdb6aa185bdd2d597356799dd697faeb523f4a77d038c106d46147",
        "texture_hook_kernel": "f7547a7edf01c61e7e38571a84a8a597981fa46a160206a6123df3b8e99129bd",
        "texture_roots_kernel": "893083e8514ad00327e0c01afed44c256fda6d91d431887b606a44b23bf63978",
        "texture_chart_init_kernel": "91c0e4e2ca12995220b5c58674e6a7548acbaae71fe3c41337d7a741d9865a60",
        "texture_rect_kernel": "6d3625b08bf8ea1b2c34ffb3603e69caa045deced410b25110d83ae56fd98cb5",
        "texture_uv_kernel": "4d1c07eca38d483978dff647d471c6d5206f1a6bdbbf6781235cc4d7818953b2",
        "texture_atlas_kernel": "d4ab6aeef9c12ae741f26bbf07ef894e602b1d5164822c952dff116bd74f0963"}


def test_texture_kernels_are_unchanged():
    nvcc = build.nvcc_path()
    if nvcc is None or "V12.9.86" not in subprocess.run([nvcc, "--version"], stdout=subprocess.PIPE,
                                                        text=True).stdout:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    build.build_library()
    fs = _sass(os.path.join(build.OBJDIR, "texture.o"))
    for name, digest in SASS.items():
        key = [f for f in fs if re.search(r"\d+%sE" % name, f)]
        assert len(key) == 1, (name, sorted(fs))
        assert hashlib.sha256("\n".join(fs[key[0]]).encode()).hexdigest() == digest, name
