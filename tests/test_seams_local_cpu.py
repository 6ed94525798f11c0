"""CPU checks of local seam levelling (tests/seam_local_oracle.py) and of cs_level_texture_seams_local's argument
checks: the analytic ramp across one straight seam, an unchanged constant atlas, the oracle on the scene with a gain,
an offset and a radial falloff per view (A symmetric positive definite, texels past the strip and outside the domain
unchanged, the seam step well below the global call's alone), the sweep that fixed the default tol and checked the
strip width, every CS_E_ARG case with the overlap sweeps, and seams.o's global kernels unchanged by the helpers the
local call now shares with them."""
import ctypes
import hashlib
import math
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.sparse.linalg as spl

import cudasift_b200 as cs
import seam_local_oracle as lo
import seam_oracle as so
import texture_cases as tc
import texture_oracle as to
from cudasift_b200 import build
from test_arg_ranges_cpu import BASE, MSG, _buf, _layout, _share
from test_bundle_intrinsics_cpu import _sass

CS_E_ARG = -2


def vignetted(imgs, seed=1):
    """Every view with its own gain, offset and radial falloff 1 - f r^2 (r = 1 at the image corners)."""
    rng = np.random.default_rng(seed)
    H, W = imgs[0].shape
    yy, xx = np.mgrid[0:H, 0:W]
    r2 = ((xx - W / 2) ** 2 + (yy - H / 2) ** 2) / ((W / 2) ** 2 + (H / 2) ** 2)
    gain, off, fall = (1 + rng.uniform(-0.2, 0.2, len(imgs)), rng.uniform(-20, 20, len(imgs)),
                       rng.uniform(0.1, 0.4, len(imgs)))
    return [np.ascontiguousarray(im * g * (1 - f * r2) + o, np.float32) for im, g, o, f in zip(imgs, gain, off, fall)]


def seam_step(tris, labels, uv, charts, faceChart, img):
    """The mean |I_a - I_b| over seam edges, each side read bilinearly at its uv midpoint."""
    nbr = to.adjacency(tris)
    steps = []
    for f in range(len(tris)):
        for k in range(3):
            g = nbr[f, k]
            if g <= f or labels[f] < 0 or labels[g] < 0 or labels[f] == labels[g]:
                continue
            P, Q = tris[f, k], tris[f, (k + 1) % 3]
            side = []
            for h in (f, g):
                kp, kq = list(tris[h]).index(P), list(tris[h]).index(Q)
                m = 0.5 * (uv[h, kp].astype(np.float64) + uv[h, kq].astype(np.float64))
                side.append(so.bilinear(img, charts[faceChart[h]], m[0], m[1]))
            steps.append(abs(side[0] - side[1]))
    return float(np.mean(steps))


def ramp(c=8, L=40, gap=4):
    """Two charts of constant 100 and 140 meeting along one straight vertical seam of L edges of c texels: a column of
    L quads of label 0 beside one of label 1, every vertex on integer uv, the seam on each chart's outer column."""
    verts = np.array([[i, j, 0.0] for j in range(L + 1) for i in range(3)], np.float32)
    tris = np.array([[3 * j + i, 3 * j + i + 1, 3 * (j + 1) + i + 1] if h == 0 else
                     [3 * j + i, 3 * (j + 1) + i + 1, 3 * (j + 1) + i]
                     for i in range(2) for j in range(L) for h in range(2)], np.int32)
    labels = np.repeat(np.arange(2, dtype=np.int32), 2 * L)
    ox1 = c + 1 + gap
    col, row = tris % 3, tris // 3
    u = np.where(labels[:, None] == 0, col * c, ox1 + (col - 1) * c)
    uv = np.stack([u, row * c], -1).astype(np.float32)
    rows, width = L * c + 1, ox1 + c + 1
    charts = np.array([[0, 0, 0, c + 1, rows, 0, 0, L], [1, 0, 0, c + 1, rows, ox1, 0, L]], np.int32)
    atlas = np.zeros((rows, width), np.float32)
    atlas[:, :c + 1] = 100.0
    atlas[:, ox1:] = 140.0
    return verts, tris, labels, uv, charts, atlas


def test_analytic_ramp():
    c, L, w = 8, 40, 5
    v, t, lab, uv, charts, atlas = ramp(c, L)
    r = lo.level(v, t, lab, uv, charts, atlas, padding=0, stripWidth=w)
    assert r["stats"][7] == 0 and r["stats"][1] == L
    out = r["atlas"]
    ox1 = c + 5
    assert (out[1:, c] == 120).all() and (out[1:, ox1] == 120).all()          # every seam texel (row 0 is missed)
    delta = r["delta"]
    free = r["free"]
    rows = atlas.shape[0]
    far = 3 * (w + 1)
    for yy in range(far, rows - far):
        for d in range(1, w + 1):
            want = 20.0 * (1 - d / (w + 1))
            for x, sign in ((c - d, 1.0), (ox1 + d, -1.0)):
                got = delta[np.searchsorted(free, yy * atlas.shape[1] + x)]
                assert abs(got - sign * want) <= 1e-3 * want, (yy, x, got, want)
    # past the strip: unchanged
    assert (out[:, :c - w] == 100).all() and (out[:, ox1 + w + 1:] == 140).all()


def test_constant_atlas_is_unchanged():
    imgs, Ks, Rs, ts, _ = tc.scene_views()
    v, t = tc.scene_mesh()
    q = to.texture(imgs, Ks, Rs, ts, v, t, lam=0.5)
    atlas = np.full(q["atlas"].shape, 128.0, np.float32)
    r = lo.level(v, t, q["labels"], q["uv"], q["charts"], atlas)
    assert r["stats"][7] == 0 and r["stats"][6] == 0 and r["stats"][3] > 0 and r["stats"][4] > 0
    assert np.array_equal(r["atlas"].view(np.uint32), atlas.view(np.uint32))


@pytest.fixture(scope="module")
def levelled():
    imgs, Ks, Rs, ts, _ = tc.scene_views()
    v, t = tc.scene_mesh()
    q = to.texture(vignetted(imgs), Ks, Rs, ts, v, t, lam=0.5)
    g = so.level(v, t, q["labels"], q["uv"], q["charts"], q["atlas"])
    return v, t, q, g


def test_scene_oracle(levelled):
    v, t, q, g = levelled
    w = 20
    r = lo.level(v, t, q["labels"], q["uv"], q["charts"], g["atlas"], stripWidth=w)
    A = r["A"]
    assert abs(A - A.T).max() == 0
    lmin = spl.eigsh(A, k=1, sigma=0, which="LM", return_eigenvectors=False)[0]
    assert lmin > 0
    # texels past the strip and outside the domain are copied; the domain is the global call's texel set
    d = r["d"]
    keep = (d < 0) | (d > w)
    assert np.array_equal(r["atlas"].reshape(-1)[keep].view(np.uint32), g["atlas"].reshape(-1)[keep].view(np.uint32))
    assert r["stats"][5] == g["stats"][6]
    fc = r["faceChart"]
    before = seam_step(t, q["labels"], q["uv"], q["charts"], fc, q["atlas"])
    glob = seam_step(t, q["labels"], q["uv"], q["charts"], fc, g["atlas"])
    loc = seam_step(t, q["labels"], q["uv"], q["charts"], fc, r["atlas"])
    print("stats %s, lambda_min %.3g; mean seam step %.2f, global %.2f, global + local %.2f (ratio %.3f)"
          % (r["stats"], lmin, before, glob, loc, loc / glob))
    # on this scene: 18.35 before, 2.19 after the global call, 1.00 after the local call too (ratio 0.46)
    assert loc <= 0.5 * glob


def test_sweep_of_strip_width_and_tol(levelled):
    """CG iterations and max |delta - delta*| (grey levels) against stripWidth and tol on the scene.  At the default
    tol 1e-4 the error stays below 0.1 grey level for every strip width up to 40, and at the default stripWidth 20 the
    CG count is 84; tol 1e-3 leaves up to 0.44."""
    v, t, q, g = levelled
    rows = {}
    for w in (5, 10, 20, 40):
        r = lo.level(v, t, q["labels"], q["uv"], q["charts"], g["atlas"], stripWidth=w)
        for tol in (1e-3, 1e-4, 1e-5):
            x, its, conv = lo.pcg(r["A"], r["b"], tol, 1000)
            rows[(w, tol)] = (its, float(np.abs(x - r["delta"]).max()))
            print("stripWidth %-3d tol %-6g iterations %-4d max error %.4f" % (w, tol, *rows[(w, tol)]))
    assert all(rows[(w, 1e-4)][1] < 0.1 for w in (5, 10, 20, 40))
    assert rows[(5, 1e-4)][0] < rows[(20, 1e-4)][0] < rows[(40, 1e-4)][0] < 1000


# ---- library --------------------------------------------------------------------------------------------------------
CHARTS = np.array([[0, 0, 0, 10, 4, 0, 0, 3], [1, 0, 0, 12, 3, 10, 0, 2]], np.int32)


def _call(verts=0x1000, V=4, tris=0x2000, T=4, view=0x3000, uv=0x4000, charts=CHARTS, nc=2, atlas=0x10000, rows=4,
          width=32, pad=2, strip=20, its=1000, tol=1e-4, out=0x20000):
    p = charts.ctypes.data_as(ctypes.c_void_p) if charts is not None else None
    return cs.lib().cs_level_texture_seams_local(verts, V, tris, T, view, uv, p, nc, atlas, rows, width, pad, strip,
                                                 its, tol, out, None, None, None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    assert msg.startswith("cs_level_texture_seams_local: invalid argument (CS_E_ARG)"), msg
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
    for strip in (0, -1, 129):
        _rejects(_call(strip=strip), "stripWidth")
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
    _rejects(_call(atlas=None), "d_atlas")
    _rejects(_call(atlas=0x10001), "d_atlas")
    _rejects(_call(out=None), "d_outAtlas")
    _rejects(_call(out=0x20002), "d_outAtlas")
    for rects, pair in (([(0, 0, 20, 4), (5, 1, 3, 2)], (0, 1)),
                        ([(0, 0, 10, 4), (9, 3, 5, 1)], (0, 1)),
                        ([(2, 0, 6, 2), (0, 2, 3, 2), (0, 1, 3, 1)], (0, 2))):
        c = np.array([[l, 0, 0, w, h, ox, oy, 1] for l, (ox, oy, w, h) in enumerate(rects)], np.int32)
        _rejects(_call(charts=c, nc=len(c)), "charts[%d] and charts[%d] must not overlap" % pair)
    _rejects(_call(out=0x10000), "d_outAtlas and d_atlas overlap")


@pytest.mark.parametrize("make", ["topology", "occluder", "coplanar", "single_charts", "atlas", "atlas16",
                                  "deep_strip", "raster_edges", "depth_ratio", "labelling"])
def test_texturing_chart_tables_pass_the_overlap_check(make):
    c = tc.atlas(16) if make == "atlas16" else getattr(tc, make)()
    r = to.texture(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], **c["kw"])
    ch = np.ascontiguousarray(r["charts"], np.int32)
    rows, width = r["atlas"].shape
    assert len(ch) > 0
    res = _call(charts=ch, nc=len(ch), rows=rows, width=width, out=0x10000)
    msg = cs.lib().cs_last_error().decode()
    assert res == CS_E_ARG and "charts[" not in msg and msg.endswith("overlap"), msg


def test_every_overlap_is_rejected_and_named():
    rng = np.random.default_rng(17)
    for _ in range(300):
        V, T, rows = (int(rng.integers(1, 40)) for _ in range(3))
        sizes = {"d_vertices": 12 * V, "d_triangles": 12 * T, "d_faceView": 4 * T, "d_uv": 24 * T,
                 "d_atlas": 4 * rows * 32, "d_outAtlas": 4 * rows * 32}
        forbidden = lambda a, b: "d_outAtlas" in (a, b)
        at = _layout(rng, sizes, forbidden)
        g = lambda x: BASE + at[x]
        r = _call(verts=g("d_vertices"), V=V, tris=g("d_triangles"), T=T, view=g("d_faceView"), uv=g("d_uv"),
                  charts=np.zeros((0, 8), np.int32), nc=0, atlas=g("d_atlas"), rows=rows, out=g("d_outAtlas"))
        msg = cs.lib().cs_last_error().decode()
        assert r == CS_E_ARG, (r, msg)
        m = MSG.match(msg)
        assert m, msg
        _, a, b = m.groups()
        assert forbidden(a, b) and _share((at[a], sizes[a]), (at[b], sizes[b])), (msg, at, sizes)
    assert not _buf.any()


def test_header_declares_the_call():
    hdr = open(os.path.join(os.path.dirname(cs.__file__), "..", "include", "cudasift_b200.h")).read()
    assert "int cs_level_texture_seams_local(" in hdr
    assert "15 + stripWidth whatever the data" in hdr and "244 bytes per face" in hdr
    assert isinstance(cs.lib().cs_level_texture_seams_local, ctypes._CFuncPtr)


# ---- seams.o's global kernels are the parent's, instruction for instruction ----
# sha256 of the normalised `cuobjdump -sass` of cs_level_texture_seams's kernels before the sample sides and the chart
# row index were shared with the local call, from nvcc 12.9 (V12.9.86) with the library's flags.
SASS = {"seams_check_kernel": "51de83e04c1f8988db168a1dd12d8f314cd05cf591b9b60efe06ba9f6f4e53ac",
        "seams_keys_kernel": "96247572adaca70cdb6fce804bc784de44e5ad6d9c4978ee9f8a3a3b38843e43",
        "seams_adjacency_kernel": "dfa450138b376d12e5f7362996a9699610ffc4b5bf6ea758fef181fe4705f3c0",
        "seams_unknown_kernel": "1c38dfd240cdb9de5cef2eeec8c4d3a48164300062218fd6c368dd496d95d562",
        "seams_smooth_keys_kernel": "a0789d219782c67b99a1fc457929f94598a4fc5ba6f0b5182b5d29cd90302b4a",
        "seams_smooth_heads_kernel": "6b86793302c2b9d154cb45218be6726e62e1d27ada00f547ffd28f4798ef58d9",
        "seams_sample_kernel": "13d0c2826ec1307fba6aa4d4e2236f4b956a9dbe01a194af4838dbb68ce4f17a",
        "seams_row_heads_kernel": "c701875fcfbc85d25daf63ee11a6c8dbba7314470a84d92d8beab4d79f64f20e",
        "seams_rows_kernel": "eddb0390be27d9fd55c6923c4349368e2d425f9511cdb0e15d9a3bc3aaef6671",
        "seams_solve_kernel": "498604ad394ff2430d931fb791f7bed585446c6225df467eaae6bb46091a3f31",
        "seams_raster_kernel": "61f3e014d8d87bfc593bf7dd348ff0e77115af429719ebe546c20c6bdfbe8f8f",
        "seams_texel_kernel": "91db7861df10a23d92d559cfa63e4de9f60114261ee6cd5e988d040690798ec9"}


def test_global_seam_kernels_are_unchanged():
    nvcc = build.nvcc_path()
    if nvcc is None or "V12.9.86" not in subprocess.run([nvcc, "--version"], stdout=subprocess.PIPE,
                                                        text=True).stdout:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    build.build_library()
    fs = _sass(os.path.join(build.OBJDIR, "seams.o"))
    for name, digest in SASS.items():
        key = [f for f in fs if re.search(r"\d+%sE" % name, f)]
        assert len(key) == 1, (name, sorted(fs))
        assert hashlib.sha256("\n".join(fs[key[0]]).encode()).hexdigest() == digest, name
