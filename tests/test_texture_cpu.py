"""CPU checks of the texturing rules (tests/texture_oracle.py) and of cs_texture_mesh's argument checks: depth buffers
without holes on shared edges and in agreement with the scene's true depth, proper colourings with at most 4 colours,
an energy that never increases, packed charts that neither overlap nor leave the atlas, charts that are exact copies of
their images, and every CS_E_ARG case, overlaps included."""
import ctypes
import math
import os

import numpy as np
import pytest

import cudasift_b200 as cs
import simplify_cases as scs
import texture_cases as tc
import texture_oracle as to
from test_arg_ranges_cpu import BASE, MSG, _buf, _layout, _share

CS_E_ARG = -2


@pytest.fixture(scope="module")
def scene():
    imgs, Ks, Rs, ts, views = tc.scene_views()
    v, t = tc.scene_mesh()
    r = to.texture(imgs, Ks, Rs, ts, v, t, lam=0.5)
    return imgs, Ks, Rs, ts, views, v, t, r


@pytest.mark.parametrize("jitter", [0.0, 0.3])
def test_depth_buffer_has_no_hole_on_shared_edges(jitter):
    v, t, K, R, tt, W, H, (x0, x1, y0, y1) = tc.flat_grid(jitter=jitter)
    buf = to.depth_buffer(K, R, tt, W, H, v, t)
    cov = buf != to.EMPTY
    inside = np.zeros_like(cov)
    inside[y0:y1 + 1, x0:x1 + 1] = True
    assert (cov == inside).all(), (int((inside & ~cov).sum()), int((cov & ~inside).sum()))
    d = (buf[cov] >> np.uint64(32)).astype(np.uint32).view(np.float32)
    assert (d == np.float32(5.0)).all()


def test_depth_buffer_agrees_with_the_true_depth(scene):
    imgs, Ks, Rs, ts, views, v, t, r = scene
    share = []
    for a, buf in enumerate(r["bufs"]):
        cov = buf != to.EMPTY
        d = (buf[cov] >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
        true = views[a][1][cov]
        share.append(np.mean(np.abs(d - true) <= 1e-5 * true))
        assert cov.mean() > 0.5
    print("share of covered pixels within 1e-5 of the true depth: %s" % np.round(share, 4))
    assert min(share) >= 0.98         # the rest lie on silhouettes and where the box meets the ground


@pytest.mark.parametrize("case", ["scene", "sphere", "torus", "scene_jittered"])
def test_colouring_is_proper(case):
    if case.startswith("scene"):
        v, t = tc.scene_mesh(jitter=0.3 if case.endswith("jittered") else 0.0)
    elif case == "sphere":
        v, t = scs.sphere_mesh(16, 5.3)[:2]
    else:
        v, t = scs.torus_mesh(16, 4.6, 1.9)[:2]
    nbr = to.adjacency(t)
    col, rounds = to.colouring(nbr)
    assert (col >= 0).all() and col.max() <= 3
    for k in range(3):
        g = nbr[:, k]
        ok = g >= 0
        assert (col[ok] != col[g[ok]]).all()
    if case in ("sphere", "torus"):
        assert (nbr >= 0).all()


@pytest.mark.parametrize("lam", [0.5, 5.0])
def test_energy_never_increases(scene, lam):
    imgs, Ks, Rs, ts, _, v, t, r = scene
    for jitter in (0.0, 0.3):
        vv, tt = tc.scene_mesh(jitter=jitter)
        q = to.texture(imgs, Ks, Rs, ts, vv, tt, lam=lam)
        assert q["stats"][10] == 0 and q["info"][1] <= q["info"][0], q["info"]


def test_lambda_zero_keeps_the_best_candidate(scene):
    imgs, Ks, Rs, ts, _, v, t, r = scene
    q = to.texture(imgs, Ks, Rs, ts, v, t, lam=0.0, bufs=r["bufs"])
    assert np.array_equal(q["labels"], q["start"]) and q["stats"][6] == 0 and q["stats"][5] == 1


def test_packing_has_no_overlap_and_stays_inside(scene):
    imgs, Ks, Rs, ts, _, v, t, r = scene
    for width in (160, 300, 1024):
        q = to.texture(imgs, Ks, Rs, ts, v, t, lam=0.5, atlasWidth=width, bufs=r["bufs"])
        ch = q["charts"]
        used = np.zeros((q["stats"][8], width), np.int32)
        for e in ch:
            assert 0 <= e[5] and e[5] + e[3] <= width and 0 <= e[6] and e[6] + e[4] <= q["stats"][8]
            used[e[6]:e[6] + e[4], e[5]:e[5] + e[3]] += 1
        assert used.max() == 1 and ch[:, 7].sum() == len(t) - q["stats"][1]


def test_charts_are_copies_of_their_images(scene):
    imgs, Ks, Rs, ts, _, v, t, r = scene
    atlas = r["atlas"]
    covered = np.zeros(atlas.shape, bool)
    for a, x0, y0, w, h, ox, oy, _ in r["charts"]:
        assert np.array_equal(atlas[oy:oy + h, ox:ox + w], imgs[a][y0:y0 + h, x0:x0 + w])
        covered[oy:oy + h, ox:ox + w] = True
    assert (atlas[~covered] == 0).all()
    # every seen corner's coordinate lies in its chart's rectangle, padding inside
    for f in np.nonzero(r["labels"] >= 0)[0]:
        e = r["charts"][r["faceChart"][f]]
        x, y = r["uv"][f, :, 0], r["uv"][f, :, 1]
        assert (x >= e[5]).all() and (x <= e[5] + e[3] - 1).all() and (y >= e[6]).all() and (y <= e[6] + e[4] - 1).all()


def test_invalid_inputs(scene):
    imgs, Ks, Rs, ts, _, v, t, _ = scene
    bad = t.copy()
    bad[0, 0] = len(v)
    assert to.texture(imgs, Ks, Rs, ts, v, bad)["stats"][10] == 2
    bad = t.copy()
    bad[0, 1] = bad[0, 2]
    assert to.texture(imgs, Ks, Rs, ts, v, bad)["stats"][10] == 2


def test_energy_total_order():
    """The three-level total depends on the item count alone; it equals the exact sum for integers."""
    for n in (1, 5, 2048, 2049, 300000):
        e = np.arange(n, dtype=np.float64) % 7
        assert to.tree_total(e) == float(e.sum())


# ---- library --------------------------------------------------------------------------------------------------------
K = np.array([[100.0, 0, 80], [0, 100, 60], [0, 0, 1]])
R = np.eye(3)
T0 = np.zeros(3)
IMG = (cs.StereoImage * 2)(cs.StereoImage(0x100000, 160, 120, 160), cs.StereoImage(0x200000, 200, 100, 200))
KS, RS, TS = np.stack([K, K]), np.stack([R, R]), np.stack([T0, T0])


def _call(images=IMG, n=2, Ks=KS, Rs=RS, ts=TS, verts=0x1000, V=4, tris=0x2000, T=4, lam=0.5, angle=75.0, tol=0.01,
          pad=2, width=1024, sweeps=100, atlas=0x400000, rows=4, uv=0x10000, view=0x20000, chart=None,
          charts=np.zeros((4, 8), np.int32), nc=4):
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p) if a is not None else None
    return cs.lib().cs_texture_mesh(images, n, p(Ks), p(Rs), p(ts), verts, V, tris, T, lam, angle, tol, pad, width,
                                    sweeps, atlas, rows, uv, view, chart, p(charts), nc, None, None, None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    assert msg.startswith("cs_texture_mesh: invalid argument (CS_E_ARG)"), msg
    for w in words:
        assert w in msg, (w, msg)


def test_argument_checks():
    _rejects(_call(n=0), "numImages")
    _rejects(_call(images=None), "images")
    _rejects(_call(Ks=np.stack([K, K * 0])), "Ks[1]")
    _rejects(_call(Rs=np.stack([R, 2 * R])), "Rs[1]")
    _rejects(_call(ts=np.stack([T0, T0 + np.inf])), "ts[1]")
    bad = (cs.StereoImage * 2)(cs.StereoImage(0x100002, 160, 120, 160), IMG[1])
    _rejects(_call(images=bad), "images[0].d_img")
    bad = (cs.StereoImage * 2)(IMG[0], cs.StereoImage(0x200000, 200, 100, 199))
    _rejects(_call(images=bad), "pitch")
    _rejects(_call(V=-1), "numVertices")
    _rejects(_call(V=(1 << 30) + 1), "numVertices")
    _rejects(_call(T=-1), "numTriangles")
    _rejects(_call(T=(1 << 29) + 1), "numTriangles")
    for lam in (-0.1, math.inf, math.nan):
        _rejects(_call(lam=lam), "lambda")
    for angle in (0.0, -1.0, 90.5, math.nan):
        _rejects(_call(angle=angle), "maxViewAngleDeg")
    for tol in (-0.01, 1.5, math.nan, math.inf):
        _rejects(_call(tol=tol), "depthTol")
    for pad in (-1, 17):
        _rejects(_call(pad=pad), "padding")
    for width in (199, 32769):
        _rejects(_call(width=width), "atlasWidth", "200")
    for sweeps in (-1, 1001):
        _rejects(_call(sweeps=sweeps), "maxSweeps")
    _rejects(_call(rows=-1), "maxAtlasRows")
    _rejects(_call(nc=-1), "maxCharts")
    _rejects(_call(verts=None), "d_vertices")
    _rejects(_call(verts=0x1002), "d_vertices")
    _rejects(_call(tris=None), "d_triangles")
    _rejects(_call(tris=0x2001), "d_triangles")
    _rejects(_call(uv=None), "d_uv")
    _rejects(_call(uv=0x10002), "d_uv")
    _rejects(_call(view=None), "d_faceView")
    _rejects(_call(view=0x20001), "d_faceView")
    _rejects(_call(chart=0x30001), "d_faceChart")
    _rejects(_call(atlas=None), "d_atlas")
    _rejects(_call(atlas=0x400002), "d_atlas")
    _rejects(_call(charts=None), "charts_out")
    # accepted edges of the ranges reach the overlap sweep only
    _rejects(_call(uv=0x1000), "overlap")


def test_empty_mesh_makes_no_cuda_call():
    stats = np.full(11, -1, np.int64)
    info = np.full(2, -1.0)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    r = cs.lib().cs_texture_mesh(IMG, 2, p(KS), p(RS), p(TS), None, 0, None, 0, 0.5, 75.0, 0.01, 2, 1024, 100, None,
                                 0, None, None, None, None, 0, p(info), p(stats), None)
    assert r == 0 and (stats == 0).all() and (info == 0).all()


def _texture_layout(rng):
    V, T, rows = (int(rng.integers(1, 40)) for _ in range(3))
    with_chart = bool(rng.integers(0, 2))
    sizes = {"d_vertices": 12 * V, "d_triangles": 12 * T, "d_atlas": 4 * rows * 256, "d_uv": 24 * T,
             "d_faceView": 4 * T, "images[0].d_img": 4 * (3 * 16 + 10), "images[1].d_img": 4 * (2 * 12 + 12)}
    if with_chart:
        sizes["d_faceChart"] = 4 * T
    outs = {"d_atlas", "d_uv", "d_faceView", "d_faceChart"}
    Ks, Rs, ts = np.stack([K, K]), np.stack([R, R]), np.stack([T0, T0])

    def make(at):
        imgs = (cs.StereoImage * 2)(cs.StereoImage(at["images[0].d_img"], 10, 4, 16),
                                    cs.StereoImage(at["images[1].d_img"], 12, 3, 12))
        g = lambda x: at.get(x)
        return _call(images=imgs, Ks=Ks, Rs=Rs, ts=ts, verts=g("d_vertices"), V=V, tris=g("d_triangles"), T=T,
                     width=256, atlas=g("d_atlas"), rows=rows, uv=g("d_uv"), view=g("d_faceView"),
                     chart=g("d_faceChart"))

    return sizes, (lambda a, b: a in outs or b in outs), make


def test_every_overlap_is_rejected_and_named():
    rng = np.random.default_rng(12)
    for _ in range(300):
        sizes, forbidden, make = _texture_layout(rng)
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
    assert "int cs_texture_mesh(" in hdr
    assert "14 + 2 G + rounds + colours x sweeps" in hdr and "272 bytes per face" in hdr
    assert isinstance(cs.lib().cs_texture_mesh, ctypes._CFuncPtr)
    assert cs.lib().cs_set_tuning(b"texture_group_bytes", 0) == 0


def test_save_textured_obj(scene, tmp_path):
    """OBJ + MTL + PNG: a valid 8-bit grey PNG of the atlas, one vt per corner of every seen face, unseen faces without
    texture coordinates."""
    import struct
    import zlib
    imgs, Ks, Rs, ts, _, v, t, r = scene
    objp, mtlp, pngp = cs.save_textured_obj(str(tmp_path / "scene.obj"), v, t, r["uv"], r["atlas"])
    data = open(pngp, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    W, H, depth, kind = struct.unpack(">IIBB", data[16:26])
    n = struct.unpack(">I", data[33:37])[0]
    raw = np.frombuffer(zlib.decompress(data[41:41 + n]), np.uint8).reshape(H, W + 1)
    assert (W, H, depth, kind) == (r["atlas"].shape[1], r["atlas"].shape[0], 8, 0)
    assert np.array_equal(raw[:, 1:], np.clip(np.rint(r["atlas"]), 0, 255).astype(np.uint8))
    lines = open(objp).read().splitlines()
    seen = int((r["labels"] >= 0).sum())
    assert sum(x.startswith("vt ") for x in lines) == 3 * seen
    faces = [x for x in lines if x.startswith("f ")]
    assert len(faces) == len(t) and sum("/" in x for x in faces) == seen
    assert "map_Kd scene.png" in open(mtlp).read()
