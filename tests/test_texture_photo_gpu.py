"""GPU checks of cs_texture_mesh_photo (TextureMeshPhoto) against tests/texture_photo_oracle.py: every output (labels,
charts, texture coordinates, atlas, info, stats [16]) bit-equal to the oracle on the scene mesh (jitter 0 and 0.3,
lambda 0, 0.5 and 5), on a PoissonMesh -> SimplifyMesh sphere and on every case of tests/texture_photo_cases.py, with
both data terms and the outlier test on and off; with both off, cs_texture_mesh's outputs with one more launch; image
groups of 3, 2 and 1 images and the launch count; truncation prefixes and statuses; pitched images; and the two effects
the view selection is for: a transient occluder painted into one view stops texturing the faces it covers, and a
blurred view loses faces to sharp ones under GMI."""
import ctypes

import numpy as np
import pytest

import cudasift_b200 as cs
import mesh_cases as mc
import texture_cases as tc
import texture_photo_cases as pc
import texture_oracle as to
import texture_photo_oracle as tpo
from cudasift_b200 import synth
from test_dense_pitch_gpu import _pitched_upload, _same

pytestmark = pytest.mark.gpu

ATLAS_WIDTH = 1024
SETTINGS = {"area": dict(dataTerm=0, outlierK=0.0), "gmi": dict(dataTerm=1, outlierK=0.0),
            "area_outliers": dict(dataTerm=0), "gmi_outliers": dict(dataTerm=1)}
# Transient occluder: of the faces whose corners all lie inside the painted rectangle and whose label was the painted
# view, the share that no longer take it with outlier rejection, and the mean |atlas - clean view| over those faces'
# centroids against TextureMesh's.  Blurred view: the faces the blurred view labels under GMI over those under the
# area term, and the mean Sobel magnitude of the chart texels under GMI over that under the area term.  Measured on an
# H100 80GB HBM3 (the outputs are the oracle's bit for bit, so these are exact): 16 of 17 faces moved (0.941), error
# 99.4 -> 6.15 grey levels (ratio 0.062); the blurred view labels 105 faces under the area term and 39 under GMI (ratio
# 0.371), chart sharpness 4.219 -> 4.275 (gain 1.013, so the bound only asks that it rises).
OCCLUDER_MOVED = 0.8
OCCLUDER_ERROR_RATIO = 0.25
BLUR_LABEL_RATIO = 0.6
BLUR_SHARPNESS_GAIN = 1.0


def run(c, maxRows=None, maxCharts=None, cap=None, upload=None, **photo):
    """cs_texture_mesh_photo on a case (texture_cases' dict; photo overrides its kw) with every output, maxRows atlas
    rows (None: the oracle's full height) and maxCharts chart rows (None: one per face); cap the texture_group_bytes.
    Returns the outputs as the oracle names them, and the launches counted."""
    kw = dict(lam=0.5, maxViewAngleDeg=75.0, depthTol=0.01, padding=2, atlasWidth=ATLAS_WIDTH, maxSweeps=100,
              dataTerm=1, outlierK=3.0, outlierMinSigma=4.0) | c["kw"] | photo
    v, t, imgs = c["v"], c["t"], c["imgs"]
    T, W = len(t), kw["atlasWidth"]
    maxRows = 4096 if maxRows is None else maxRows
    arrs, bufs, table = (upload or cs._upload_images)(imgs)
    K, R, tt = (np.ascontiguousarray(np.asarray(a, np.float64)) for a in (c["Ks"], c["Rs"], c["ts"]))
    if maxCharts is None:
        maxCharts = max(T, 1)
    try:
        ins = [cs.DeviceBuffer(max(v.nbytes, 4)), cs.DeviceBuffer(max(t.nbytes, 4))]
        outs = [cs.DeviceBuffer(4 * max(maxRows, 1) * W), cs.DeviceBuffer(24 * T), cs.DeviceBuffer(4 * T),
                cs.DeviceBuffer(4 * T)]
        bufs += ins + outs
        ins[0].upload(np.ascontiguousarray(v, np.float32))
        ins[1].upload(np.ascontiguousarray(t, np.int32))
        charts = np.full((max(maxCharts, 1), 8), -7, np.int32)
        info, stats = np.full(2, -1.0), np.full(16, -1, np.int64)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        if cap is not None:
            assert cs.lib().cs_set_tuning(b"texture_group_bytes", cap) == 0
        try:
            before = cs.lib().cs_launch_count()
            C = cs.lib().cs_texture_mesh_photo(table, len(imgs), p(K), p(R), p(tt), ins[0].ptr, len(v), ins[1].ptr, T,
                                               kw["dataTerm"], kw["outlierK"], kw["outlierMinSigma"], kw["lam"],
                                               kw["maxViewAngleDeg"], kw["depthTol"], kw["padding"], W,
                                               kw["maxSweeps"], outs[0].ptr if maxRows else None, maxRows,
                                               outs[1].ptr, outs[2].ptr, outs[3].ptr, p(charts) if maxCharts else None,
                                               maxCharts, p(info), p(stats), None)
            launches = cs.lib().cs_launch_count() - before
        finally:
            if cap is not None:
                cs.lib().cs_set_tuning(b"texture_group_bytes", 0)
        assert C >= 0, cs.lib().cs_last_error()
        rows = int(min(stats[9], maxRows))
        return dict(ret=C, stats=[int(x) for x in stats], info=info, charts=charts,
                    atlas=outs[0].download(np.float32, rows * W).reshape(rows, W),
                    uv=outs[1].download(np.float32, 6 * T).reshape(T, 3, 2), labels=outs[2].download(np.int32, T),
                    faceChart=outs[3].download(np.int32, T)), launches
    finally:
        for b in bufs:
            b.free()


def oracle(c, **photo):
    kw = dict(atlasWidth=ATLAS_WIDTH) | c["kw"] | photo
    return tpo.texture_photo(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], **kw)


def compare(got, ref, launches=None, groups=1):
    st = ref["stats"]
    assert got["stats"] == st, (got["stats"], st)
    assert got["ret"] == ref["ret"]
    assert np.array_equal(np.asarray(got["info"]).view(np.uint64), np.asarray(ref["info"], np.float64).view(np.uint64))
    assert np.array_equal(got["labels"], ref["labels"])
    assert np.array_equal(got["faceChart"], ref["faceChart"])
    C = ref["ret"]
    assert np.array_equal(got["charts"][:C], ref["charts"]) and (got["charts"][C:] == -7).all()
    assert np.array_equal(got["atlas"].view(np.uint32), ref["atlas"].view(np.uint32))
    assert np.array_equal(got["uv"].view(np.uint32), ref["uv"].view(np.uint32))
    if launches is not None:
        assert launches == 15 + 2 * groups + st[4] + st[3] * st[5], (launches, groups, st)


def _scene_case(jitter, lam):
    imgs, Ks, Rs, ts, _ = tc.scene_views()
    v, t = tc.scene_mesh(jitter=jitter)
    return tc._case(imgs, Ks, Rs, ts, v, t, lam=lam)


@pytest.mark.parametrize("setting", sorted(SETTINGS))
@pytest.mark.parametrize("jitter", [0.0, 0.3])
@pytest.mark.parametrize("lam", [0.0, 0.5, 5.0])
def test_oracle_equality_scene(lam, jitter, setting):
    c = _scene_case(jitter, lam)
    ref = oracle(c, **SETTINGS[setting])
    got, launches = run(c, **SETTINGS[setting])
    print("scene lambda %g jitter %g %s: stats %s" % (lam, jitter, setting, got["stats"]))
    compare(got, ref, launches)


@pytest.fixture(scope="module")
def sphere():
    x, n = mc.sphere(20000)
    v, t, _, _, _, _, _ = cs.PoissonMesh(x, n, depth=5)
    gv, gt, _, _, _, _ = cs.SimplifyMesh(v, t, targetTriangles=len(t) // 4)
    Ks, Rs, ts = tc.ring_cameras(8, 160, 120, mc.CENTRE, 3.0)
    imgs = [synth.synth_image(160, 120, seed=50 + a).astype(np.float32) for a in range(8)]
    return tc._case(imgs, Ks, Rs, ts, gv, gt, lam=0.5)


@pytest.mark.parametrize("setting", sorted(SETTINGS))
def test_oracle_equality_sphere(sphere, setting):
    ref = oracle(sphere, **SETTINGS[setting])
    got, launches = run(sphere, **SETTINGS[setting])
    print("sphere %s: %d faces, stats %s" % (setting, len(sphere["t"]), got["stats"]))
    compare(got, ref, launches)


_cases = {}


def _rule_case(name):
    if name not in _cases:
        _cases[name] = pc.CASES[name]()
    return _cases[name]


@pytest.mark.parametrize("setting", sorted(SETTINGS))
@pytest.mark.parametrize("name", sorted(pc.CASES))
def test_rules(name, setting):
    c = _rule_case(name)
    ref = oracle(c, **SETTINGS[setting])
    got, launches = run(c, **SETTINGS[setting])
    print("%s %s: stats %s" % (name, setting, got["stats"]))
    compare(got, ref, launches)


def _texture_mesh_raw(c, maxRows):
    """cs_texture_mesh on the same arguments (the parent call), with its launches."""
    kw = dict(lam=0.5) | c["kw"]
    v, t, imgs = c["v"], c["t"], c["imgs"]
    T = len(t)
    arrs, bufs, table = cs._upload_images(imgs)
    K, R, tt = (np.ascontiguousarray(np.asarray(a, np.float64)) for a in (c["Ks"], c["Rs"], c["ts"]))
    try:
        ins = [cs.DeviceBuffer(max(v.nbytes, 4)), cs.DeviceBuffer(max(t.nbytes, 4))]
        outs = [cs.DeviceBuffer(4 * maxRows * ATLAS_WIDTH), cs.DeviceBuffer(24 * T), cs.DeviceBuffer(4 * T),
                cs.DeviceBuffer(4 * T)]
        bufs += ins + outs
        ins[0].upload(np.ascontiguousarray(v, np.float32))
        ins[1].upload(np.ascontiguousarray(t, np.int32))
        charts = np.full((T, 8), -7, np.int32)
        info, stats = np.full(2, -1.0), np.full(11, -1, np.int64)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        before = cs.lib().cs_launch_count()
        C = cs.lib().cs_texture_mesh(table, len(imgs), p(K), p(R), p(tt), ins[0].ptr, len(v), ins[1].ptr, T,
                                     kw["lam"], 75.0, 0.01, 2, ATLAS_WIDTH, 100, outs[0].ptr, maxRows, outs[1].ptr,
                                     outs[2].ptr, outs[3].ptr, p(charts), T, p(info), p(stats), None)
        launches = cs.lib().cs_launch_count() - before
        rows = int(min(stats[9], maxRows))
        return dict(ret=C, stats=[int(x) for x in stats], info=info, charts=charts,
                    atlas=outs[0].download(np.float32, rows * ATLAS_WIDTH).reshape(rows, ATLAS_WIDTH),
                    uv=outs[1].download(np.float32, 6 * T).reshape(T, 3, 2), labels=outs[2].download(np.int32, T),
                    faceChart=outs[3].download(np.int32, T)), launches
    finally:
        for b in bufs:
            b.free()


@pytest.mark.parametrize("which", ["scene", "sphere", "occluded", "capped"])
def test_both_off_is_texture_mesh(which, sphere):
    c = {"scene": lambda: _scene_case(0.3, 0.5), "sphere": lambda: sphere}.get(which, lambda: _rule_case(which))()
    a, la = _texture_mesh_raw(c, 4096)
    b, lb = run(c, dataTerm=0, outlierK=0.0)
    assert b["stats"][:11] == a["stats"] and b["stats"][13:] == [0, 0, 0] and lb == la + 1
    for k in ("ret", "info", "charts", "atlas", "uv", "labels", "faceChart"):
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def test_groups(sphere):
    a, _ = run(sphere)
    counts = []
    for per, groups in ((3, 3), (2, 4), (1, 8)):
        g, launches = run(sphere, cap=per * 160 * 120 * 8)
        for k in ("ret", "stats", "info", "charts", "atlas", "uv", "labels", "faceChart"):
            assert np.asarray(a[k]).tobytes() == np.asarray(g[k]).tobytes(), (per, k)
        st = g["stats"]
        assert launches == 15 + 2 * groups + st[4] + st[3] * st[5], (launches, groups, st)
        counts.append(launches)
    assert counts[2] - counts[1] == 8 and counts[1] - counts[0] == 2


def test_truncation_prefixes():
    c = _scene_case(0.3, 0.5)
    ref = oracle(c)
    C, full = ref["ret"], ref["stats"][8]
    for rows, nc in ((full // 3, C // 2), (0, 0), (full + 5, C + 3), (1, 1)):
        g, _ = run(c, maxRows=rows, maxCharts=nc)
        assert g["ret"] == C and g["stats"][9] == min(rows, full)
        assert g["stats"][:9] == ref["stats"][:9] and g["stats"][10:] == ref["stats"][10:]
        assert np.array_equal(g["atlas"], ref["atlas"][:rows])
        assert np.array_equal(g["charts"][:min(nc, C)], ref["charts"][:nc])
        assert (g["charts"][min(nc, C):] == -7).all()
        assert np.array_equal(g["uv"].view(np.uint32), ref["uv"].view(np.uint32))
        assert np.array_equal(g["faceChart"], ref["faceChart"])


def test_statuses_and_launches():
    c = _scene_case(0.0, 0.5)
    g, launches = run(c)
    st = g["stats"]
    assert st[10] == 0 and launches == 15 + 2 + st[4] + st[3] * st[5]
    c5 = _scene_case(0.0, 5.0)
    g3, _ = run(c5, maxSweeps=1)
    ref = oracle(c5, maxSweeps=1)
    assert g3["stats"][10] == 3 == ref["stats"][10] and g3["stats"][5] == 1 and g3["stats"] == ref["stats"]
    assert np.array_equal(g3["labels"], ref["labels"])
    g0, _ = run(c, maxSweeps=0)
    assert g0["stats"][10] == 3 and g0["stats"][5] == 0
    assert np.array_equal(g0["labels"], oracle(c, maxSweeps=0)["start"].astype(np.int32))
    bad = dict(c, t=c["t"].copy())
    bad["t"][3, 2] = bad["t"][3, 0]
    g2, launches = run(bad)
    assert g2["ret"] == 0 and g2["stats"][10] == 2 and launches == 1 and g2["stats"][11:] == [0] * 5
    assert (g2["charts"] == -7).all()
    nan = dict(c, v=c["v"].copy())
    nan["v"][c["t"][7, 1], 0] = np.nan
    assert run(nan)[0]["stats"][10] == 2


def test_pitched_images(monkeypatch):
    c = _scene_case(0.3, 0.5)
    for setting in ("gmi_outliers", "area_outliers"):
        dense = cs.TextureMeshPhoto(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], padding=5,
                                    **dict(SETTINGS[setting], dataTerm=["area", "gmi"][SETTINGS[setting]["dataTerm"]]))
        with monkeypatch.context() as m:
            m.setattr(cs, "_upload_images", _pitched_upload)
            pitched = cs.TextureMeshPhoto(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], padding=5,
                                          **dict(SETTINGS[setting],
                                                 dataTerm=["area", "gmi"][SETTINGS[setting]["dataTerm"]]))
        _same(dense, pitched)
        assert dense[5][11] > 0 and np.isfinite(pitched[0]).all()


# ---- the effects ------------------------------------------------------------------------------------------------------
def _project_faces(c, a):
    X = np.asarray(c["v"], np.float64)[np.asarray(c["t"], np.int64)]
    u, v, _ = to.project(c["Ks"][a], c["Rs"][a], c["ts"][a], X)
    return u, v


def _atlas_at_centroids(atlas, uv, faces):
    x, y = uv[faces, :, 0].mean(1), uv[faces, :, 1].mean(1)
    return atlas[np.floor(y).astype(int), np.floor(x).astype(int)].astype(np.float64)


def test_transient_occluder():
    """A constant rectangle painted into the view that textures most faces: with outlier rejection the faces inside
    it take other views, and their texture is closer to the clean view than TextureMesh's."""
    c = _scene_case(0.0, 0.5)
    base = cs.TextureMesh(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], atlasWidth=ATLAS_WIDTH)
    a = int(np.bincount(base[2][base[2] >= 0]).argmax())
    u, v = _project_faces(c, a)
    won = np.flatnonzero(base[2] == a)
    cu, cv = u[won].mean(1), v[won].mean(1)
    x0, y0 = max(0, int(np.median(cu)) - 40), max(0, int(np.median(cv)) - 30)
    x1, y1 = x0 + 80, y0 + 60
    painted = [im.copy() for im in c["imgs"]]
    painted[a][y0:y1, x0:x1] = 255.0
    inside = np.flatnonzero((base[2] == a) & (u >= x0 + 1).all(1) & (u <= x1 - 2).all(1) & (v >= y0 + 1).all(1) &
                            (v <= y1 - 2).all(1))
    assert len(inside) >= 10, len(inside)
    area = cs.TextureMesh(painted, c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], atlasWidth=ATLAS_WIDTH)
    photo = cs.TextureMeshPhoto(painted, c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], dataTerm="area",
                                atlasWidth=ATLAS_WIDTH)
    moved = float(np.mean(photo[2][inside] != a))
    clean = c["imgs"][a][np.floor(v[inside].mean(1) + 0.5).astype(int), np.floor(u[inside].mean(1) + 0.5).astype(int)]
    seen = photo[2][inside] >= 0
    e_area = float(np.mean(np.abs(_atlas_at_centroids(area[0], area[1], inside) - clean)))
    e_photo = float(np.mean(np.abs(_atlas_at_centroids(photo[0], photo[1], inside[seen]) - clean[seen])))
    print("occluder: view %d, %d faces inside, %.3f moved, removed %d (best %d), mean |error| %.2f -> %.2f "
          "(ratio %.3f)" % (a, len(inside), moved, photo[5][14], photo[5][15], e_area, e_photo, e_photo / e_area))
    assert moved >= OCCLUDER_MOVED and seen.all()
    assert e_photo <= OCCLUDER_ERROR_RATIO * e_area


def _box_blur(img, r=2):
    p = np.pad(img.astype(np.float64), r, mode="edge")
    H, W = img.shape
    out = np.zeros((H, W))
    for dy in range(2 * r + 1):
        for dx in range(2 * r + 1):
            out += p[dy:dy + H, dx:dx + W]
    return (out / (2 * r + 1) ** 2).astype(np.float32)


def _chart_sharpness(atlas, charts):
    g, n = 0.0, 0
    for _, _, _, w, h, ox, oy, _ in charts:
        s = tpo.sobel(atlas[oy:oy + h, ox:ox + w])
        g += float(s.sum())
        n += s.size
    return g / n


def test_blurred_view():
    """One view box-blurred: under GMI it textures clearly fewer faces than under the area term, and the charts'
    texels are sharper."""
    c = _scene_case(0.0, 0.5)
    base = cs.TextureMesh(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], atlasWidth=ATLAS_WIDTH)
    a = int(np.bincount(base[2][base[2] >= 0]).argmax())
    imgs = [im.copy() for im in c["imgs"]]
    imgs[a] = _box_blur(imgs[a])
    area = cs.TextureMeshPhoto(imgs, c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], dataTerm="area", outlierK=0.0,
                               atlasWidth=ATLAS_WIDTH)
    gmi = cs.TextureMeshPhoto(imgs, c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], dataTerm="gmi", outlierK=0.0,
                              atlasWidth=ATLAS_WIDTH)
    na, ng = int((area[2] == a).sum()), int((gmi[2] == a).sum())
    sa, sg = _chart_sharpness(area[0], area[3]), _chart_sharpness(gmi[0], gmi[3])
    print("blur: view %d labels %d faces under the area term, %d under GMI (ratio %.3f); chart sharpness %.3f -> %.3f "
          "(gain %.3f)" % (a, na, ng, ng / max(na, 1), sa, sg, sg / sa))
    assert na > 0 and ng <= BLUR_LABEL_RATIO * na
    assert sg > BLUR_SHARPNESS_GAIN * sa
