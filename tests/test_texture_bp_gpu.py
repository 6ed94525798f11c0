"""GPU checks of cs_texture_mesh_bp (TextureMeshBP) against tests/texture_bp_oracle.py: every output (labels, charts,
texture coordinates, atlas, info [3], stats [20]) bit-equal to the oracle on the scene mesh (jitter 0 and 0.3, lambda
0.5 and 5), on a PoissonMesh -> SimplifyMesh sphere, on the strip and the island, with both data terms and the
outlier test on and off; with maxBpSweeps 0, cs_texture_mesh_photo's outputs byte for byte; image groups of 3, 2 and 1
images and two calls in a row give the same bytes; the launch count; statuses 0, 2 and 3; truncation prefixes; and
pitched images."""
import ctypes

import numpy as np
import pytest

import cudasift_b200 as cs
import texture_bp_cases as bc
import texture_bp_oracle as bo
import texture_cases as tc
from test_dense_pitch_gpu import _pitched_upload, _same
from test_texture_photo_gpu import SETTINGS, _scene_case, sphere  # noqa: F401  (sphere is a fixture)
from test_texture_photo_gpu import run as run_photo

pytestmark = pytest.mark.gpu

ATLAS_WIDTH = 1024


def run(c, maxRows=None, maxCharts=None, cap=None, upload=None, **over):
    """cs_texture_mesh_bp on a case (texture_cases' dict; over overrides its kw) with every output, maxRows atlas rows
    (None: 4096) and maxCharts chart rows (None: one per face); cap the texture_group_bytes.  Returns the outputs as the
    oracle names them, and the launches counted."""
    kw = dict(lam=0.5, maxViewAngleDeg=75.0, depthTol=0.01, padding=2, atlasWidth=ATLAS_WIDTH, maxSweeps=100,
              dataTerm=1, outlierK=3.0, outlierMinSigma=4.0, maxBpSweeps=32) | c["kw"] | over
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
        info, stats = np.full(3, -1.0), np.full(20, -1, np.int64)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        if cap is not None:
            assert cs.lib().cs_set_tuning(b"texture_group_bytes", cap) == 0
        try:
            before = cs.lib().cs_launch_count()
            C = cs.lib().cs_texture_mesh_bp(table, len(imgs), p(K), p(R), p(tt), ins[0].ptr, len(v), ins[1].ptr, T,
                                            kw["dataTerm"], kw["outlierK"], kw["outlierMinSigma"], kw["maxBpSweeps"],
                                            kw["lam"], kw["maxViewAngleDeg"], kw["depthTol"], kw["padding"], W,
                                            kw["maxSweeps"], outs[0].ptr if maxRows else None, maxRows, outs[1].ptr,
                                            outs[2].ptr, outs[3].ptr, p(charts) if maxCharts else None, maxCharts,
                                            p(info), p(stats), None)
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


def oracle(c, **over):
    kw = dict(atlasWidth=ATLAS_WIDTH, maxBpSweeps=32) | c["kw"] | over
    return bo.texture_bp(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], **kw)


def launch_count(st, groups=1):
    return 15 + 2 * groups + st[4] + st[3] * st[5] + (st[3] + 3) * st[16]


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
        assert launches == launch_count(st, groups), (launches, groups, st)


@pytest.mark.parametrize("setting", sorted(SETTINGS))
@pytest.mark.parametrize("jitter", [0.0, 0.3])
@pytest.mark.parametrize("lam", [0.5, 5.0])
def test_oracle_equality_scene(lam, jitter, setting):
    c = _scene_case(jitter, lam)
    ref = oracle(c, **SETTINGS[setting])
    got, launches = run(c, **SETTINGS[setting])
    print("scene lambda %g jitter %g %s: info %s stats %s" % (lam, jitter, setting, got["info"], got["stats"]))
    compare(got, ref, launches)
    assert ref["info"][1] <= ref["info"][2] <= ref["info"][0]


@pytest.mark.parametrize("setting", sorted(SETTINGS))
def test_oracle_equality_sphere(sphere, setting):
    ref = oracle(sphere, **SETTINGS[setting])
    got, launches = run(sphere, **SETTINGS[setting])
    print("sphere %s: %d faces, info %s stats %s" % (setting, len(sphere["t"]), got["info"], got["stats"]))
    compare(got, ref, launches)


@pytest.mark.parametrize("setting", [None] + sorted(SETTINGS))
@pytest.mark.parametrize("name", sorted(bc.CASES))
def test_cases(name, setting):
    c = bc.CASES[name]()
    over = SETTINGS[setting] if setting else {}
    ref = oracle(c, **over)
    got, launches = run(c, **over)
    print("%s %s: info %s stats %s" % (name, setting, got["info"], got["stats"]))
    compare(got, ref, launches)
    if name == "island" and setting is None:
        assert got["info"][2] < got["info"][0] and (got["labels"] == 0).all() and got["ret"] == 1


@pytest.mark.parametrize("which", ["scene", "sphere", "island"])
def test_no_sweeps_is_the_photo_call(which, sphere):
    c = {"scene": lambda: _scene_case(0.3, 0.5), "sphere": lambda: sphere, "island": bc.island}[which]()
    over = dict(dataTerm=c["kw"].get("dataTerm", 1), outlierK=c["kw"].get("outlierK", 3.0))
    a, la = run_photo(c, **over)
    b, lb = run(c, maxBpSweeps=0, **over)
    assert b["stats"][:16] == a["stats"] and b["stats"][16:] == [0] * 4 and lb == la
    assert np.asarray(b["info"])[:2].tobytes() == np.asarray(a["info"]).tobytes() and b["info"][2] == b["info"][0]
    for k in ("ret", "charts", "atlas", "uv", "labels", "faceChart"):
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def test_groups_and_repeats(sphere):
    a, _ = run(sphere)
    keys = ("ret", "stats", "info", "charts", "atlas", "uv", "labels", "faceChart")
    again, _ = run(sphere)
    for k in keys:
        assert np.asarray(a[k]).tobytes() == np.asarray(again[k]).tobytes(), k
    for per, groups in ((3, 3), (2, 4), (1, 8)):
        g, launches = run(sphere, cap=per * 160 * 120 * 8)
        for k in keys:
            assert np.asarray(a[k]).tobytes() == np.asarray(g[k]).tobytes(), (per, k)
        assert launches == launch_count(g["stats"], groups), (launches, groups, g["stats"])


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
    assert st[10] == 0 and launches == launch_count(st) and st[16] > 0
    c5 = _scene_case(0.0, 5.0)
    for sweeps in (1, 3):
        g3, l3 = run(c5, maxSweeps=1, maxBpSweeps=sweeps)
        ref = oracle(c5, maxSweeps=1, maxBpSweeps=sweeps)
        assert g3["stats"] == ref["stats"] and g3["stats"][5] == 1 and g3["stats"][16] == sweeps
        assert np.array_equal(g3["labels"], ref["labels"]) and l3 == launch_count(g3["stats"])
    g0, _ = run(c, maxSweeps=0)
    ref0 = oracle(c, maxSweeps=0)
    assert g0["stats"][10] == 3 == ref0["stats"][10] and g0["stats"][5] == 0
    assert np.array_equal(g0["labels"], ref0["kept"].astype(np.int32))
    bad = dict(c, t=c["t"].copy())
    bad["t"][3, 2] = bad["t"][3, 0]
    g2, launches = run(bad)
    assert g2["ret"] == 0 and g2["stats"][10] == 2 and launches == 1 and g2["stats"][11:] == [0] * 9
    assert (g2["charts"] == -7).all() and (g2["info"] == 0).all()


def test_pitched_images(monkeypatch):
    c = _scene_case(0.3, 0.5)
    dense = cs.TextureMeshBP(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], padding=5)
    with monkeypatch.context() as m:
        m.setattr(cs, "_upload_images", _pitched_upload)
        pitched = cs.TextureMeshBP(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], padding=5)
    _same(dense, pitched)
    assert dense[5][16] > 0 and len(dense[4]) == 3 and np.isfinite(pitched[0]).all()
