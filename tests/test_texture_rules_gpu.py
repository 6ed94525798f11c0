"""GPU checks of cs_texture_mesh rule by rule against tests/texture_oracle.py: every case of tests/texture_cases.py runs
on the GPU and in the float64 oracle with the same arguments, and the return value, stats, info, labels, faceChart,
chart table, atlas and texture coordinates (as uint32) must be equal, with the launch count the header states
(14 + 2 G + rounds + colours x sweeps).  The cases reach edges with 1, 3 and 4 faces and repeated faces (rule 1), pixel
centres on shared edges, ties of coplanar copies at depthTol 0, A == 0, faces crossing Y_z = 0 and clipped boxes
(rule 2), more than 8 passing images with ties, the view angle at 4 and 90 degrees, both sides of 1 + depthTol and
images of every size in several groups (rule 3), lambda 0 and 1000, the sweep cap and 4 colours (rule 4), a 10^5-face
chart, a deep strip and one-face charts (rule 5), padding clamped at both borders, a chart as wide as the atlas, an
exactly filled shelf, a row cut through a chart and an empty atlas (rule 6), and more than 2^21 faces.  No tolerances."""
import ctypes
import time

import numpy as np
import pytest

import cudasift_b200 as cs
import texture_cases as tc
import texture_oracle as to

pytestmark = pytest.mark.gpu

GROUP_CAP = 1 << 30             # the call's default image-group cap (texture_group_bytes 0)

CASES = {
    "topology": tc.topology,
    "occluder": tc.occluder,
    "occluder_jittered": lambda: tc.occluder(0.3),
    "coplanar_tol0": tc.coplanar,
    "coplanar_tol1": lambda: tc.coplanar(1.0),
    "raster_edges": tc.raster_edges,
    "many_views": tc.many_views,
    "many_views_90deg": lambda: tc.many_views(90.0),
    "many_views_4deg": lambda: tc.many_views(4.0),
    "depth_ratio": tc.depth_ratio,
    "depth_ratio_tol0": lambda: tc.depth_ratio(0.0),
    "depth_ratio_tol1": lambda: tc.depth_ratio(1.0),
    "mixed_sizes": tc.mixed_sizes,
    "labelling": tc.labelling,
    "labelling_lam0": lambda: tc.labelling(lam=0.0),
    "labelling_lam1000": lambda: tc.labelling(lam=1e3),
    "labelling_sweeps1": lambda: tc.labelling(lam=5.0, maxSweeps=1),
    "labelling_sweeps2": lambda: tc.labelling(lam=5.0, maxSweeps=2),
    "big_chart": tc.big_chart,
    "deep_strip": tc.deep_strip,
    "single_charts": tc.single_charts,
    "atlas_pad0": tc.atlas,
    "atlas_pad16": lambda: tc.atlas(16),
    "unseen": tc.unseen,
}
_made, _refs = {}, {}


def case(name):
    if name not in _made:
        _made[name] = tc.scale() if name == "scale" else CASES[name]()
    return _made[name]


def oracle(name):
    if name not in _refs:
        c = case(name)
        t0 = time.perf_counter()
        _refs[name] = to.texture(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], **c["kw"])
        print("%s: %d faces, %d images, oracle %.1f s, stats %s" % (name, len(c["t"]), len(c["imgs"]),
                                                                   time.perf_counter() - t0, _refs[name]["stats"]))
    return _refs[name]


def run(c, maxRows, maxCharts=None, cap=None):
    """cs_texture_mesh on the case's arguments with every output, faceChart included, maxRows atlas rows (at least 1
    allocated) and maxCharts chart rows (None: one per face); cap the texture_group_bytes to run under.  Returns the
    outputs as the oracle names them, and the launches counted."""
    kw = dict(lam=0.5, maxViewAngleDeg=75.0, depthTol=0.01, padding=2, atlasWidth=1024, maxSweeps=100) | c["kw"]
    v, t, imgs = c["v"], c["t"], c["imgs"]
    T, W = len(t), kw["atlasWidth"]
    arrs, bufs, table = cs._upload_images(imgs)
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
        info, stats = np.full(2, -1.0), np.full(11, -1, np.int64)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        if cap is not None:
            assert cs.lib().cs_set_tuning(b"texture_group_bytes", cap) == 0
        try:
            before = cs.lib().cs_launch_count()
            C = cs.lib().cs_texture_mesh(table, len(imgs), p(K), p(R), p(tt), ins[0].ptr, len(v), ins[1].ptr, T,
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


def compare(got, ref, launches=None, groups=1):
    st = ref["stats"]
    assert got["stats"] == st
    assert got["ret"] == ref["ret"]
    assert np.array_equal(np.asarray(got["info"]).view(np.uint64), np.asarray(ref["info"], np.float64).view(np.uint64))
    assert np.array_equal(got["labels"], ref["labels"])
    assert np.array_equal(got["faceChart"], ref["faceChart"])
    C = ref["ret"]
    assert np.array_equal(got["charts"][:C], ref["charts"]) and (got["charts"][C:] == -7).all()
    assert np.array_equal(got["atlas"].view(np.uint32), ref["atlas"].view(np.uint32))
    assert np.array_equal(got["uv"].view(np.uint32), ref["uv"].view(np.uint32))
    if launches is not None:
        assert launches == 14 + 2 * groups + st[4] + st[3] * st[5], (launches, groups, st)


def _shapes(c):
    return [im.shape for im in c["imgs"]]


@pytest.mark.parametrize("name", sorted(CASES))
def test_rules(name):
    c = case(name)
    ref = oracle(name)
    got, launches = run(c, ref["stats"][8])
    print("%s: GPU stats %s, info %s" % (name, got["stats"], list(got["info"])))
    compare(got, ref, launches, tc.image_groups(_shapes(c), GROUP_CAP))


def test_mixed_sizes_under_group_caps():
    c = case("mixed_sizes")
    ref = oracle("mixed_sizes")
    seen = []
    for cap in c["groups"]:
        G = tc.image_groups(_shapes(c), cap)
        seen.append(G)
        got, launches = run(c, ref["stats"][8], cap=cap)
        compare(got, ref, launches, G)
    assert seen == [4, 5, len(c["imgs"])], seen


def test_rows_cut_a_chart():
    """maxAtlasRows through the middle of the second shelf's charts: the prefix of the rows, everything else whole."""
    c = case("atlas_pad0")
    ref = oracle("atlas_pad0")
    oy, h = ref["charts"][:, 6], ref["charts"][:, 4]
    cut = int(oy.max() + h[oy.argmax()] // 2)
    assert 0 < cut < ref["stats"][8]
    got, _ = run(c, maxRows=cut, maxCharts=1)
    assert got["stats"][:9] == ref["stats"][:9] and got["stats"][9] == cut and got["stats"][10] == ref["stats"][10]
    assert np.array_equal(got["atlas"].view(np.uint32), ref["atlas"][:cut].view(np.uint32))
    assert np.array_equal(got["charts"][:1], ref["charts"][:1]) and (got["charts"][1:] == -7).all()
    assert np.array_equal(got["uv"].view(np.uint32), ref["uv"].view(np.uint32))


def _bytes(got):
    return [np.asarray(got[k]).tobytes() for k in ("ret", "stats", "info", "charts", "atlas", "uv", "labels",
                                                     "faceChart")]


@pytest.mark.parametrize("name", ["big_chart", "scale"])
def test_twice_the_same_bytes(name):
    """The 10^5-face chart (the union-find under load) and the 2^21-face mesh: equal to the oracle, twice."""
    c = case(name)
    ref = oracle(name)
    a, launches = run(c, ref["stats"][8])
    compare(a, ref, launches, tc.image_groups(_shapes(c), GROUP_CAP))
    b, _ = run(c, ref["stats"][8])
    assert _bytes(a) == _bytes(b)
    if name == "scale":
        assert len(c["t"]) > 1 << 21 and ref["stats"][7] > 0
