"""CPU checks of cs_texture_mesh_photo: (a) the cases of tests/texture_photo_cases.py reach the rules they are built
for, on the oracle (tests/texture_photo_oracle.py); (b) each oracle mutation of a rule changes the output of at least
one case, so a kernel with the same slip would fail the GPU comparison in test_texture_photo_gpu.py; (c) the oracle
with both features off is cs_texture_mesh's oracle; (d) every CS_E_ARG case of the three new arguments, with the call
named; (e) the header declares the call, the library exports it and ctypes types it."""
import ctypes
import math
import os

import numpy as np
import pytest

import cudasift_b200 as cs
import texture_cases as tc
import texture_oracle as to
import texture_photo_cases as pc
import texture_photo_oracle as tpo
from test_texture_cpu import IMG, KS, RS, TS

CS_E_ARG = -2
_memo = {}


def _run(c, **over):
    kw = c["kw"] | over
    return tpo.texture_photo(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], **kw)


def _case(name):
    if name not in _memo:
        _memo[name] = pc.CASES[name]()
    return _memo[name]


def _ref(name):
    k = ("ref", name)
    if k not in _memo:
        _memo[k] = _run(_case(name))
    return _memo[k]


def _labels(name, **over):
    return _run(_case(name), **over)["labels"]


# ---- (a) the cases reach their rules --------------------------------------------------------------------------------
def test_subpixel_faces_fall_back():
    r = _ref("subpixel")
    T = len(_case("subpixel")["t"])
    assert r["stats"][11] == 0 and r["stats"][12] == r["stats"][2] == 3 * T
    c = _case("subpixel")
    u, v, _ = to.project(c["Ks"][0], c["Rs"][0], c["ts"][0], np.asarray(c["v"], np.float64)[c["t"]].mean(1))
    assert ((np.floor(u + 0.5) != np.floor(u)) & (np.floor(v + 0.5) == np.floor(v))).any()
    assert len(set(r["labels"].tolist())) == 3 and r["stats"][13] == T


def test_border_samples_use_clamped_taps():
    c = _case("border")
    r = _ref("border")
    on = np.zeros((64, 64), bool)
    on[[0, -1], :] = on[:, [0, -1]] = True
    hit = on & (r["bufs"][0] != to.EMPTY)
    assert hit[0].any() and hit[-1].any() and hit[:, 0].any() and hit[:, -1].any()
    assert r["stats"][12] < r["stats"][2] and len(set(r["labels"].tolist())) == 3
    assert not np.array_equal(tpo.sobel(c["imgs"][0])[0], tpo.sobel(np.pad(c["imgs"][0], 1))[1, 1:-1])


def test_occluded_faces_lose_some_box_pixels():
    c = _case("occluded")
    buf = to.depth_buffer(c["Ks"][0], c["Rs"][0], c["ts"][0], 64, 64, c["v"], c["t"])
    r = _ref("occluded")
    assert all(r["cands"][f] for f in range(12))
    owners = (buf & np.uint64(0xFFFFFFFF)).astype(np.int64)
    for f in range(12):
        x, y = 4 + 14 * (f % 4), 4 + 18 * (f // 4)
        assert (owners[y + 1:y + 3, x + 7:x + 11] >= 12).all()
        assert (owners[y:y + 10, x:x + 6] == f).all()


def test_equal_q_ties_to_the_lower_image():
    for dt in (0, 1):
        r = _run(_case("equal_q"), dataTerm=dt, outlierK=0.0)
        for c in r["cands"]:
            q = {a: x for x, a in c}
            assert q[0] == q[1] and [a for _, a in c if a < 2] == [0, 1]
        assert (r["labels"] != 1).all()


@pytest.mark.parametrize("name, tested, removed, best", [("m2", 0, 0, 0), ("m3", 32, 32, 0), ("even_m", 32, 32, 0),
                                                          ("textureless", 0, 0, 0),
                                                          ("mad0", 32, 32, 0), ("best_removed", 32, 32, 32),
                                                          ("at_limit", 32, 0, 0), ("capped", 32, 0, 0)])
def test_outlier_cases(name, tested, removed, best):
    r = _ref(name)
    assert r["stats"][13:16] == [tested, removed, best], r["stats"]
    assert r["stats"][1] == 0
    if name == "best_removed":
        assert (r["labels"] == 1).all()
    if name == "capped":
        assert r["stats"][2] == 10 * 32 and all(len(c) == 8 for c in r["cands"])
    if name == "textureless":
        r0 = _run(_case(name), dataTerm=0)
        assert np.array_equal(r["labels"], r0["labels"]) and (r["labels"] == 0).all()
        assert all(x > 0 for c in r["cands"] for x, _ in c)
    if name == "mad0":
        assert all([a for _, a in c] == [0, 1, 2, 3] for c in r["cands"])


def test_outlier_k_of_1_never_leaves_a_face_unseen():
    for name in pc.CASES:
        c = _case(name)
        off = _run(c, outlierK=0.0)
        on = _run(c, outlierK=1.0, outlierMinSigma=1e-3)
        assert on["stats"][1] == off["stats"][1], name
        for a, b in zip(off["cands"], on["cands"]):
            if len(a) >= 3:
                assert len(b) >= -(-len(a) // 2)


def test_both_features_off_is_texture_mesh():
    for name in ("occluded", "equal_q", "capped"):
        c = _case(name)
        a = to.texture(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], lam=c["kw"]["lam"])
        b = _run(c, dataTerm=0, outlierK=0.0)
        assert b["stats"][:11] == a["stats"] and b["stats"][13:] == [0, 0, 0]
        for k in ("labels", "uv", "atlas", "charts", "faceChart"):
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), (name, k)
        assert a["info"] == b["info"]


# ---- (b) sensitivity ------------------------------------------------------------------------------------------------
def _sobel_zero_pad(img):
    return ORIG["sobel"](np.pad(np.asarray(img, np.float32), 1))[1:-1, 1:-1]


def _median_upper(x):
    s = sorted(x)
    return s[len(s) // 2]


def _outliers_from_m2(c, K, s):
    if len(c) == 2 and K > 0:
        keep, _, b = ORIG["outliers"](c + [c[0]], K, s)
        return keep[:len(keep) - 1], True, b
    return ORIG["outliers"](c, K, s)


def _outliers_keep_best(c, K, s):
    keep, t, b = ORIG["outliers"](c, K, s)
    if b:
        keep = [c[0]] + keep
    return keep, t, False


def _outliers_ge(c, K, s):
    if not K > 0 or len(c) < 3:
        return c, False, False
    mu = [e[2] for e in c]
    med = tpo.median(mu)
    lim = K * tpo.spread(tpo.median([abs(x - med) for x in mu]), s)
    keep = [e for e in c if not abs(e[2] - med) >= lim]
    return keep, True, abs(mu[0] - med) >= lim


ORIG = {"outliers": tpo.outliers, "sobel": tpo.sobel}
MUTATIONS = {
    "fallback_floor": ("centroid_pixel", lambda uc, vc: (int(np.floor(uc)), int(np.floor(vc))), ["subpixel"]),
    "sobel_zero_pad": ("sobel", _sobel_zero_pad, ["border"]),
    "samples_any_face": ("visible", lambda keys, f: keys != to.EMPTY, ["occluded"]),
    "tie_image_descending": ("best8", lambda c: sorted(c, key=lambda e: (-e[0], -e[1]))[:8], ["equal_q"]),
    "gmi_without_floor": ("quality", lambda area, g, dt: area * g if dt else area, ["textureless"]),
    "tested_from_m2": ("outliers", _outliers_from_m2, ["m2"]),
    "median_upper_middle": ("median", _median_upper, ["even_m"]),
    "mad_without_floor": ("spread", lambda mad, s: 1.4826 * mad, ["mad0"]),
    "best_never_removed": ("outliers", _outliers_keep_best, ["best_removed"]),
    "removed_at_the_limit": ("outliers", _outliers_ge, ["at_limit"]),
    "test_before_the_cap": ("best8", lambda c: sorted(c, key=lambda e: (-e[0], e[1])), ["capped"]),
}


def _outputs(r):
    return [np.asarray(r[k]).tobytes() for k in ("ret", "stats", "info", "labels", "faceChart", "charts", "uv",
                                                 "atlas")]


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_every_mutation_is_seen(mutation, monkeypatch):
    name, fn, cases = MUTATIONS[mutation]
    changed = []
    for key in cases:
        ref = _outputs(_ref(key))
        with monkeypatch.context() as m:
            m.setattr(tpo, name, fn)
            out = _outputs(_run(_case(key)))
        if out != ref:
            changed.append(key)
    print("%s: changes %s" % (mutation, changed))
    assert changed, mutation


# ---- (d) argument checks ----------------------------------------------------------------------------------------------
def _call(dataTerm=1, K=3.0, sigma=4.0, T=4, V=4, lam=0.5, **kw):
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    charts = np.zeros((4, 8), np.int32)
    return cs.lib().cs_texture_mesh_photo(IMG, 2, p(KS), p(RS), p(TS), kw.get("verts", 0x1000), V, 0x2000, T, dataTerm,
                                          K, sigma, lam, 75.0, 0.01, 2, 1024, 100, 0x400000, 4, 0x10000, 0x20000,
                                          None, p(charts), 4, None, None, None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    assert msg.startswith("cs_texture_mesh_photo: invalid argument (CS_E_ARG)"), msg
    for w in words:
        assert w in msg, (w, msg)


def test_argument_checks():
    for dt in (-1, 2, 7):
        _rejects(_call(dataTerm=dt), "dataTerm")
    for K in (-1.0, 0.5, 0.999, 100.5, math.inf, math.nan, -math.inf):
        _rejects(_call(K=K), "outlierK")
    for s in (0.0, -1.0, 1000.5, math.inf, math.nan):
        _rejects(_call(sigma=s), "outlierMinSigma")
    # cs_texture_mesh's checks, under the new call's name
    _rejects(_call(lam=-1.0), "lambda")
    _rejects(_call(verts=0x1002), "d_vertices")
    _rejects(_call(T=-1), "numTriangles")


def test_accepted_settings_reach_the_overlap_sweep():
    """The ends of the accepted ranges pass the three checks (an overlapping layout then fails the sweep)."""
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    for dt, K, s in ((0, 0.0, 1e-9), (1, 1.0, 1000.0), (1, 100.0, 4.0)):
        r = cs.lib().cs_texture_mesh_photo(IMG, 2, p(KS), p(RS), p(TS), 0x1000, 4, 0x2000, 4, dt, K, s, 0.5, 75.0,
                                           0.01, 2, 1024, 100, 0x400000, 4, 0x1000, 0x20000, None,
                                           p(np.zeros((4, 8), np.int32)), 4, None, None, None)
        _rejects(r, "overlap")


def test_empty_mesh_makes_no_cuda_call():
    stats = np.full(16, -1, np.int64)
    info = np.full(2, -1.0)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    r = cs.lib().cs_texture_mesh_photo(IMG, 2, p(KS), p(RS), p(TS), None, 0, None, 0, 1, 3.0, 4.0, 0.5, 75.0, 0.01,
                                       2, 1024, 100, None, 0, None, None, None, None, 0, p(info), p(stats), None)
    assert r == 0 and (stats == 0).all() and (info == 0).all()


# ---- (e) header, export, ctypes -------------------------------------------------------------------------------------
def test_header_declares_the_call():
    hdr = open(os.path.join(os.path.dirname(cs.__file__), "..", "include", "cudasift_b200.h")).read()
    assert "int cs_texture_mesh_photo(" in hdr
    assert "15 + 2 G + rounds + colours x sweeps" in hdr and "64 bytes per face" in hdr
    f = cs.lib().cs_texture_mesh_photo
    assert isinstance(f, ctypes._CFuncPtr)
    assert len(f.argtypes) == 28 and f.argtypes[9] is ctypes.c_int and f.argtypes[10] is ctypes.c_double
    assert f.argtypes[11] is ctypes.c_double and f.restype is ctypes.c_int
    with pytest.raises(ValueError):
        cs.TextureMeshPhoto([], [], [], [], np.zeros((0, 3)), np.zeros((0, 3)), dataTerm="sharpness")
