"""CPU checks of the describe stage's float64 restatement (tests/describe_ref.py) and of cs_describe_points' argument
checks.  The restatement is tied to the C oracle (which test_golden_cpu ties to the reference) on the oracle's own
pyramid levels and keypoints, and checked on hand-computed windows: a linear ramp, a flat window (quirk Q21) and a
saturated edge (quirk Q22)."""
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import describe_ref as dr
import oracle
from cudasift_b200 import build
from cudasift_b200.synth import synth_image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_E_ARG = -2
LIBM_SIN_ERR = 2.0 ** -23      # glibc sinf / cosf: below one ulp of a value in [-1, 1]


def oracle_levels(img, octaves):
    lev = [oracle.lowpass(img, 1.0)]
    for _ in range(1, octaves):
        lev.append(oracle.scaledown(lev[-1]))
    return lev


def level_keypoints(recs, i):
    """The oracle's primaries of level i, back in level coordinates (as the detector left them)."""
    s = float(1 << i)
    p = recs[recs["subsampling"] == s].copy()
    for f in ("xpos", "ypos", "scale"):
        p[f] /= s
    # secondaries repeat a primary's position: keep the first record of each (x, y, scale)
    _, first = np.unique(np.stack([p["xpos"], p["ypos"], p["scale"]], 1), axis=0, return_index=True)
    return p[np.sort(first)]


@pytest.mark.parametrize("seed,w,h", [(1000, 640, 480), (7, 800, 600), (31, 321, 241)])
def test_restatement_matches_oracle(seed, w, h):
    """Orientations, secondaries and descriptors of the restatement equal the oracle's within float32 rounding, and
    both count the same Q22 votes."""
    img = synth_image(w, h, seed=seed)
    recs, _ = oracle.extract(img, 5, 1.0, 3.0)
    lev = oracle_levels(img, 5)
    seen = dict(kp=0, q22=0, amb=0)
    for i in range(5):
        p = level_keypoints(recs, i)
        if len(p) == 0:
            continue
        lv = lev[i]
        o = dr.orientations(lv, p["xpos"], p["ypos"], p["scale"])
        got = oracle.orientations(lv, p)
        prim, sec = got[:len(p)], got[len(p):]
        assert dr.match_orientation(o, prim["orientation"], o["cand1"]).all(), ("primary orientation", i)
        ok = dr.match_orientation(o, prim["orientation"], o["cand1"] & ~o["near_tie"][:, None])
        assert ok.sum() == (~o["near_tie"]).sum(), i
        # a secondary exactly where the restatement decides one (ties aside)
        has2 = np.zeros(len(p), bool)
        key = {(a, b, c): k for k, (a, b, c) in enumerate(zip(p["xpos"], p["ypos"], p["scale"]))}
        idx2 = np.array([key[(a, b, c)] for a, b, c in zip(sec["xpos"], sec["ypos"], sec["scale"])], np.int64)
        has2[idx2] = True
        sure = o["has2_certain"]
        assert np.array_equal(has2[sure], o["has2"][sure]), i
        if len(idx2):
            assert dr.match_orientation({k: v[idx2] for k, v in o.items()}, sec["orientation"], o["cand2"][idx2]).all()
        # descriptors at the oracle's orientations (primaries and secondaries)
        d_in = got
        od, q22 = oracle.descriptors(lv, d_in, 1.0)
        d = dr.descriptors(lv, d_in["xpos"], d_in["ypos"], d_in["scale"], d_in["orientation"], sin_err=LIBM_SIN_ERR)
        assert q22 == d["q22"].sum(), ("Q22 votes", i, q22, d["q22"].sum())
        q21 = d["q21"]
        assert np.all(np.abs(od["data"][q21] - dr.R32) < 1e-6), "Q21 rows are constant"
        r = np.nonzero(~q21)[0]
        ok, bmax, _ = dr.within_bound(d, od["data"][r].astype(np.float64), r)
        # a bound of 0.2 (the clamp) leaves an element unchecked: such rows must stay under the 1 % of rows a
        # blanket allowance would exempt
        assert ok.all() and (bmax >= 0.2).sum() <= 0.01 * len(r), i
        err = np.abs(od["data"][r].astype(np.float64) - d["desc"][r])
        assert err.max(initial=0) < 1e-5, (i, err.max())
        seen["kp"] += len(d_in)
        seen["q22"] += q22
    assert seen["kp"] > 100


def test_ramp_orientation_and_support():
    """A linear ramp: every gradient is (a, b), so the histogram has one bin and the orientation is atan2(b, a); the
    descriptor of orientation 0 puts all weight into one angle bin of every cell."""
    h, w = 96, 96
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = (2.0 * xx + 1.0 * yy).astype(np.float32)
    o = dr.orientations(img, [48.0], [48.0], [2.0])
    ang = np.degrees(np.arctan2(2 * 1.0, 2 * 2.0))       # dx = 2a, dy = 2b
    # single-bin histogram: the parabola through (sm[b-1], sm[b], sm[b+1]) of a [1 4 6 4 1] kernel centres on the bin
    b = int(16.0 * np.radians(ang) / dr.PI_Q14 + 16.5)
    assert o["i1"][0] == b and not o["has2"][0]
    assert abs(o["ori1"][0] - 11.25 * b) < 1e-9
    img2 = np.tile(np.arange(w, dtype=np.float32) * 3.0, (h, 1))     # pure x ramp, gradient (6, 0)
    d = dr.descriptors(img2, [48.0], [48.0], [2.0], [0.0])
    assert not d["q21"][0] and d["q22"][0] == 0
    v = d["raw"][0].reshape(16, 8)
    # angle of (6, 0) is 0: angf = 4 exactly -> every vote lands in angle bin 4 of its cells
    assert np.all(v[:, [0, 1, 2, 3, 5, 6, 7]] == 0.0) and np.all(v[:, 4] > 0)
    # the support: the gaussian-weighted bilinear split over a 16x16 grid of 4x4 cells, with the cell profile
    g16 = dr._gauss16()
    prof = np.zeros(4)
    for x in range(16):
        hori = (x + 2) // 4 - 1
        horf = (x - 1.5) * 0.25 - hori
        if 0 <= hori <= 3:
            prof[hori] += (1 - horf) * g16[x]
        if 0 <= hori + 1 <= 3:
            prof[hori + 1] += horf * g16[x]
    want = 6.0 * np.outer(prof, prof).ravel()
    assert np.allclose(v[:, 4], want, rtol=1e-6)


def test_flat_window_is_q21():
    """A window on an exactly constant region: all gradients are zero, fast_atan2(0, 0) is NaN, the NaN votes make
    the first norm NaN and fminf turns every element into 0.2: a constant 1/sqrt(128) row.  The orientation window
    has no peak at all (NaN orientation, no secondary)."""
    img = np.full((64, 64), 77.0, np.float32)
    o = dr.orientations(img, [32.0], [32.0], [2.0])
    assert not o["has1"][0] and np.isnan(o["ori1"][0]) and not o["has2"][0] and o["has2_certain"][0]
    d = dr.descriptors(img, [32.0], [32.0], [2.0], [30.0])
    assert d["q21"][0] and np.allclose(d["desc"][0], dr.R32, rtol=0, atol=1e-12)


def edge_image(w=64, h=64):
    """A saturated edge: every column constant (so dy == +0 exactly at orientation 0), falling to the right."""
    x = np.arange(w, dtype=np.float64)
    return np.tile((100.0 - 80.0 * np.tanh((x - w / 2) / 8.0)).astype(np.float32), (h, 1))


def test_saturated_edge_is_q22():
    """Columns constant, values falling to the right: dy == +0 and dx < 0 for every sample at orientation 0, so
    angf = 8.0001 and angi == 8 everywhere; the restatement carries those votes into bin 0 of the next cell, and the
    variant without the carry differs exactly there."""
    img = edge_image()
    d = dr.descriptors(img, [32.0], [32.0], [2.0], [0.0])
    assert d["q22"][0] > 100 and not d["q21"][0]
    d0 = dr.descriptors(img, [32.0], [32.0], [2.0], [0.0], q22_carry=False)
    assert d0["q22"][0] == d["q22"][0]
    diff = np.abs(d["raw"][0] - d0["raw"][0]).reshape(16, 8)
    assert diff[:, 1:].max() == 0.0 and diff[1:, 0].min() > 0.0 and diff[0, 0] == 0.0
    assert np.abs(d["desc"][0] - d0["desc"][0]).max() > 1e-2
    od, q22 = oracle.descriptors(img, _rec(32.0, 32.0, 2.0, 0.0))
    assert q22 == d["q22"][0]
    assert np.abs(od["data"][0] - d["desc"][0]).max() < 1e-5


def _rec(x, y, s, o):
    r = np.zeros(1, oracle.SIFT_DTYPE)
    r["xpos"], r["ypos"], r["scale"], r["orientation"], r["subsampling"] = x, y, s, o, 1.0
    return r


def test_tex2d_matches_oracle():
    img = synth_image(64, 48, seed=3)
    rng = np.random.default_rng(0)
    x = rng.uniform(-3, 67, 2000).astype(np.float32)
    y = rng.uniform(-3, 51, 2000).astype(np.float32)
    x[:3] = [np.nan, 1e20, -1e20]
    assert np.array_equal(dr.tex2d(img, x, y), oracle.tex2d(img, x, y))


def test_symbol_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    assert re.search(r"\bcs_describe_points\s*\(", header)
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    assert "cs_describe_points" in {line.split()[-1] for line in out.splitlines() if line.strip()}


def test_describe_points_rejects_bad_arguments():
    """Every invalid argument fails with CS_E_ARG before any CUDA call, so also without a device."""
    img = np.zeros(64 * 64, np.float32)
    pts = np.zeros(8 * 576, np.uint8)
    pi, pp = img.ctypes.data, pts.ctypes.data
    ok = dict(img=pi, w=64, h=64, pitch=64, pts=pp, n=4, maxPts=8, fin=1.0)
    cases = [("NULL image", dict(img=None)), ("NULL records", dict(pts=None)), ("w 0", dict(w=0)), ("h 0", dict(h=0)),
             ("pitch < w", dict(pitch=63)), ("n < 0", dict(n=-1)), ("n > maxPts", dict(n=9)),
             ("maxPts 0", dict(maxPts=0, n=0)), ("maxPts < 0", dict(maxPts=-1, n=0))]
    f = cs.lib().cs_describe_points
    for what, change in cases:
        a = dict(ok, **change)
        assert f(a["img"], a["w"], a["h"], a["pitch"], a["pts"], a["n"], a["maxPts"], a["fin"]) == CS_E_ARG, what
        assert b"cs_describe_points" in cs.lib().cs_last_error()
