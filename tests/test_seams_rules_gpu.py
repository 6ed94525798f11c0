"""GPU checks of cs_level_texture_seams rule by rule against tests/seam_oracle.py on every case of tests/seam_cases.py:
the return value, stats[0..4], stats[6] and the status exactly, the CG count within 1 of a float64 PCG, the seam energy
before levelling bit for bit, the levelled atlas bit for bit against the oracle's texel stage given the device's
corner offsets, NaN corners on unseen faces, 13 launches (2 for invalid input) and the same bytes from a second call.
The cases reach touching, gapped and edge-aligned charts and every input failure (rule 1), uv edges of length 0, at an
exact integer and 2500 texels long, samples on texel centres, clamped taps, 3- and 4-face edges, unseen sides, fans
whose ends meet at one vertex (one of them so that the ends' order reaches the seam energy's bits) and a vertex on 8
labels up to 2^31 - 2 (rule 3), smoothness 0 and 50, regularization 1e-6 and 1, tol 0, maxIterations 0, b = 0, an
unknown with 3000 incidences and row counts either side of 256 and 2048 (rules 4-6), and padding 0 to 16, A = 0, A < 0,
texel centres on edges and vertices, key ties and clamped boxes (rule 7); a scale case past 2048 x 256 unknowns and seam
rows (all three levels of every total) runs against the vectorised oracle.  Every valid small case is solved again at
tol 1e-12, and the corner offsets and the energy after levelling must match the exact solution within the bound the
true residual and scipy's smallest eigenvalue of A give."""
import ctypes
import time

import numpy as np
import pytest
import scipy.sparse.linalg as spl

import cudasift_b200 as cs
import seam_cases as sc
import seam_oracle as so

pytestmark = pytest.mark.gpu

CS_E_ARG = -2
DEFAULTS = dict(padding=2, smoothness=0.1, regularization=1e-3, tol=1e-4, maxIterations=1000)
SENTINEL = np.float32(-12345.5)
TIGHT = dict(tol=1e-12, maxIterations=100000)
_made, _refs = {}, {}


def case(name):
    if name not in _made:
        _made[name] = sc.scale() if name == "scale" else sc.CASES[name]()
    return _made[name]


def oracle(name):
    """The oracle's rules 1-4 (the vectorised build for the scale case)."""
    if name not in _refs:
        c = case(name)
        t0 = time.perf_counter()
        b = (so.build_np if name == "scale" else so.build)(c["v"], c["t"], c["labels"], c["uv"], c["charts"],
                                                           c["atlas"], (DEFAULTS | c["kw"])["smoothness"])
        _refs[name] = b
        print("%s: %d faces, oracle build %.2f s" % (name, len(c["t"]), time.perf_counter() - t0))
    return _refs[name]


def run(c, **over):
    """cs_level_texture_seams through the C ABI with the output atlas and corner buffers filled with SENTINEL and the
    info and stats words with -1.  Returns (return value, stats, info, atlas, corner, launches)."""
    kw = DEFAULTS | c["kw"] | over
    v, t = np.ascontiguousarray(c["v"], np.float32), np.ascontiguousarray(c["t"], np.int32)
    lab, uv = np.ascontiguousarray(c["labels"], np.int32), np.ascontiguousarray(c["uv"], np.float32)
    atlas, charts = np.ascontiguousarray(c["atlas"], np.float32), np.ascontiguousarray(c["charts"], np.int32)
    T, (H, W) = len(t), atlas.shape
    bufs = [cs.DeviceBuffer(max(a.nbytes, 4)) for a in (v, t, lab, uv, atlas, atlas, np.zeros((T, 3), np.float32))]
    try:
        for b, a in zip(bufs, (v, t, lab, uv, atlas, np.full_like(atlas, SENTINEL),
                               np.full((T, 3), SENTINEL, np.float32))):
            b.upload(a)
        info, stats = np.full(3, -1.0), np.full(8, -1, np.int64)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        before = cs.lib().cs_launch_count()
        r = cs.lib().cs_level_texture_seams(bufs[0].ptr, len(v), bufs[1].ptr, T, bufs[2].ptr, bufs[3].ptr, p(charts),
                                            len(charts), bufs[4].ptr, H, W, kw["padding"], kw["smoothness"],
                                            kw["regularization"], kw["maxIterations"], kw["tol"], bufs[5].ptr,
                                            bufs[6].ptr, p(info), p(stats), None)
        launches = cs.lib().cs_launch_count() - before
        out = bufs[5].download(np.float32, H * W).reshape(H, W)
        corner = bufs[6].download(np.float32, 3 * T).reshape(T, 3)
        return r, stats, info, out, corner, launches
    finally:
        for b in bufs:
            b.free()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def compare(name, cg=True, **over):
    """The call on case `name` against the oracle; returns the device's outputs for further checks.  cg: compare the
    CG count and the status with the float64 PCG's (at tol 1e-12 their rounding may part them by more than one
    iteration)."""
    c = case(name)
    kw = DEFAULTS | c["kw"] | over
    b = oracle(name)
    got = run(c, **over)
    r, stats, info, out, corner, launches = got
    print("%s %s: ret %d, stats %s, info %s, launches %d" % (name, over or "", r, list(stats), list(info), launches))
    if b is None:
        assert r == 0 and list(stats) == [0] * 7 + [2] and np.array_equal(info.view(np.uint64), np.zeros(3, np.uint64))
        assert launches == 2
        assert (_bits(out) == _bits(np.full_like(out, SENTINEL))).all()
        assert (_bits(corner) == _bits(np.full_like(corner, SENTINEL))).all()
        return got
    _, its, conv = so.pcg(b, kw["regularization"], kw["tol"], kw["maxIterations"])
    status = 1 if not b["seam"] else 0 if conv else 3
    lab = np.asarray(c["labels"])
    t0 = time.perf_counter()
    texels = so.texels_np if name == "scale" else so.texels
    want_atlas, visited = texels(c["t"], lab, c["uv"], c["charts"], b["faceChart"], c["atlas"], corner,
                                 kw["padding"], copy_all=not b["seam"])
    print("%s: oracle PCG and texels %.2f s" % (name, time.perf_counter() - t0))
    want = [b["seen"], len(b["keys"]), b["edges"], len(b["seam"]), len(b["smooth"])]
    assert r == len(b["keys"])
    assert list(stats[:5]) == want and stats[6] == visited, (list(stats), want, visited)
    if cg:
        assert stats[7] == status and abs(int(stats[5]) - its) <= 1, (list(stats), its, status)
    assert np.array_equal(np.float64(info[0]).view(np.uint64), np.float64(so.energy(b)).view(np.uint64))
    assert launches == 13
    assert np.isnan(corner[lab < 0]).all() and np.isfinite(corner[lab >= 0]).all()
    assert np.array_equal(out.view(np.uint32), want_atlas.view(np.uint32))
    again = run(c, **over)
    for x, y in zip(got, again):
        assert np.array_equal(_bits(np.asarray(x)), _bits(np.asarray(y)))
    return got


VALID = sorted(n for n in sc.CASES if not n.startswith("invalid_"))


@pytest.mark.parametrize("name", sorted(n for n in sc.CASES if n != "invalid_overlap"))
def test_rules(name):
    compare(name)


def test_overlapping_charts_are_rejected():
    """Chart 0 widened over charts 1..7: the oracle's first-chart rule and the device's row-index search would disagree,
    so the table is rejected before any CUDA call, naming the first overlapping pair the sweep meets."""
    r, stats, info, out, corner, launches = run(case("invalid_overlap"))
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG and "charts[0] and charts[1] must not overlap" in msg, (r, msg)
    assert launches == 0 and (stats == -1).all() and (info == -1.0).all()
    assert (_bits(out) == _bits(np.full_like(out, SENTINEL))).all()


def test_scale():
    """320 000 faces whose unknowns (640 000) and seam rows (638 400) both pass 2048 x 256: all three levels of every
    total against the oracle (the seam energy bit for bit, the CG count within 1), and the texel stage bit for bit."""
    t0 = time.perf_counter()
    b = oracle("scale")
    print("scale: oracle build %.1f s" % (time.perf_counter() - t0))
    assert len(b["keys"]) > 2048 * 256 and len(b["seam"]) > 2048 * 256
    r, stats, info, out, corner, launches = compare("scale")
    assert stats[7] == 0 and info[2] <= DEFAULTS["tol"] and info[1] < info[0]
    print("scale: oracle wall time %.1f s in all" % (time.perf_counter() - t0))


@pytest.mark.parametrize("name", VALID)
def test_tight_solve(name):
    """At tol 1e-12: |x - g*| <= |b - A x| / lambda_min(A), with the true residual the device reports (info[2] |b|) and
    lambda_min from scipy; the float corner offsets add half an ulp.  The energy after levelling within the bound that
    gives through the seam rows."""
    c = case(name)
    kw = DEFAULTS | c["kw"] | TIGHT
    r, stats, info, out, corner, launches = compare(name, cg=False, **TIGHT)
    b = oracle(name)
    A, rhs = so.system(b, kw["regularization"])
    g = so.solve_exact(b, kw["regularization"])
    assert stats[7] == (1 if not b["seam"] else 0)
    bn = float(np.linalg.norm(rhs))
    if bn == 0.0:
        assert stats[5] == 0 and info[2] == 0.0 and (corner[c["labels"] >= 0] == 0).all()
        return
    lmin = float(spl.eigsh(A, k=1, sigma=0, which="LM", return_eigenvectors=False)[0])
    lmin *= 1 - 1e-9
    # every corner of an unknown holds the same float; the true residual the device reports against the one those
    # floats give, within what their rounding moves it (|A| <= 2 max diag by Gershgorin)
    cu, seen = b["cu"], b["cu"] >= 0
    xf = np.zeros(len(g))
    xf[cu[seen]] = corner[seen]
    assert np.array_equal(xf[cu[seen]].astype(np.float32).view(np.uint32), corner[seen].view(np.uint32))
    slack = 2 * A.diagonal().max() * 2.0 ** -24 * np.linalg.norm(xf)
    assert abs(info[2] * bn - np.linalg.norm(rhs - A @ xf)) <= slack * (1 + 1e-6) + 1e-9 * bn, info[2]
    assert info[2] <= 1e-10, info[2]
    err_x = max(info[2], TIGHT["tol"]) * bn / lmin
    err = np.abs(corner[seen].astype(np.float64) - g[cu[seen]])
    bound = err_x * (1 + 2.0 ** -24) + 2.0 ** -24 * np.abs(g[cu[seen]])
    print("%s: lambda_min %.3g, |b| %.3g, residual %.3g, max error %.3g (bound %.3g)"
          % (name, lmin, bn, info[2], err.max(), bound.max()))
    assert (err <= bound).all(), (err.max(), err_x)
    # the energy after: |E(x) - E(g*)| <= 2 sqrt(E(g*)) |D dx| + |D dx|^2, |D dx| <= sigma_max(D) |dx|, plus the
    # rounding of the sum
    Rs = len(b["seam"])
    deg = np.bincount(np.array([[i, j] for i, j, _, _ in b["seam"]]).reshape(-1), minlength=len(g))
    dd = np.sqrt(2.0 * deg.max()) * err_x
    e = so.energy(b, g)
    assert abs(info[1] - e) <= 2 * np.sqrt(e) * dd + dd * dd + 4 * Rs * 2.0 ** -52 * (e + info[0]), (info[1], e)
