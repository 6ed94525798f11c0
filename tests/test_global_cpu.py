"""cs_rotation_averaging without a device: the symbol, every argument check, the overlap sweep, the call that makes no
CUDA call, the wrapper through a fake library, and the float64 statement (its log, its linearisation against central
differences, the spanning-tree rule and recovery of a noise-free graph)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import global_cases as gc
import rotavg_oracle as ro
import test_arg_ranges_cpu as ar
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_E_ARG = -2


def test_symbol_declared_exported_and_typed():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE,
                         text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert "cs_rotation_averaging" in declared and "cs_rotation_averaging" in exported
    f = cs.lib().cs_rotation_averaging
    assert f.restype is ctypes.c_int and len(f.argtypes) == 18
    assert [f.argtypes[i] for i in (8, 9, 10)] == [ctypes.c_double] * 3
    assert "RotationAveraging" in cs.__all__ and hasattr(cs, "RotationAveraging")


def _graph():
    """Three images, two edges {0, 1}, {1, 2}, with rotations and weights that pass every check."""
    Q = np.stack([ro.exp_rot(np.array([0.1, 0.0, 0.0])), ro.exp_rot(np.array([0.0, 0.2, 0.0]))])
    return dict(N=3, edges=np.array([[0, 1], [1, 2]], np.int32), Rrel=Q, weights=np.array([10.0, 20.0]), ref=0,
                maxIt=10, maxLin=50, tol=1e-8, sigma=5.0, maxAngle=5.0)


def _call(g, R_out=None, res=True, inl=True, cost=True, trace=True, edgesPtr=True):
    """The call with g's arguments; the outputs pre-filled with 5 (7 for the statistics)."""
    ed = np.ascontiguousarray(g["edges"], np.int32)
    Q = np.ascontiguousarray(g["Rrel"], np.float64)
    w = np.ascontiguousarray(g["weights"], np.float64)
    E = len(ed) if "E" not in g else g["E"]
    out = dict(R=np.full((max(g["N"], 1), 9), 5.0), res=np.full(max(E, 1), 5.0), inl=np.full(max(E, 1), 5, np.uint8),
               cost=np.full(2, 5.0), trace=np.full((max(g["maxIt"], 1), 3), 5.0))
    stats, ms = np.full(6, 7, np.int64), np.full(2, 5.0)
    r = cs.lib().cs_rotation_averaging(
        g["N"], ed.ctypes.data if edgesPtr else None, E, Q.ctypes.data, w.ctypes.data, g["ref"], g["maxIt"],
        g["maxLin"], g["tol"], g["sigma"], g["maxAngle"], R_out if R_out is not None else out["R"].ctypes.data,
        out["res"].ctypes.data if res else None, out["inl"].ctypes.data if inl else None,
        out["cost"].ctypes.data if cost else None, out["trace"].ctypes.data if trace else None, stats.ctypes.data,
        ms.ctypes.data)
    return r, ms, out, stats


def test_rejects_every_invalid_argument():
    nan, inf = float("nan"), float("inf")

    def with_edge(e, i, j):
        def ch(g):
            g["edges"] = g["edges"].copy()
            g["edges"][e] = (i, j)
        return ch

    def with_R(e, f):
        def ch(g):
            g["Rrel"] = g["Rrel"].copy()
            f(g["Rrel"][e])
        return ch

    def with_w(e, v):
        def ch(g):
            g["weights"] = g["weights"].copy()
            g["weights"][e] = v
        return ch

    def scale(R):
        R *= 1.01

    def flip(R):
        R[:] = -R

    def put_nan(R):
        R[1, 1] = nan

    cases = [
        ("numImages 0", dict(N=0), "numImages"),
        ("numImages 2^24 + 1", dict(N=(1 << 24) + 1), "numImages"),
        ("numEdges < 0", dict(E=-1), "numEdges"),
        ("refImage < 0", dict(ref=-1), "refImage"),
        ("refImage = numImages", dict(ref=3), "refImage"),
        ("maxIterations -1", dict(maxIt=-1), "maxIterations"),
        ("maxIterations 1001", dict(maxIt=1001), "maxIterations"),
        ("maxLinearIterations 0", dict(maxLin=0), "maxLinearIterations"),
        ("maxLinearIterations 10001", dict(maxLin=10001), "maxLinearIterations"),
        ("linearTol 0", dict(tol=0.0), "linearTol"),
        ("linearTol 1", dict(tol=1.0), "linearTol"),
        ("linearTol NaN", dict(tol=nan), "linearTol"),
        ("sigmaDeg < 0", dict(sigma=-1.0), "sigmaDeg"),
        ("sigmaDeg > 180", dict(sigma=181.0), "sigmaDeg"),
        ("sigmaDeg NaN", dict(sigma=nan), "sigmaDeg"),
        ("maxAngleDeg 0", dict(maxAngle=0.0), "maxAngleDeg"),
        ("maxAngleDeg inf", dict(maxAngle=inf), "maxAngleDeg"),
        ("image out of range", with_edge(1, 1, 3), "edges[1]"),
        ("negative image", with_edge(0, -1, 1), "edges[0]"),
        ("self edge", with_edge(1, 2, 2), "edges[1] joins image 2"),
        ("R not orthogonal", with_R(1, scale), "Rrel[1]"),
        ("R a reflection", with_R(0, flip), "Rrel[0]"),
        ("R not finite", with_R(1, put_nan), "Rrel[1]"),
        ("weight 0", with_w(1, 0.0), "weights[1]"),
        ("weight < 0", with_w(0, -3.0), "weights[0]"),
        ("weight inf", with_w(1, inf), "weights[1]"),
        ("weight NaN", with_w(0, nan), "weights[0]"),
    ]
    for what, ch, name in cases:
        g = _graph()
        if callable(ch):
            ch(g)
        else:
            g.update(ch)
        r, ms, out, stats = _call(g)
        assert r == CS_E_ARG, (what, r)
        msg = cs.lib().cs_last_error().decode()
        assert msg.startswith("cs_rotation_averaging:") and "invalid argument" in msg and name in msg, (what, msg)
        assert not ms.any() and all((v == 5).all() for v in out.values()) and (stats == 7).all(), what
    for what, kw, name in [("NULL edges", dict(edgesPtr=False), "edges"), ("NULL R_out", dict(R_out=0), "R_out"),
                           ("NULL cost_out", dict(cost=False), "cost_out")]:
        g = _graph()
        r, ms, out, stats = _call(g, **kw)
        msg = cs.lib().cs_last_error().decode()
        assert r == CS_E_ARG and name in msg, (what, msg)
    # an output over an input, and two outputs over each other
    g = _graph()
    r, *_ = _call(g, R_out=g["Rrel"].ctypes.data + 8)
    assert r == CS_E_ARG and "R_out and Rrel overlap" in cs.lib().cs_last_error().decode()


def test_no_edges_makes_no_cuda_call():
    """numEdges == 0 returns R = I for refImage and NaN elsewhere, zero costs and trace, and holds without a device."""
    g = _graph()
    g.update(edges=np.zeros((0, 2), np.int32), Rrel=np.zeros((0, 3, 3)), weights=np.zeros(0), ref=1)
    r, ms, out, stats = _call(g)
    assert r == 0 and not ms.any()
    R = out["R"].reshape(3, 3, 3)
    assert (R[1] == np.eye(3)).all() and np.isnan(R[[0, 2]]).all()
    assert not out["cost"].any() and not out["trace"].any() and stats.tolist() == [0, 0, 1, 0, 0, 0]
    assert (out["res"] == 5).all() and (out["inl"] == 5).all()
    # optional outputs may be NULL
    r, *_ = _call(g, res=False, inl=False, trace=False)
    assert r == 0


# ---- the overlap sweep (the rule of test_arg_ranges_cpu.py) ----

def _rotavg(rng):
    N, E, it = int(rng.integers(1, 5)), int(rng.integers(1, 5)), int(rng.integers(1, 4))
    sizes = {"R_out": 72 * N, "residuals_out": 8 * E, "inlier_out": E, "cost_out": 16, "trace_out": 24 * it,
             "edges": 8 * E, "Rrel": 72 * E, "weights": 8 * E}
    outs = {"R_out", "residuals_out", "inlier_out", "cost_out", "trace_out"}

    def call(at):
        # the ranges are checked before any input is read
        return cs.lib().cs_rotation_averaging(N, at["edges"], E, at["Rrel"], at["weights"], 0, it, 10, 0.1, 5.0, 5.0,
                                           at["R_out"], at["residuals_out"], at["inlier_out"], at["cost_out"],
                                           at["trace_out"], None, None)

    return sizes, lambda a, b: a in outs or b in outs, call


def test_every_overlap_is_rejected_and_named():
    rng = np.random.default_rng(7)
    for _ in range(ar.LAYOUTS):
        sizes, forbidden, call = _rotavg(rng)
        at = ar._layout(rng, sizes, forbidden)
        r = call({x: ar.BASE + v for x, v in at.items()})
        msg = cs.lib().cs_last_error().decode()
        m = ar.MSG.match(msg)
        assert r == CS_E_ARG and m, (msg, at, sizes)
        _, a, b = m.groups()
        assert a in sizes and b in sizes and forbidden(a, b), msg
        assert ar._share((at[a], sizes[a]), (at[b], sizes[b])), (msg, at, sizes)
    assert not ar._buf.any()


# ---- the wrapper through a fake library ----

class _FakeLib:
    def __init__(self):
        self.calls = []

    def cs_rotation_averaging(self, *args):
        self.calls.append(args)
        stats = np.ctypeslib.as_array(ctypes.cast(args[16], ctypes.POINTER(ctypes.c_int64)), (6,))
        stats[3] = 2
        return 2


def test_wrapper_takes_verification_outputs(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    Q = np.stack([np.eye(3)] * 3)                                 # VerifyEssentialBatch's R: [J, 3, 3]
    R, res, inl, cost, trace, stats, ms = cs.RotationAveraging(4, [[0, 1], [1, 2], [2, 3]], Q, np.array([9, 8, 7]))
    args = fake.calls[-1]
    assert args[0] == 4 and args[2] == 3 and args[5] == 0
    assert args[6:11] == (50, 200, 1e-8, 5.0, 5.0)
    assert R.shape == (4, 3, 3) and res.shape == (3,) and inl.dtype == bool and trace.shape == (2, 3)
    w = np.ctypeslib.as_array(ctypes.cast(args[4], ctypes.POINTER(ctypes.c_double)), (3,))
    assert w.tolist() == [9.0, 8.0, 7.0]
    cs.RotationAveraging(2, np.zeros((0, 2)), np.zeros((0, 3, 3)), [], refImage=1, sigmaDeg=0.0, maxIterations=0)
    args = fake.calls[-1]
    assert args[1] is None and args[2] == 0 and args[5] == 1 and args[9] == 0.0 and args[15] is None
    with pytest.raises(ValueError):
        cs.RotationAveraging(3, [[0, 1]], Q, [1.0])


# ---- the float64 statement ----

def test_log_inverts_exp_at_every_angle():
    rng = np.random.default_rng(3)
    for th in list(np.linspace(0.0, np.pi - 1e-6, 40)) + [np.pi / 2, 2.5, 3.1, np.pi - 1e-9]:
        a = rng.normal(size=3)
        a /= np.linalg.norm(a)
        rho, t = ro.log_rot(ro.exp_rot(th * a))
        assert abs(t - th) < 1e-9 and np.allclose(rho, th * a, atol=1e-7), th
    assert ro.log_rot(np.eye(3))[1] == 0.0


def test_linearisation_against_central_differences():
    """rho_e(x) = log(exp(-[x_j]) D exp([x_i])) has Jacobian blocks Jr^-1(rho), -Jl^-1(rho); the cost's gradient is
    exactly that of the header's linear model rho + x_i - x_j."""
    rng = np.random.default_rng(5)
    for th in (0.05, 0.8, 2.0, 3.0):
        a = rng.normal(size=3)
        Ri, Rj = gc.random_rotation(rng), gc.random_rotation(rng)
        Q = Rj @ ro.exp_rot(th * a / np.linalg.norm(a)) @ Ri.T
        f = lambda xi, xj: ro.log_rot((Rj @ ro.exp_rot(xj)).T @ Q @ (Ri @ ro.exp_rot(xi)))[0]
        rho = f(np.zeros(3), np.zeros(3))
        h, Ji, Jj = 1e-6, np.empty((3, 3)), np.empty((3, 3))
        for k in range(3):
            d = np.zeros(3)
            d[k] = h
            Ji[:, k] = (f(d, np.zeros(3)) - f(-d, np.zeros(3))) / (2 * h)
            Jj[:, k] = (f(np.zeros(3), d) - f(np.zeros(3), -d)) / (2 * h)
        assert np.allclose(Ji, ro.jr_inv(rho), atol=1e-7) and np.allclose(Jj, -ro.jr_inv(-rho), atol=1e-7), th
        assert np.allclose(Ji.T @ rho, rho, atol=1e-7) and np.allclose(Jj.T @ rho, -rho, atol=1e-7), th
        # the world-frame update is the left update of vp_rotate: R exp([x]) = exp([R x]) R
        x = rng.normal(size=3) * 0.3
        assert np.allclose(Ri @ ro.exp_rot(x), ro.exp_rot(Ri @ x) @ Ri, atol=1e-14)


def test_spanning_tree_rule():
    """Heaviest edges first, ties to the lower index; the walk from the reference propagates R_j = Q R_i."""
    Q = [ro.exp_rot(np.array([0.1 * (e + 1), 0.0, 0.0])) for e in range(4)]
    edges = np.array([[0, 1], [1, 2], [0, 2], [2, 3]])
    R, reached = ro.spanning_tree(5, edges, np.stack(Q), np.array([5.0, 5.0, 5.0, 1.0]), 2)
    # {0, 1} and {1, 2} win the tie against {0, 2}; image 4 has no edge
    assert reached.tolist() == [True, True, True, True, False] and np.isnan(R[4]).all()
    assert np.allclose(R[2], np.eye(3)) and np.allclose(R[1], Q[1].T) and np.allclose(R[0], Q[0].T @ Q[1].T)
    assert np.allclose(R[3], Q[3])


@pytest.mark.parametrize("sigmaDeg", [0.0, 5.0])
def test_noise_free_graph_is_recovered(sigmaDeg):
    g = gc.view_graph(1, 50)
    out = ro.average(50, g["edges"], g["Rrel"], g["weights"], sigmaDeg=sigmaDeg)
    _, err = ro.align(out["R"], g["Rs"])
    assert np.max(err) < np.degrees(1e-10) and out["inlier"].all() and out["cost"][1] < 1e-20
    assert out["stats"].tolist()[:3] == [len(g["edges"]), 49, 50]


def test_start_with_noise_is_improved():
    """From the tree's start, IRLS lowers the cost and the rotation error on a noisy graph."""
    g = gc.view_graph(2, 60, noiseDeg=0.5)
    out = ro.average(60, g["edges"], g["Rrel"], g["weights"], sigmaDeg=0.0, maxIterations=20)
    R0, _ = ro.spanning_tree(60, g["edges"], g["Rrel"], g["weights"], 0)
    _, e0 = ro.align(R0, g["Rs"])
    _, e1 = ro.align(out["R"], g["Rs"])
    assert out["cost"][1] < 0.2 * out["cost"][0] and np.median(e1) < 0.5 * np.median(e0)
    assert out["trace"][-1, 2] <= ro.STOP or len(out["trace"]) == 20


# ---- global positioning ----

import globalpos_oracle as go                                    # noqa: E402
import triangulate_cases as tc                                   # noqa: E402


def test_positioning_symbol_and_wrapper(monkeypatch):
    f = cs.lib().cs_global_positioning
    assert f.restype is ctypes.c_int and len(f.argtypes) == 22 and f.argtypes[10] is ctypes.c_ulonglong
    assert "GlobalPositioning" in cs.__all__
    calls = []

    class Fake:
        def cs_device_alloc(self, n):
            return 4096 * (len(calls) + 1)

        def cs_device_free(self, p):
            return 0

        def cs_memcpy_h2d(self, d, s, n):
            return 0

        def cs_memcpy_d2h(self, d, s, n):
            return 0

        def cs_global_positioning(self, *args):
            calls.append(args)
            return 0

    class D:
        d_data, numPts = 1 << 20, 2

    monkeypatch.setattr(cs, "lib", lambda: Fake())
    cs.GlobalPositioning([D(), D()], np.eye(3), np.stack([np.eye(3)] * 2), [0, 2], [[0, 0], [1, 1]], refImage=1,
                         seed=7, loss="cauchy", lossScale=0.5)
    args = calls[-1]
    assert args[1] == 2 and args[5] == 1 and args[7] == 2 and args[8] is None
    assert args[9:16] == (1, 7, 2, 0.5, 100, 100, 1e-6)
    with pytest.raises(ValueError):
        cs.GlobalPositioning([D(), D()], np.eye(3), np.eye(3), [0, 2], [[0, 0], [1, 1]], loss="huber")


def _gp_call(**ch):
    K = np.stack([np.array([[800.0, 0, 640], [0, 800, 480], [0, 0, 1]])] * 2)
    buf = np.zeros(8192, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 64
    a = dict(S=2, K=K, R=np.stack([np.eye(3)] * 2), off=base, T=1, mem=base + 64, M=2, use=None, ref=0, loss=0,
             scale=1.0, it=10, lin=50, tol=1e-6, pts=base + 128, t=np.full((2, 3), 5.0), cost=np.full(2, 5.0))
    a.update(ch)
    if callable(a["pts"]):
        a["pts"] = a["pts"](a)
    sets = (cs.MatchSet * 2)(cs.MatchSet(base + 1024, 2), cs.MatchSet(base + 1024 + 2 * 576, 2))
    R = np.ascontiguousarray(a["R"])
    r = cs.lib().cs_global_positioning(sets, a["S"], a["K"].ctypes.data, R.ctypes.data, a["off"], a["T"], a["mem"],
                                       a["M"], a["use"], a["ref"], 0, a["loss"], a["scale"], a["it"], a["lin"],
                                       a["tol"], a["t"].ctypes.data if a["t"] is not None else None, a["pts"],
                                       a["cost"].ctypes.data, None, None, None)
    assert not buf.any()
    return r, cs.lib().cs_last_error().decode(), a


def test_positioning_rejects_every_invalid_argument():
    nan = float("nan")
    Rbad = np.stack([np.eye(3)] * 2)
    Rbad[1, 0, 0] = nan                                         # partly NaN: neither a rotation nor all NaN
    Rrefl = np.stack([np.eye(3), -np.eye(3)])
    cases = [
        (dict(S=0), "numImages"), (dict(T=-1), "numTracks"), (dict(M=-1), "numMembers"), (dict(ref=2), "refImage"),
        (dict(loss=3), "loss"), (dict(scale=0.0), "lossScale"), (dict(it=1001), "maxIterations"),
        (dict(lin=0), "maxLinearIterations"), (dict(tol=1.0), "linearTol"), (dict(t=None), "t_out"),
        (dict(off=None), "d_offsets"), (dict(mem=None), "d_members"), (dict(R=Rbad), "Rs[1]"),
        (dict(R=Rrefl), "Rs[1]"), (dict(pts=0), "d_points"),
    ]
    for ch, name in cases:
        r, msg, _ = _gp_call(**ch)
        assert r == CS_E_ARG and msg.startswith("cs_global_positioning:") and name in msg, (ch, msg)
    r, msg, a = _gp_call(pts=None)
    assert r == CS_E_ARG
    # d_points at d_members of the same call: no valid call is made (on a machine with a device it would launch a
    # kernel on the host buffer's address)
    r, msg, _ = _gp_call(pts=lambda a: a["mem"])
    assert r == CS_E_ARG and "d_points and d_members overlap" in msg, msg


def test_positioning_no_tracks_makes_no_cuda_call():
    t, cost = np.full((2, 3), 5.0), np.full(2, 5.0)
    R = np.stack([np.eye(3), np.full((3, 3), np.nan)])           # a NaN rotation is allowed
    r, msg, _ = _gp_call(T=0, M=0, R=R, t=t, cost=cost)
    assert r == 0 and np.isnan(t).all() and not cost.any()


def test_positioning_overlaps_are_rejected_and_named():
    rng = np.random.default_rng(11)
    for _ in range(ar.LAYOUTS):
        T, M, n0, n1 = (int(x) for x in rng.integers(1, 5, 4))
        sizes = {"d_points": 24 * T, "d_offsets": 4 * (T + 1), "d_members": 8 * M, "d_use": M,
                 "sets[0].pts": ar.REC * n0, "sets[1].pts": ar.REC * n1}
        at = ar._layout(rng, sizes, lambda x, y: "d_points" in (x, y))
        p = {x: ar.BASE + v for x, v in at.items()}
        K = np.stack([ar.K] * 2)
        R = np.stack([np.eye(3)] * 2)
        t, cost = np.zeros((2, 3)), np.zeros(2)
        sets = (cs.MatchSet * 2)(cs.MatchSet(p["sets[0].pts"], n0), cs.MatchSet(p["sets[1].pts"], n1))
        r = cs.lib().cs_global_positioning(sets, 2, K.ctypes.data, R.ctypes.data, p["d_offsets"], T, p["d_members"], M,
                                           p["d_use"], 0, 0, 0, 1.0, 10, 10, 0.1, t.ctypes.data, p["d_points"],
                                           cost.ctypes.data, None, None, None)
        m = ar.MSG.match(cs.lib().cs_last_error().decode())
        assert r == CS_E_ARG and m, cs.lib().cs_last_error()
        _, a, b = m.groups()
        assert "d_points" in (a, b) and ar._share((at[a], sizes[a]), (at[b], sizes[b]))
    assert not ar._buf.any()


def test_positioning_linearisation_against_central_differences():
    """r = v - s (X - c): dr/dc = s I, dr/dX = -s I, dr/ds = -(X - c); and the eliminated blocks P, beta of the header
    equal the Schur complement of the damped 7 x 7 normal matrix of one observation."""
    rng = np.random.default_rng(2)
    v = rng.normal(size=3)
    v /= np.linalg.norm(v)
    c, X, s = rng.normal(size=3), rng.normal(size=3), 1.3
    f = lambda z: v - z[6] * (z[3:6] - z[0:3])
    z0, h = np.concatenate([c, X, [s]]), 1e-6
    J = np.stack([(f(z0 + h * e) - f(z0 - h * e)) / (2 * h) for e in np.eye(7)], 1)
    d = X - c
    np.testing.assert_allclose(J, np.hstack([s * np.eye(3), -s * np.eye(3), -d[:, None]]), atol=1e-8)
    w2, lam = 0.7, 1e-2
    Jw, r = np.sqrt(w2) * J, np.sqrt(w2) * f(z0)
    H, g = Jw.T @ Jw, Jw.T @ r
    hh = go.damp(H[6, 6], lam)
    S = H[:6, :6] - np.outer(H[:6, 6], H[6, :6]) / hh
    bb = -g[:6] + H[:6, 6] * g[6] / hh
    P = w2 * s * s * (np.eye(3) - w2 * np.outer(d, d) / hh)
    beta = w2 * s * (f(z0) - w2 * d * (d @ f(z0)) / hh)
    np.testing.assert_allclose(S, np.block([[P, -P], [-P, P]]), atol=1e-12)
    np.testing.assert_allclose(bb, np.concatenate([-beta, beta]), atol=1e-12)


def _exact_scene(seed, N=20, T=120):
    """Noise-free float64 positions (the float32 of records would floor the recovery near 1e-7)."""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts = tc.cameras(rng, N)
    pts = rng.uniform(-3, 3, (T, 3))
    xy, off, mem = [[] for _ in range(N)], [0], []
    for k in range(T):
        for a in rng.choice(N, int(rng.integers(3, 8)), replace=False):
            xy[a].append(tc.project(Ks[a], Rs[a], ts[a], pts[k]))
            mem.append((int(a), len(xy[a]) - 1))
        off.append(len(mem))
    return [np.array(p).reshape(-1, 2) for p in xy], Ks, Rs, ts, np.array(off), np.array(mem), pts


def test_positioning_recovers_a_noise_free_scene_up_to_a_similarity():
    xy, Ks, Rs, ts, off, mem, pts = _exact_scene(4)
    out = go.position(xy, Ks, Rs, off, mem, seed=3, maxIterations=200, maxLinear=500, tol=1e-12)
    C, Ce = -np.einsum("aji,aj->ai", Rs, ts), -np.einsum("aji,aj->ai", Rs, out["t"])
    sc, R, t = go.umeyama(Ce, C)
    assert np.max(np.linalg.norm(sc * Ce @ R.T + t - C, axis=1)) < 1e-8 * tc.scale(Ks, Rs, ts)
    assert np.max(np.linalg.norm(sc * out["points"] @ R.T + t - pts, axis=1)) < 1e-8 * tc.scale(Ks, Rs, ts)
    # the gauge: the positioned centres' RMS distance from refImage's is 1
    assert abs(np.sqrt(np.mean(np.sum((Ce - Ce[0]) ** 2, 1))) - 1.0) < 1e-12


def test_positioning_optimum_matches_scipy():
    """At a small noisy scene, scipy's least_squares from the oracle's result (slightly moved) on the same residuals,
    with c_ref = 0 and the scale fixed by one point coordinate, reaches the oracle's cost and positions."""
    from scipy.optimize import least_squares
    xy, Ks, Rs, ts, off, mem, pts = tc.scene(6, numImages=8, numTracks=40, lengths=(3, 6), noise=0.5,
                                             outliers=(0.0, 0.0), away=0)
    out = go.position(xy, Ks, Rs, off, mem, seed=1, maxIterations=300, maxLinear=500, tol=1e-12)
    k, a, v = go.observations(xy, Ks, Rs, off, mem)
    C, T, O = len(xy), len(off) - 1, len(k)
    c0, X0, s0 = out["c"], out["X"], out["s"]
    fix = X0[0, 0]

    def unpack(z):
        c = np.vstack([np.zeros(3), z[:3 * (C - 1)].reshape(C - 1, 3)])
        X = np.concatenate([[fix], z[3 * (C - 1):3 * (C - 1) + 3 * T - 1]]).reshape(T, 3)
        return c, X, z[3 * (C - 1) + 3 * T - 1:]

    fun = lambda z: go.residual(*unpack(z), k, a, v)[1].ravel()
    z0 = np.concatenate([c0[1:].ravel(), X0.ravel()[1:], s0])
    res = least_squares(fun, z0 * (1 + 1e-4 * np.random.default_rng(0).normal(size=len(z0))), xtol=1e-15,
                        ftol=1e-15, gtol=1e-15, method="lm")
    assert abs(np.sum(res.fun ** 2) - out["cost"][1]) <= 1e-6 * out["cost"][1]
    c, X, s = unpack(res.x)
    np.testing.assert_allclose(c, c0, atol=1e-5 * np.abs(c0).max())
    np.testing.assert_allclose(X, X0, atol=1e-5 * np.abs(X0).max())
