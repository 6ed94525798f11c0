"""CPU checks of triangulation (cs_triangulate_tracks): the entry point is declared, exported and typed, every invalid
argument is rejected with the offending set, camera or buffer named before any CUDA call, numTracks == 0 returns 0
without a device, the numpy statement (triangulate_oracle) recovers the points of noise-free scenes, its sampler replays
the header's formula and its Jacobi agrees with numpy's eigen-decomposition, and the Python wrapper builds its tables."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import triangulate_cases as tc
import triangulate_oracle as to
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_E_ARG = -2
RECORD = 576


def test_symbol_declared_exported_and_typed():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert "cs_triangulate_tracks" in declared and "cs_triangulate_tracks" in exported
    f = cs.lib().cs_triangulate_tracks
    assert f.restype is ctypes.c_int and len(f.argtypes) == 19
    assert f.argtypes[10] is ctypes.c_double and f.argtypes[11] is ctypes.c_double
    assert f.argtypes[12] is ctypes.c_ulonglong
    assert "TriangulateTracks" in cs.__all__ and callable(cs.TriangulateTracks)


class Arena:
    """Host memory laid out as on the device: two record sets of 4 records, the offsets (3 tracks), 8 members, then
    d_points, d_counts, d_errors and d_inlier, 8-byte aligned.  Nothing is dereferenced: every case fails its checks."""

    def __init__(self):
        self.buf = np.zeros(2 * 4 * RECORD + 16 + 64 + 72 + 16 + 32 + 8 + 64, np.uint8)
        base = self.buf.ctypes.data + (-self.buf.ctypes.data) % 16
        self.sets = [base, base + 4 * RECORD]
        o = base + 8 * RECORD
        self.offsets, self.members = o, o + 16
        self.points, self.counts = o + 80, o + 152
        self.errors, self.inlier = o + 168, o + 200

    def common(self):
        K = np.array([[800.0, 1.0, 640], [0, 790, 480], [0, 0, 1]])
        return dict(sets=[(self.sets[0], 4), (self.sets[1], 4)], Ks=np.stack([K, K]), Rs=np.stack([np.eye(3)] * 2),
                    ts=np.array([[0.0, 0, 0], [-1, 0, 0]]), offsets=self.offsets, numTracks=3, members=self.members,
                    numMembers=8, numTrials=64, maxError=4.0, minTriAngle=1.5, points=self.points,
                    counts=self.counts, errors=self.errors, inlier=self.inlier)


def _call(c):
    S = c.get("numImages", len(c["sets"]))
    sets = (cs.MatchSet * max(len(c["sets"]), 1))(*[cs.MatchSet(p, n) for p, n in c["sets"]])
    K, R, t = (np.ascontiguousarray(c[k], np.float64) for k in ("Ks", "Rs", "ts"))
    stats = np.full(8, 7, np.int64)
    ms = ctypes.c_double(-1.0)
    r = cs.lib().cs_triangulate_tracks(sets if c.get("setsPtr", 1) else None, S, K.ctypes.data if c.get("KPtr", 1) else None,
                                       R.ctypes.data, t.ctypes.data, c["offsets"], c["numTracks"], c["members"],
                                       c["numMembers"], c["numTrials"], c["maxError"], c["minTriAngle"], 5, c["points"],
                                       c["counts"], c["errors"], c["inlier"], stats.ctypes.data, ctypes.byref(ms))
    return r, ms.value, stats


def _expect(r, ms, stats, what, name):
    assert r == CS_E_ARG, (what, r)
    msg = cs.lib().cs_last_error().decode()
    assert "invalid argument" in msg and "CS_E_ARG" in msg, (what, msg)
    assert name in msg, (what, name, msg)
    assert ms == 0.0 and (stats == 7).all(), what


def test_rejects_every_invalid_argument():
    a = Arena()
    nan, inf = float("nan"), float("inf")

    def K(**kw):
        k = a.common()["Ks"].copy()
        for key, v in kw.items():
            k[1][int(key[1]) // 3, int(key[1]) % 3] = v
        return k

    def R(m):
        return np.stack([np.eye(3), m])

    rot = np.array([[0.0, -1, 0], [1, 0, 0], [0, 0, 1]])
    cases = [
        ("numImages < 0", dict(numImages=-1), "numImages"),
        ("numImages 2^24 + 1", dict(numImages=(1 << 24) + 1), "numImages"),
        ("numTracks < 0", dict(numTracks=-1), "numTracks"),
        ("numMembers < 0", dict(numMembers=-1), "numMembers"),
        ("NULL sets", dict(setsPtr=0), "sets"),
        ("NULL Ks", dict(KPtr=0), "Ks"),
        ("negative n", dict(sets=[(a.sets[0], 4), (a.sets[1], -1)]), "sets[1]"),
        ("NULL pts", dict(sets=[(None, 2), (a.sets[1], 4)]), "sets[0]"),
        ("K[8] != 1", dict(Ks=K(k8=2.0)), "Ks[1]"),
        ("K[3] != 0", dict(Ks=K(k3=0.5)), "Ks[1]"),
        ("K[0] <= 0", dict(Ks=K(k0=0.0)), "Ks[1]"),
        ("K not finite", dict(Ks=K(k2=nan)), "Ks[1]"),
        ("R not finite", dict(Rs=R(np.where(np.eye(3) > 0, inf, 0))), "Rs[1]"),
        ("R not orthonormal", dict(Rs=R(np.eye(3) * (1 + 3e-6))), "Rs[1]"),
        ("R a reflection", dict(Rs=R(np.diag([1.0, 1, -1]))), "Rs[1]"),
        ("t not finite", dict(ts=np.array([[0.0, 0, 0], [nan, 0, 0]])), "ts[1]"),
        ("numTrials 0", dict(numTrials=0), "numTrials"),
        ("numTrials 2^20 + 1", dict(numTrials=(1 << 20) + 1), "numTrials"),
        ("maxError 0", dict(maxError=0.0), "maxError"),
        ("maxError inf", dict(maxError=inf), "maxError"),
        ("maxError NaN", dict(maxError=nan), "maxError"),
        ("minTriAngle < 0", dict(minTriAngle=-1.0), "minTriAngle"),
        ("minTriAngle 180", dict(minTriAngle=180.0), "minTriAngle"),
        ("minTriAngle NaN", dict(minTriAngle=nan), "minTriAngle"),
        ("NULL offsets", dict(offsets=None), "d_offsets"),
        ("NULL points", dict(points=None), "d_points"),
        ("NULL counts", dict(counts=None), "d_counts"),
        ("NULL members", dict(members=None), "d_members"),
        ("offsets unaligned", dict(offsets=a.offsets + 2), "d_offsets"),
        ("errors unaligned", dict(errors=a.errors + 2), "d_errors"),
        ("points unaligned", dict(points=a.points + 4), "d_points"),
        ("members unaligned", dict(members=a.members + 4), "d_members"),
        ("points over counts", dict(points=a.counts - 16), "d_points and d_counts"),
        ("errors over inlier", dict(inlier=a.errors + 28), "d_errors and d_inlier"),
        ("inlier over members", dict(inlier=a.members + 60), "d_inlier and d_members"),
        ("counts over offsets", dict(counts=a.offsets + 12), "d_counts and d_offsets"),
        ("errors over a set", dict(errors=a.sets[1] + 4 * RECORD - 4), "d_errors and sets[1].pts"),
    ]
    for what, ch, name in cases:
        c = a.common()
        c.update(ch)
        _expect(*_call(c), what, name)
    assert not a.buf.any()
    # rotations pass; touching ranges pass; inputs may overlap each other (read only) -- and then numTracks == 0 stops
    c = a.common()
    c.update(Rs=R(rot), numTracks=0, members=a.sets[0], errors=None, inlier=None)
    r, ms, stats = _call(c)
    assert r == 0 and ms == 0.0 and not stats.any()


def test_no_tracks_returns_zero_before_any_cuda_call():
    ms = ctypes.c_double(-1.0)
    stats = np.full(8, 7, np.int64)
    L = cs.lib()
    assert L.cs_triangulate_tracks(None, 0, None, None, None, None, 0, None, 0, 256, 4.0, 1.5, 0, None, None, None, None,
                                   stats.ctypes.data, ctypes.byref(ms)) == 0
    assert ms.value == 0.0 and not stats.any()
    assert L.cs_triangulate_tracks(None, 0, None, None, None, None, 0, None, 0, 1, 0.5, 0.0, 0, None, None, None, None,
                                   None, None) == 0


@pytest.mark.parametrize("seed", range(3))
def test_oracle_recovers_noise_free_points(seed):
    """Without noise or outliers every track has a point with every member an inlier.  The records hold float32
    positions (about 6e-5 px of rounding at 1280 px), which moves a point by far less than 1e-6 of the scene scale."""
    xy, K, R, t, off, mem, X = tc.scene(seed, numImages=30, numTracks=120, lengths=(2, 20), noise=0.0,
                                        outliers=(0, 0), away=0)
    o = to.triangulate(xy, K, R, t, off, mem, numTrials=32, maxError=1.0)
    assert o["stats"][5] == 120 and (o["counts"] == np.diff(off)).all() and o["inlier"].all()
    assert np.abs(o["points"] - X).max() <= 1e-6 * tc.scale(K, R, t)
    assert (o["errors"] < 1e-3).all()
    assert o["stats"].tolist()[:3] == [120, 0, 0] and o["stats"][7] == len(mem)


def test_oracle_sampler_replays_the_header():
    M = (1 << 64) - 1

    def splitmix(z):
        z = (z + 0x9E3779B97F4A7C15) & M
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        return z ^ (z >> 31)

    for seed, k, V in ((0, 0, 3), (12345, 77, 100), (M, (1 << 31) - 1, 100000), (7, 5, 2)):
        s = np.arange(300)
        p, q, ok = to.draw(seed, k, s, V)
        for j in range(300):
            got = []
            for d in range(16):
                x = splitmix((seed + 0x9E3779B97F4A7C15 * ((k << 24) | (j << 4) | d)) & M)
                i = ((x >> 32) * V) >> 32
                if not got or (len(got) == 1 and i != got[0]):
                    got.append(i)
                if len(got) == 2:
                    break
            assert ok[j] == (len(got) == 2) and p[j] == got[0] and (not ok[j] or q[j] == got[1])


def test_oracle_jacobi_agrees_with_eigh():
    rng = np.random.default_rng(3)
    B = rng.normal(size=(500, 6, 4))
    A = np.einsum("bri,brj->bij", B, B)
    a, v = to.jacobi4(A)
    w = np.linalg.eigvalsh(A)
    assert np.allclose(np.sort(np.diagonal(a, axis1=1, axis2=2), 1), w, rtol=1e-12, atol=1e-12 * np.abs(w).max())
    assert np.allclose(np.einsum("bij,bjk->bik", A, v), v * np.diagonal(a, axis1=1, axis2=2)[:, None, :], atol=1e-10)


def test_oracle_rules_on_small_cases():
    """Two cameras one unit apart: a point seen by both, an invalid member of each kind, two members of one image, an
    empty track and a malformed one."""
    K = np.array([[800.0, 0, 640], [0, 800, 480], [0, 0, 1]])
    R = np.stack([np.eye(3)] * 2)
    t = np.array([[0.0, 0, 0], [-1.0, 0, 0]])
    X = np.array([0.2, -0.1, 6.0])
    p0, p1 = [tc.project(K, R[a], t[a], X) for a in range(2)]
    xy = [np.array([p0, [np.nan, 3.0], p0 + 50], np.float32), np.array([p1], np.float32)]
    offsets = [0, 6, 6, 9, 4]
    members = [[0, 0], [1, 0], [2, 0], [0, 3], [0, 1], [-1, 0], [0, 2], [0, 0], [1, 0]]
    o = to.triangulate(xy, [K, K], R, t, offsets, members, 16, 2.0, 1.5, 0)
    assert o["stats"].tolist() == [3, 1, 4, 4, 3, 2, 2, 4]
    assert np.abs(o["points"][[0, 2]] - X).max() < 1e-5 and np.isnan(o["points"][[1, 3]]).all()
    assert o["counts"].tolist() == [2, 0, 2, 0]
    assert o["inlier"].tolist() == [1, 1, 0, 0, 0, 0, 0, 1, 1]
    assert np.isnan(o["errors"][2:6]).all() and o["errors"][6] > 40


class _FakeLib:
    def __init__(self, found=3):
        self.calls, self.found, self.uploads = [], found, {}

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            if name == "cs_triangulate_tracks":
                S = args[1]
                sets = [cs.MatchSet.from_address(ctypes.addressof(args[0]) + k * ctypes.sizeof(cs.MatchSet))
                        for k in range(S)]
                self.sets = [(x.pts, x.n) for x in sets]
                self.cams = [np.ctypeslib.as_array((ctypes.c_double * (m * S)).from_address(args[i].value)).copy()
                             for i, m in ((2, 9), (3, 9), (4, 3))]
                return self.found
            if name == "cs_device_alloc":
                return 4096 * (1 + len(self.calls))
            if name == "cs_memcpy_h2d":
                self.uploads[args[0]] = ctypes.string_at(args[1].value, args[2])
            return 0
        return f


class _Data:
    def __init__(self, ptr, n):
        self.d_data, self.numPts = ptr, n


def test_wrapper_builds_its_tables(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    K = np.array([[800.0, 0, 640], [0, 800, 480], [0, 0, 1]])
    Rs = np.stack([np.eye(3), np.eye(3)[[1, 0, 2]] * [1, 1, -1]])
    offsets = np.array([0, 2, 5], np.int64)
    members = np.array([[0, 1], [1, 0], [0, 0], [1, 2], [1, 3]])
    pts, counts, errors, inlier, stats, ms = cs.TriangulateTracks([_Data(4096, 7), _Data(8192, 9)], K, Rs, [0, 0, 1],
                                                                  offsets, members, numTrials=16, maxError=2.5,
                                                                  minTriAngle=2.0, seed=11)
    (name, a), = [c for c in fake.calls if c[0] == "cs_triangulate_tracks"]
    assert fake.sets == [(4096, 7), (8192, 9)] and a[1] == 2
    assert np.array_equal(fake.cams[0], np.concatenate([K.ravel()] * 2))
    assert np.array_equal(fake.cams[1], Rs.ravel()) and np.array_equal(fake.cams[2], [0, 0, 1, 0, 0, 1])
    assert a[6] == 2 and a[8] == 5 and a[9:13] == (16, 2.5, 2.0, 11)
    assert fake.uploads[a[5]] == offsets.astype(np.int32).tobytes()
    assert fake.uploads[a[7]] == members.astype(np.int32).tobytes()
    assert pts.shape == (2, 3) and counts.shape == (2,) and errors.shape == (5,) and inlier.shape == (5,)
    assert pts.dtype == np.float64 and counts.dtype == np.int32 and errors.dtype == np.float32 and inlier.dtype == bool
    with pytest.raises(ValueError):
        cs.TriangulateTracks([_Data(4096, 7)] * 3, K, Rs, [0, 0, 1], offsets, members)
