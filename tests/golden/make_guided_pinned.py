#!/usr/bin/env python
"""Pinned bytes of guided matching: for seeded two-view sets, sha256 digests of the cs_match_knn2_guided lists and of
the cs_match_guided pairs (with and without the cross-check), with every cs_match_guided_stats quadruple.  The cases
cover F and H at 1, 4 and 16 px on planted 1 000 x 1 200 and 5 000 x 5 000 views, the three ways a row falls back to
scanning every candidate (a position beyond 1e12 px, |pw| < 1e-12 for H, a threshold of 1e5 px), non-finite positions
and models that admit nothing.  The equality tests compare with the CPU statement; this file pins the bits and the
statistics themselves, so a change to the kernels that moves a visit count or a last bit shows.

Runs on a GPU with whatever library CUDASIFT_B200_LIB names (else the tree's own build):

  python tests/golden/make_guided_pinned.py      -> tests/golden/guided_pinned.npz

tests/test_guided_pinned_gpu.py replays the stored cases and compares.
"""
import ctypes
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "guided_pinned.npz")
REC = 576
W, H_ = 1920, 1080
CODES = {"H": 1, "F": 2}


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _records(xy, seed):
    from cudasift_b200.synth import synth_descriptors
    r = synth_descriptors(len(xy), seed, sift_like=True)
    r["xpos"], r["ypos"] = xy[:, 0], xy[:, 1]
    return r


def _positions(n, seed):
    return np.random.default_rng(seed).uniform([0, 0], [W, H_], (n, 2))


def views(spec):
    """(s1, s2, model 3x3) of a view spec:
    ["planted", n1, n2, planar, seed]: test_guided_gpu.planted;
    ["far", n, seed, planar]: planted n x n views with one set-1 and one set-2 position moved beyond 1e12 px;
    ["tinypw", n, seed]: random positions under an H whose third row makes |pw| < 1e-12 everywhere;
    ["nonfinite", n, seed, planar]: planted n x n views, every 7th position NaN or infinite in both sets;
    ["nothing", n, seed, model]: random positions, set 2 the same shifted by 1 px, under a model that admits nothing
      (H: a translation by 1e6 px; F: only F[2][2] non-zero)."""
    from test_guided_gpu import planted
    kind = spec[0]
    if kind == "planted":
        _, n1, n2, planar, seed = spec
        s1, s2, M = planted(n1, n2, bool(planar), seed)
        return s1.copy(), s2.copy(), M
    if kind == "far":
        _, n, seed, planar = spec
        s1, s2, M = planted(n, n, bool(planar), seed)
        s1, s2 = s1.copy(), s2.copy()
        s1["xpos"][3] = 2e12
        s2["ypos"][5] = -3e12
        return s1, s2, M
    if kind == "tinypw":
        _, n, seed = spec
        p = _positions(n, seed).astype(np.float32)
        s1, s2 = _records(p, seed + 1), _records(p + 0.5, seed + 2)
        s2["data"] = s1["data"] * 0.8 + s2["data"] * 0.2
        return s1, s2, np.array([[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1e-13]])
    if kind == "nonfinite":
        _, n, seed, planar = spec
        s1, s2, M = planted(n, n, bool(planar), seed)
        s1, s2 = s1.copy(), s2.copy()
        for s, o in ((s1, 0), (s2, 3)):
            s["xpos"][o::7] = np.nan
            s["ypos"][o + 1::7] = np.inf
            s["xpos"][o + 2::7] = -np.inf
        return s1, s2, M
    if kind == "nothing":
        _, n, seed, model = spec
        p = _positions(n, seed).astype(np.float32)
        s1, s2 = _records(p, seed + 1), _records(p + 1.0, seed + 2)
        s2["data"] = s1["data"] * 0.8 + s2["data"] * 0.2
        M = np.array([[1, 0, 1e6], [0, 1, 0], [0, 0, 1.0]]) if model == "H" else np.diag([0, 0, 1.0])
        return s1, s2, M
    raise ValueError(spec)


class _Bufs:
    """Device buffers freed together."""

    def __init__(self, cs):
        self.cs, self.b = cs, []

    def new(self, nbytes, arr=None):
        d = self.cs.DeviceBuffer(max(int(nbytes), 8))
        self.b.append(d)
        if arr is not None and len(arr):
            d.upload(arr)
        return d

    def free(self):
        for d in self.b:
            d.free()


def run(cs, case):
    """The pinned outputs of one case: a dict of arrays."""
    L = cs.lib()
    s1, s2, M = views(case["views"])
    n1, n2 = len(s1), len(s2)
    m = np.ascontiguousarray(np.asarray(M, np.float64).reshape(9))
    code, t = CODES[case["model"]], float(case["t"])
    mp = m.ctypes.data_as(ctypes.c_void_p)
    bufs = _Bufs(cs)
    try:
        d1, d2 = bufs.new(REC * n1, s1), bufs.new(REC * n2, s2)
        out = {}
        if case["kind"] == "knn":
            di, ds = bufs.new(8 * n1), bufs.new(8 * n1)
            r = L.cs_match_knn2_guided(d1.ptr, n1, d2.ptr, n2, code, mp, t, di.ptr, ds.ptr, None)
            assert r == 0, L.cs_last_error()
            out["idx"] = np.array(_sha(di.download(np.int32, 2 * n1)))
            out["score"] = np.array(_sha(ds.download(np.float32, 2 * n1)))
        else:
            dp = bufs.new(8 * n1)
            k = L.cs_match_guided(d1.ptr, n1, d2.ptr, n2, code, mp, t, 0.8, 0.7, case["cross"], dp.ptr, n1, None)
            assert k >= 0, L.cs_last_error()
            out["count"] = np.int64(k)
            out["pairs"] = np.array(_sha(dp.download(np.int32, 2 * min(k, n1))))
        out["stats"] = np.array(cs.guided_stats(), np.uint64)
        return out
    finally:
        bufs.free()


def cases():
    specs = []
    for planar, model in ((0, "F"), (1, "H")):
        for n1, n2 in ((1000, 1200), (5000, 5000)):
            for t in (1.0, 4.0, 16.0):
                specs.append(("planted %dx%d" % (n1, n2), ["planted", n1, n2, planar, 11], model, t))
        specs.append(("beyond 1e12 px", ["far", 1500, 7, planar], model, 4.0))
        specs.append(("threshold 1e5", ["planted", 1000, 1200, planar, 11], model, 1e5))
        specs.append(("non-finite", ["nonfinite", 2000, 9, planar], model, 4.0))
        specs.append(("admits nothing", ["nothing", 800, 13, model], model, 4.0))
    specs.append(("|pw| < 1e-12", ["tinypw", 1200, 5], "H", 4.0))
    out = []
    for name, v, model, t in specs:
        base = {"name": name, "views": v, "model": model, "t": t}
        out.append(dict(base, kind="knn"))
        for cross in (0, 1):
            out.append(dict(base, kind="guided", cross=cross))
    return out


def main():
    import cudasift_b200 as cs
    cs.InitCuda(0)
    todo = cases()
    out = {"cases": np.array(json.dumps(todo))}
    for i, c in enumerate(todo):
        got = run(cs, c)
        for k, v in got.items():
            out["c%d_%s" % (i, k)] = v
        print(i, c["kind"], c["name"], c["model"], c["t"], c.get("cross", ""), int(got.get("count", -1)),
              [int(x) for x in got["stats"]])
    np.savez_compressed(OUT, **out)
    print("cases %d -> %s" % (len(todo), OUT))


if __name__ == "__main__":
    main()
