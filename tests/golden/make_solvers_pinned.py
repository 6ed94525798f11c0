#!/usr/bin/env python
"""Pinned bytes of the three cooperative solvers: for a fixed set of scenes, sha256 digests of every output plus the
costs and statistics of cs_bundle_adjust and cs_bundle_adjust_intrinsics (every instantiation of the kernel: camera
block 6 or 9, trivial or robust loss, with per-member errors and inlier bytes), cs_rotation_averaging (the squared loss
and Geman-McClure at 5 degrees) and cs_global_positioning (trivial and Cauchy).  The oracle tests compare to a
tolerance and cannot see a changed last bit; this file can.

Runs on a GPU with whatever library CUDASIFT_B200_LIB names (else the tree's own build):

  python tests/golden/make_solvers_pinned.py      -> tests/golden/solvers_pinned.npz

tests/test_solvers_pinned_gpu.py replays the stored cases and compares.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "solvers_pinned.npz")


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class _Records:
    """One image's records (positions only) in device memory, as the wrappers take them (d_data, numPts)."""

    def __init__(self, cs, p):
        from cudasift_b200.records import SIFT_DTYPE
        rec = np.zeros(len(p), SIFT_DTYPE)
        rec["xpos"], rec["ypos"] = p[:, 0], p[:, 1]
        self.buf = cs.DeviceBuffer(max(rec.nbytes, 8))
        if len(p):
            self.buf.upload(rec)
        self.d_data, self.numPts = self.buf.ptr, len(p)


def _digests(names, outs, raw):
    """{name: sha256 of the output} for every output, and the outputs named in raw kept as they are."""
    out = {}
    for n, v in zip(names, outs):
        v = np.asarray(v)
        out[n] = v if n in raw else np.array(_sha(v))
    return out


def _bundle(cs, c):
    import bundle_cases as bc
    import bundle_intrinsics_cases as bic
    s = bic.scene(c["seed"], noise=0.5, outlier=0.1) if c["scene"] == "intrinsics" else bc.scene(c["seed"])
    K = s["K0"] if c["scene"] == "intrinsics" else s["K"]
    datas = [_Records(cs, p) for p in s["xy"]]
    try:
        common = dict(use=s["use"], maxIterations=c["maxIterations"])
        if c["call"] == "plain":
            r = cs.BundleAdjust(datas, K, s["R0"], s["t0"], s["offsets"], s["members"], s["X0"], **common)
            names = ("R", "t", "points", "errors", "inlier", "cost", "trace", "stats")
        else:
            r = cs.BundleAdjustIntrinsics(datas, K, s["R0"], s["t0"], s["offsets"], s["members"], s["X0"],
                                          refine=c["refine"], loss=c["loss"], lossScale=2.0, **common)
            names = ("K", "dists", "R", "t", "points", "errors", "inlier", "cost", "trace", "stats")
    finally:
        for d in datas:
            d.buf.free()
    outs = [np.asarray(v).view(np.uint8) if n == "inlier" else v for n, v in zip(names, r)]
    return _digests(names, outs, ("cost", "stats"))


def _rotavg(cs, c):
    import global_cases as gc
    g = gc.view_graph(c["seed"], c["numImages"], neighbours=8, noiseDeg=0.3, outliers=0.1)
    r = cs.RotationAveraging(c["numImages"], g["edges"], g["Rrel"], g["weights"], sigmaDeg=c["sigmaDeg"],
                             maxIterations=c["maxIterations"])
    names = ("R", "residuals", "inlier", "cost", "trace", "stats")
    outs = [np.asarray(v).view(np.uint8) if n == "inlier" else v for n, v in zip(names, r[:6])]
    return _digests(names, outs, ("cost", "stats"))


def _globalpos(cs, c):
    import triangulate_cases as tc
    xy, Ks, Rs, ts, off, mem, pts = tc.scene(c["seed"], numImages=c["numImages"], numTracks=c["numTracks"],
                                             lengths=(3, 8), noise=0.5, outliers=(0.0, 0.0), away=0)
    datas = [_Records(cs, p) for p in xy]
    try:
        r = cs.GlobalPositioning(datas, Ks, Rs, off, mem, seed=c["seed"], loss=c["loss"], lossScale=0.01,
                                 maxIterations=c["maxIterations"])
    finally:
        for d in datas:
            d.buf.free()
    names = ("t", "points", "cost", "trace", "stats")
    return _digests(names, r[:5], ("cost", "stats"))


RUN = {"bundle": _bundle, "rotavg": _rotavg, "globalpos": _globalpos}


def run(cs, c):
    """The pinned outputs of one case: a digest of every output, its costs and statistics as they are."""
    return RUN[c["solver"]](cs, c)


def cases():
    b = [dict(solver="bundle", call="plain", scene="bundle", seed=s, maxIterations=30) for s in (1, 2)]
    b += [dict(solver="bundle", call="intrinsics", scene=sc, seed=s, refine=ref, loss=loss, maxIterations=30)
          for sc, s, ref, loss in (("bundle", 3, 0, "cauchy"),          # <6, true>
                                   ("bundle", 4, 0, "soft_l1"),         # <6, true>
                                   ("intrinsics", 5, 3, "trivial"),     # <9, false>
                                   ("intrinsics", 6, 7, "trivial"),     # <9, false>
                                   ("intrinsics", 5, 3, "cauchy"),      # <9, true>
                                   ("intrinsics", 7, 1, "soft_l1"))]    # <9, true>
    r = [dict(solver="rotavg", seed=s, numImages=n, sigmaDeg=sig, maxIterations=10)
         for s, n in ((11, 40), (12, 300)) for sig in (0.0, 5.0)]
    g = [dict(solver="globalpos", seed=s, numImages=n, numTracks=t, loss=loss, maxIterations=15)
         for s, n, t in ((31, 20, 150), (32, 200, 1500)) for loss in ("trivial", "cauchy")]
    return b + r + g


def main():
    import cudasift_b200 as cs
    cs.InitCuda(0)
    cs_ = cases()
    out = {"cases": np.array(json.dumps(cs_))}
    for i, c in enumerate(cs_):
        for k, v in run(cs, c).items():
            out["c%d_%s" % (i, k)] = v
        print(i, c, "cost", out["c%d_cost" % i], "stats", out["c%d_stats" % i])
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
