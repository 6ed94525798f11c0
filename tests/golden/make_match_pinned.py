#!/usr/bin/env python
"""Pinned bytes of the tensor-core matcher: for seeded record sets, sha256 digests of every output of MatchSiftData
(cs_match mode 2: all five match fields), cs_match_mutual (both sets' fields and the pairs), cs_match_knn2 mode 2 (the
neighbour lists), cs_match_ratio mode 2 with and without the cross-check (the pairs) and cs_match_ratio_batch (every
job's pairs), with every cs_match_stats quadruple and the batch's per-job statistics.  The sizes cover candidate counts
that are not multiples of 32 or 128, fewer than 32 candidates, a set tail that needs its own B-role copy in a mutual
match, one row tile against 60 000 candidates (more segments than the resolve's unrolled merge), rows that cannot be
certified (tests/test_knn_gpu.py's triplicates) and the bad-input gate, in a single call and in one job of a batch.
The equality tests compare with other paths or a CPU statement; this file pins the bits themselves, so a change to the
resolve that moves a statistic or a last bit shows.

Runs on a GPU with whatever library CUDASIFT_B200_LIB names (else the tree's own build):

  python tests/golden/make_match_pinned.py      -> tests/golden/match_pinned.npz

tests/test_match_pinned_gpu.py replays the stored cases and compares.
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
OUT = os.path.join(ROOT, "tests", "golden", "match_pinned.npz")
REC = 576


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def records(spec):
    """The record array of a set spec:
    ["synth", n, seed, sift_like]; ["near", n, seed, n0, seed0, k]: sift-like, its first k rows close to those of
    ["synth", n0, seed0, 1]; ["trip", side]: one side of the triplicates; ["big", n, seed]: one value at 8.0 (gated)."""
    from cudasift_b200.synth import synth_descriptors
    kind = spec[0]
    if kind == "synth":
        return synth_descriptors(spec[1], spec[2], sift_like=bool(spec[3]))
    if kind == "near":
        _, n, seed, n0, seed0, k = spec
        a, b = synth_descriptors(n0, seed0, sift_like=True), synth_descriptors(n, seed, sift_like=True)
        b["data"][:k] = a["data"][:k] * 0.9 + b["data"][:k] * 0.1
        return b
    if kind == "trip":
        from test_knn_gpu import _triplicates
        return _triplicates()[spec[1]]
    if kind == "big":
        s = synth_descriptors(spec[1], spec[2])
        s["data"][5, 17] = 8.0
        return s
    if kind == "empty":
        return synth_descriptors(1, 0)[:0]
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
    kind = case["kind"]
    bufs = _Bufs(cs)
    try:
        if kind == "batch":
            arrays = [records(s) for s in case["sets"]]
            dsets = [bufs.new(REC * len(a), a) for a in arrays]
            st = (cs.MatchSet * len(arrays))(*[cs.MatchSet(d.ptr if len(a) else None, len(a))
                                                 for d, a in zip(dsets, arrays)])
            room = [max(len(arrays[a]), 1) for a, _ in case["jobs"]]
            dp = [bufs.new(8 * m) for m in room]
            jt = (cs.MatchJob * len(room))(*[cs.MatchJob(a, b, d.ptr, m) for (a, b), d, m in zip(case["jobs"], dp, room)])
            counts, stats = np.full(len(room), -1, np.int32), np.zeros((len(room), 4), np.uint64)
            r = L.cs_match_ratio_batch(st, len(arrays), jt, len(room), case["ratio"], case["dist"], case["cross"],
                                       counts.ctypes.data, stats.ctypes.data, None)
            assert r == 0, L.cs_last_error()
            pairs = [d.download(np.int32, 2 * min(int(k), m)) for d, k, m in zip(dp, counts, room)]
            return {"counts": counts, "pairs": np.array([_sha(p) for p in pairs]), "stats": stats}
        s1, s2 = records(case["s1"]), records(case["s2"])
        n1, n2 = len(s1), len(s2)
        d1, d2 = bufs.new(REC * n1, s1), bufs.new(REC * n2, s2)
        out = {}
        if kind == "match":
            assert L.cs_match(d1.ptr, n1, d2.ptr, n2, None, 2, None) == 0, L.cs_last_error()
            out["s1"] = np.array(_sha(d1.download(s1.dtype, n1)))
        elif kind == "mutual":
            dp = bufs.new(8 * min(n1, n2))
            k = L.cs_match_mutual(d1.ptr, n1, d2.ptr, n2, 0.0, float("inf"), dp.ptr, min(n1, n2), 2, None)
            assert k >= 0, L.cs_last_error()
            out["s1"] = np.array(_sha(d1.download(s1.dtype, n1)))
            out["s2"] = np.array(_sha(d2.download(s2.dtype, n2)))
            out["count"] = np.int64(k)
            out["pairs"] = np.array(_sha(dp.download(np.int32, 2 * k)))
        elif kind == "knn":
            di, ds = bufs.new(8 * n1), bufs.new(8 * n1)
            assert L.cs_match_knn2(d1.ptr, n1, d2.ptr, n2, di.ptr, ds.ptr, 2, None) == 0, L.cs_last_error()
            out["idx"] = np.array(_sha(di.download(np.int32, 2 * n1)))
            out["score"] = np.array(_sha(ds.download(np.float32, 2 * n1)))
        elif kind == "ratio":
            dp = bufs.new(8 * n1)
            k = L.cs_match_ratio(d1.ptr, n1, d2.ptr, n2, case["ratio"], case["dist"], case["cross"], dp.ptr, n1, 2, None)
            assert k >= 0, L.cs_last_error()
            out["count"] = np.int64(k)
            out["pairs"] = np.array(_sha(dp.download(np.int32, 2 * min(k, n1))))
        else:
            raise ValueError(kind)
        out["stats"] = np.array(cs.match_stats(), np.uint64)
        return out
    finally:
        bufs.free()


# the record sets of the single calls: (set 1, set 2)
SYN = lambda n, seed, sl=0: ["synth", n, seed, sl]
PAIRS = {
    "1000x1037": (SYN(1000, 1, 1), ["near", 1037, 2, 1000, 1, 400]),
    "2003x517": (SYN(2003, 3), SYN(517, 4)),
    "300x20": (SYN(300, 5), SYN(20, 6)),
    "100x60000": (SYN(100, 7, 1), ["near", 60000, 8, 100, 7, 50]),
    "triplicates": (["trip", 0], ["trip", 1]),
    "gate": (SYN(600, 11), ["big", 700, 12]),
}


def cases():
    out = []
    for kind, names in (("match", list(PAIRS)), ("mutual", ["1000x1037", "2003x517", "100x60000", "triplicates", "gate"]),
                        ("knn", list(PAIRS))):
        out += [{"kind": kind, "name": k, "s1": PAIRS[k][0], "s2": PAIRS[k][1]} for k in names]
    for cross in (0, 1):
        for k in ("1000x1037", "2003x517", "100x60000", "triplicates", "gate"):
            out.append({"kind": "ratio", "name": k, "s1": PAIRS[k][0], "s2": PAIRS[k][1], "ratio": 0.8, "dist": 0.7,
                        "cross": cross})
    # shared sets, a set against itself, a repeated job, empty sets, the triplicates, one gated job and 100 x 60 000
    sets = [SYN(1000, 1, 1), ["near", 1037, 2, 1000, 1, 400], SYN(2003, 3), SYN(517, 4), ["trip", 0], ["trip", 1],
            ["big", 700, 12], SYN(600, 11), ["empty"], SYN(100, 7, 1), ["near", 60000, 8, 100, 7, 50], SYN(20, 6)]
    jobs = [[0, 1], [1, 0], [2, 3], [0, 0], [4, 5], [5, 4], [7, 6], [8, 0], [0, 8], [9, 10], [2, 2], [11, 3], [0, 1]]
    for cross in (0, 1):
        out.append({"kind": "batch", "name": "mixed", "sets": sets, "jobs": jobs, "ratio": 0.8, "dist": 0.7,
                    "cross": cross})
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
        print(i, c["kind"], c["name"], c.get("cross", ""), [int(x) for x in np.ravel(got["stats"])[:8]])
    np.savez_compressed(OUT, **out)
    print("cases %d -> %s" % (len(todo), OUT))


if __name__ == "__main__":
    main()
