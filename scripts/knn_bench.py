#!/usr/bin/env python
"""knn_bench.py -- two-nearest-neighbour matching (cs_match_knn2) and Lowe's ratio test (cs_match_ratio) against
MatchSiftData (cs_match) and mutual matching (cs_match_mutual).

  python scripts/knn_bench.py [--iters K] [--warmup W] [--repeats R]

Arms, for every size, timed alternately call by call in one process after W warm-up calls, on device-resident sets in
auto mode, outputs left on the device; the time is each call's CUDA events (*ms):
  match      cs_match(s1, s2)                   one direction, the reference's semantics
  mutual     cs_match_mutual(s1, s2)            both directions of match + the cross-checked pairs
  knn2       cs_match_knn2(s1, s2)              the true two nearest neighbours, one direction
  ratio      cs_match_ratio(s1, s2, 0.8, 0.7, crossCheck 0)
  ratio_cc   cs_match_ratio(s1, s2, 0.8, 0.7, crossCheck 1)
Sizes: synthetic descriptor sets of 2000 x 2000 and 10000 x 10000, and the records of two synthetic 1920x1080 views
(the second shifted by (7, 11) pixels) through a ranked extractor keeping N = 1000 and N = 4000 features.  Every knn
result is checked against the CPU statement (tests/knn_oracle.c) and every pair list against its numpy restatement.
Also measured: the exact fallback of a few rows against 10000 candidates (a mode-2 knn call on a set of 128 rows of
which 4 cannot be certified, minus the same call with none).  The kernel split comes from the library's
CUDASIFT_MATCH_TIMING events, in a child process.  The card's name and power limit are read in the same run.  One JSON
line on stdout.
"""
import argparse
import ctypes
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from mutual_bench import card, make_sets  # noqa: E402

ARMS = ("match", "mutual", "knn2", "ratio", "ratio_cc")


def split_child(iters):
    """Runs with CUDASIFT_MATCH_TIMING=1: a few knn2 and cross-checked ratio calls per size."""
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, (s1, s2, _) in make_sets(cs).items():
        for _ in range(iters):
            cs.match_knn2(s1, s2)
        for _ in range(iters):
            cs.match_ratio_host(s1, s2)
        sys.stderr.write("size %s\n" % name)
        sys.stderr.flush()


def parse_split(text):
    """{size: {"one-way": {kernel: median us}, "cross-check": {...}}} from the child's stderr."""
    out, rows = {}, {"one-way": [], "cross-check": []}
    for line in text.splitlines():
        m = re.match(r"knn timing \d+x\d+ \[us\]:(.*)", line)
        if m:
            toks = m.group(1).split()
            r = {toks[k]: float(toks[k + 1]) for k in range(0, len(toks), 2)}
            rows["cross-check" if "reverse-gemm" in r else "one-way"].append(r)
        elif line.startswith("size "):
            res = {}
            for kind, rs in rows.items():
                keep = rs[len(rs) // 2:]
                res[kind] = {k: round(float(np.median([r[k] for r in keep])), 1) for k in keep[0]} if keep else {}
            out[line[5:].strip()] = res
            rows = {"one-way": [], "cross-check": []}
    return out


def fallback_cost(cs, iters):
    """ms of a mode-2 knn call on 128 rows against 10000 candidates with 4 uncertifiable rows, minus the same call
    with none: what the sliced exact fallback costs for a few rows."""
    import knn_oracle
    from cudasift_b200.synth import synth_descriptors
    s2 = synth_descriptors(10000, 2)
    clean = synth_descriptors(128, 1)
    hard = clean.copy()
    s2["data"][64] = s2["data"][0]; s2["data"][128] = s2["data"][0]     # three equal group maxima in partition 0
    hard["data"][:4] = s2["data"][0] * 0.999 + hard["data"][:4] * 0.001
    L = cs.lib()
    bufs = {k: cs.DeviceBuffer(v.nbytes) for k, v in (("s2", s2), ("clean", clean), ("hard", hard))}
    for k, v in (("s2", s2), ("clean", clean), ("hard", hard)):
        bufs[k].upload(v)
    idx, sc = cs.DeviceBuffer(128 * 8), cs.DeviceBuffer(128 * 8)
    res, rows = {"clean": [], "hard": []}, {}
    for k in ("clean", "hard"):
        ms = ctypes.c_double(0.0)
        assert L.cs_match_knn2(bufs[k].ptr, 128, bufs["s2"].ptr, 10000, idx.ptr, sc.ptr, 2, ctypes.byref(ms)) == 0
        rows[k] = cs.match_stats()[2]
        wi, ws = knn_oracle.match_knn2(clean if k == "clean" else hard, s2)
        assert np.array_equal(idx.download(np.int32, 256).reshape(-1, 2), wi)
        assert sc.download(np.float32, 256).tobytes() == ws.tobytes()
    for _ in range(iters):
        for k in ("clean", "hard"):
            ms = ctypes.c_double(0.0)
            L.cs_match_knn2(bufs[k].ptr, 128, bufs["s2"].ptr, 10000, idx.ptr, sc.ptr, 2, ctypes.byref(ms))
            res[k].append(ms.value)
    for b in list(bufs.values()) + [idx, sc]:
        b.free()
    c, h = float(np.median(res["clean"])), float(np.median(res["hard"]))
    return {"fallback_rows": rows, "clean_ms": round(c, 4), "with_fallback_ms": round(h, 4),
            "fallback_ms": round(h - c, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--split-child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.split_child:
        split_child(args.iters)
        return
    import cudasift_b200 as cs
    import knn_oracle
    cs.InitCuda(0)
    L = cs.lib()
    sets = make_sets(cs)
    dev = {}
    for name, (s1, s2, _) in sets.items():
        d1, d2 = cs.DeviceBuffer(s1.nbytes), cs.DeviceBuffer(s2.nbytes)
        d1.upload(s1); d2.upload(s2)
        n1 = len(s1)
        dev[name] = dict(d1=d1, d2=d2, m1=cs.DeviceBuffer(s1.nbytes), m2=cs.DeviceBuffer(s2.nbytes),
                         idx=cs.DeviceBuffer(8 * n1), sc=cs.DeviceBuffer(8 * n1), pairs=cs.DeviceBuffer(8 * n1))
        dev[name]["m1"].upload(s1); dev[name]["m2"].upload(s2)

    def call(name, arm):
        d, n1, n2 = dev[name], len(sets[name][0]), len(sets[name][1])
        ms = ctypes.c_double(0.0)
        if arm == "match":
            r = L.cs_match(d["m1"].ptr, n1, d["d2"].ptr, n2, None, 0, ctypes.byref(ms))
        elif arm == "mutual":
            r = L.cs_match_mutual(d["m1"].ptr, n1, d["m2"].ptr, n2, 0.0, float("inf"), d["pairs"].ptr, n1, 0, ctypes.byref(ms))
        elif arm == "knn2":
            r = L.cs_match_knn2(d["d1"].ptr, n1, d["d2"].ptr, n2, d["idx"].ptr, d["sc"].ptr, 0, ctypes.byref(ms))
        else:
            r = L.cs_match_ratio(d["d1"].ptr, n1, d["d2"].ptr, n2, 0.8, 0.7, int(arm == "ratio_cc"), d["pairs"].ptr, n1, 0,
                                 ctypes.byref(ms))
        assert r >= 0, L.cs_last_error()
        return ms.value, r

    # correctness first, and the rows each call sends to the exact fallback
    checks, fallback_rows, pairs_found = {}, {}, {}
    for name, (s1, s2, _) in sets.items():
        k1, k2 = knn_oracle.match_knn2(s1, s2), knn_oracle.match_knn2(s2, s1)
        d = dev[name]
        call(name, "knn2")
        fallback_rows[name] = {"knn2": cs.match_stats()[2]}
        gi = d["idx"].download(np.int32, 2 * len(s1)).reshape(-1, 2)
        gs = d["sc"].download(np.float32, 2 * len(s1)).reshape(-1, 2)
        assert np.array_equal(gi, k1[0]) and gs.tobytes() == k1[1].tobytes(), name
        for arm, cc in (("ratio", 0), ("ratio_cc", 1)):
            _, k = call(name, arm)
            fallback_rows[name][arm] = cs.match_stats()[2]
            want, margin = knn_oracle.ratio_pairs(*k1, *k2, 0.8, 0.7, cc)
            got = d["pairs"].download(np.int32, 2 * k).reshape(-1, 2)
            assert np.array_equal(got, want), (name, arm)
            pairs_found.setdefault(name, {})[arm] = k
        checks[name] = "knn2 and ratio pairs equal the CPU statement"

    res = {name: {a: [] for a in ARMS} for name in sets}
    for rep in range(args.repeats):
        for name in sets:
            for _ in range(args.warmup):
                for a in ARMS:
                    call(name, a)
            for _ in range(args.iters):
                for a in ARMS:
                    res[name][a].append(call(name, a)[0])

    fb = fallback_cost(cs, max(args.iters, 10))
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    child = subprocess.run([sys.executable, os.path.abspath(__file__), "--split-child", "--iters", "10"], env=env,
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=1200)
    split = parse_split(child.stderr) if child.returncode == 0 else {"error": child.stderr[-300:]}

    out = {"metric": "two-nearest-neighbour matching: knn2 / ratio vs MatchSiftData / mutual (ms, median of CUDA events)",
           "card": card(), "iters": args.iters, "warmup": args.warmup, "repeats": args.repeats,
           "module_loading": os.environ.get("CUDA_MODULE_LOADING", "default"), "few_row_fallback_10000": fb, "sizes": {}}
    for name, (s1, s2, note) in sets.items():
        r = {a + "_ms": round(float(np.median(v)), 4) for a, v in res[name].items()}
        r.update({a + "_ms_min": round(float(np.min(v)), 4) for a, v in res[name].items()})
        r.update({"n1": len(s1), "n2": len(s2), "input": note, "pairs": pairs_found[name], "check": checks[name],
                  "knn2_over_match": round(r["knn2_ms"] / r["match_ms"], 3),
                  "ratio_cc_over_mutual": round(r["ratio_cc_ms"] / r["mutual_ms"], 3),
                  "fallback_rows": fallback_rows[name], "kernel_split_us": split.get(name, split)})
        out["sizes"][name] = r
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
