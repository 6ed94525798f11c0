#!/usr/bin/env python
"""mutual_bench.py -- one-call mutual matching (cs_match_mutual) against the two-call path it replaces.

  python scripts/mutual_bench.py [--iters K] [--warmup W] [--repeats R]

Arms, for every size, timed alternately in one process after W warm-up calls:
  single     cs_match(s1, s2) and, as its own arm, cs_match(s2, s1) on device-resident sets (auto mode), no host
             copy: the one-directional baselines; with the rows each direction sends to the exact fallback.
  mutual     cs_match_mutual on device-resident sets (auto mode), pairs left on the device; device time = the call's
             CUDA events (*ms).
  two-call   cs_match(s1, s2) and cs_match(s2, s1), each copying its set's five match fields to the host (*ms of both
             calls), then the cross-check in numpy on the host (wall time).
Sizes: synthetic descriptor sets of 2000 x 2000 and 10000 x 10000, and the records of two synthetic 1920x1080 views
(the second shifted by (7, 11) pixels) through a ranked extractor keeping N = 1000 and N = 4000 features (the detector
threshold is lowered until N features are found).  Every mutual result is checked against the two-call result.
The kernel split (prep, GEMM and resolve per direction, exact fallback, pairs) comes from the library's
CUDASIFT_MATCH_TIMING events, in a child process so that those events do not disturb the timed arms.  The card's name
and power limit are read in the same run.  One JSON line on stdout.
"""
import argparse
import ctypes
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FIELDS = ("score", "ambiguity", "match", "match_xpos", "match_ypos")
W, H = 1920, 1080


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:
        return {"error": str(e)[:80]}


def cross_check(a, b):
    i = np.arange(len(a))
    j = a["match"]
    ok = (j >= 0) & (j < len(b))
    ok &= b["match"][np.where(ok, j, 0)] == i
    return np.stack([i[ok], j[ok]], axis=1).astype(np.int32)


def make_sets(cs):
    """{name: (s1, s2, note)}"""
    from cudasift_b200.synth import synth_descriptors, synth_image
    sets = {"2000x2000": (synth_descriptors(2000, 1), synth_descriptors(2000, 2), "synthetic descriptors"),
            "10000x10000": (synth_descriptors(10000, 1), synth_descriptors(10000, 2), "synthetic descriptors")}
    img = synth_image(W, H, seed=1000)
    views = [img, np.ascontiguousarray(np.roll(img, (7, 11), axis=(0, 1)))]
    dimgs = []
    for v in views:
        ci = cs.CudaImage()
        ci.Allocate(W, H, hostMem=v)
        ci.Download()
        dimgs.append(ci)
    for n in (1000, 4000):
        ex = cs.Extractor(W, H, 5, n, False, maxCandidates=32768)
        for thresh in (3.0, 2.0, 1.5, 1.0, 0.75, 0.5):
            recs = []
            for ci in dimgs:
                ex.submit_device(ci.d_data, ci.pitch, 1.0, thresh, 0.0)
                recs.append(ex.device_points_at(0, ex.wait()))
            if min(len(r) for r in recs) == n:
                break
        ex.close()
        sets["ranked_%d" % n] = (recs[0], recs[1], "ranked extraction, 1920x1080 views, thresh %g" % thresh)
    return sets


def split_child(iters):
    """Runs with CUDASIFT_MATCH_TIMING=1: a few mutual calls per size; the library prints the kernel split."""
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, (s1, s2, _) in make_sets(cs).items():
        for _ in range(iters):
            cs.match_mutual_host(s1, s2)
        sys.stderr.write("size %s\n" % name)
        sys.stderr.flush()


def parse_split(text):
    """{size: {kernel: median us}} from the child's stderr."""
    out, rows = {}, []
    for line in text.splitlines():
        m = re.match(r"mutual timing \d+x\d+ \[us\]:(.*)", line)
        if m:
            toks = m.group(1).split()
            rows.append({toks[k]: float(toks[k + 1]) for k in range(0, len(toks), 2)})
        elif line.startswith("size "):
            keep = rows[len(rows) // 2:]                 # the later half: warm
            out[line[5:].strip()] = {k: round(float(np.median([r[k] for r in keep])), 1) for k in keep[0]} if keep else {}
            rows = []
    return out


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
    cs.InitCuda(0)
    L = cs.lib()
    sets = make_sets(cs)
    dev = {}
    for name, (s1, s2, _) in sets.items():
        d1, d2 = cs.DeviceBuffer(s1.nbytes), cs.DeviceBuffer(s2.nbytes)
        d1.upload(s1); d2.upload(s2)
        room = min(len(s1), len(s2))
        dp = cs.DeviceBuffer(max(room, 1) * 8)
        h1, h2 = s1.copy(), s2.copy()
        dev[name] = (d1, d2, dp, room, h1, h2)

    def mutual(name):
        d1, d2, dp, room, _, _ = dev[name]
        n1, n2 = len(sets[name][0]), len(sets[name][1])
        ms = ctypes.c_double(0.0)
        t0 = time.perf_counter()
        k = L.cs_match_mutual(d1.ptr, n1, d2.ptr, n2, 0.0, float("inf"), dp.ptr, room, 0, ctypes.byref(ms))
        wall = (time.perf_counter() - t0) * 1e3
        assert k >= 0, L.cs_last_error()
        return ms.value, wall, k

    def two_call(name):
        d1, d2, _, _, h1, h2 = dev[name]
        n1, n2 = len(h1), len(h2)
        m1, m2 = ctypes.c_double(0.0), ctypes.c_double(0.0)
        t0 = time.perf_counter()
        assert L.cs_match(d1.ptr, n1, d2.ptr, n2, h1.ctypes.data, 0, ctypes.byref(m1)) >= 0
        assert L.cs_match(d2.ptr, n2, d1.ptr, n1, h2.ctypes.data, 0, ctypes.byref(m2)) >= 0
        t1 = time.perf_counter()
        pairs = cross_check(h1, h2)
        t2 = time.perf_counter()
        return m1.value + m2.value + (t2 - t1) * 1e3, (t2 - t0) * 1e3, (t2 - t1) * 1e3, pairs

    def single(name, reverse=False):
        d1, d2 = dev[name][0], dev[name][1]
        n1, n2 = len(sets[name][0]), len(sets[name][1])
        if reverse:
            d1, d2, n1, n2 = d2, d1, n2, n1
        ms = ctypes.c_double(0.0)
        assert L.cs_match(d1.ptr, n1, d2.ptr, n2, None, 0, ctypes.byref(ms)) >= 0
        return ms.value

    # correctness first: the mutual call's fields and pairs against the two-call path
    for name in sets:
        _, _, _, want = two_call(name)
        s1, s2, _ = sets[name]
        g1, g2, pairs, _ = cs.match_mutual_host(s1, s2)
        h1, h2 = dev[name][4], dev[name][5]
        assert all(g1[f].tobytes() == h1[f].tobytes() for f in FIELDS), name
        assert all(g2[f].tobytes() == h2[f].tobytes() for f in FIELDS), name
        assert np.array_equal(pairs, want), name

    res = {name: {"mutual_ms": [], "mutual_wall_ms": [], "two_call_ms": [], "two_call_wall_ms": [], "single_ms": [],
                  "single_reverse_ms": [], "host_check_ms": []} for name in sets}
    pairs_found, fallback_rows = {}, {}
    for name in sets:                                    # rows each direction sends to the exact fallback
        fallback_rows[name] = []
        for rev in (False, True):
            single(name, rev)
            fallback_rows[name].append(cs.match_stats()[2])
    for rep in range(args.repeats):
        for name in sets:
            for _ in range(args.warmup):
                mutual(name); two_call(name); single(name); single(name, True)
            for _ in range(args.iters):                  # the arms alternate call by call
                ms, wall, k = mutual(name)
                res[name]["mutual_ms"].append(ms); res[name]["mutual_wall_ms"].append(wall)
                pairs_found[name] = k
                ms, wall, host, _ = two_call(name)
                res[name]["two_call_ms"].append(ms); res[name]["two_call_wall_ms"].append(wall)
                res[name]["host_check_ms"].append(host)
                res[name]["single_ms"].append(single(name))
                res[name]["single_reverse_ms"].append(single(name, True))

    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    child = subprocess.run([sys.executable, os.path.abspath(__file__), "--split-child", "--iters", "10"], env=env,
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=1200)
    split = parse_split(child.stderr) if child.returncode == 0 else {"error": child.stderr[-300:]}

    out = {"metric": "mutual matching: cs_match_mutual vs cs_match both ways + host cross-check (ms, median)",
           "card": card(), "iters": args.iters, "warmup": args.warmup, "repeats": args.repeats,
           "module_loading": os.environ.get("CUDA_MODULE_LOADING", "default"), "sizes": {}}
    for name, (s1, s2, note) in sets.items():
        r = {k: round(float(np.median(v)), 4) for k, v in res[name].items()}
        r.update({"n1": len(s1), "n2": len(s2), "input": note, "pairs": pairs_found[name],
                  "mutual_over_single": round(r["mutual_ms"] / r["single_ms"], 3),
                  "mutual_over_two_call": round(r["mutual_ms"] / r["two_call_ms"], 3),
                  "mutual_over_both_singles": round(r["mutual_ms"] / (r["single_ms"] + r["single_reverse_ms"]), 3),
                  "fallback_rows_forward_reverse": fallback_rows[name],
                  "mutual_ms_min": round(float(np.min(res[name]["mutual_ms"])), 4),
                  "mutual_ms_max": round(float(np.max(res[name]["mutual_ms"])), 4),
                  "kernel_split_us": split.get(name, split)})
        out["sizes"][name] = r
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
