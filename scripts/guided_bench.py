#!/usr/bin/env python
"""guided_bench.py -- guided matching (cs_match_guided, cs_match_knn2_guided) against the unguided matchers.

  python scripts/guided_bench.py [--iters K] [--warmup W]

Inputs: planted two-view sets of 2000 x 2000 and 10000 x 10000 points in 1920x1080 views (half of them true
correspondences whose set-2 descriptor is a noisy copy, the rest random), and the two ranked (N = 1000) shifted views of
tests/test_verify_gpu.py; models F and H at 2, 4 and 16 px (for the planted sets the planted model, for the shifted
views the model VerifyPairs finds on the ratio pairs).
Arms, timed alternately call by call after W warm-up calls, on device-resident sets, outputs left on the device; the
time is each call's CUDA events (*ms):
  ratio_cc    cs_match_ratio(s1, s2, 0.8, 0.7, crossCheck 1)
  guided_cc   cs_match_guided(s1, s2, model, M, t, 0.8, 0.7, crossCheck 1)
  knn2        cs_match_knn2(s1, s2)
  knn2_guided cs_match_knn2_guided(s1, s2, model, M, t)
Reported: medians, the guided statistics and pair counts, and the kernel split of the guided calls
(CUDASIFT_MATCH_TIMING events, in a child process).  Every guided list of the 2000-point sets is checked against the
CPU statement (tests/guided_oracle.c).  The card's name and power limit are read in the same run.  One JSON line."""
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

from mutual_bench import card  # noqa: E402

ARMS = ("ratio_cc", "guided_cc", "knn2", "knn2_guided")
THRESHOLDS = (2.0, 4.0, 16.0)


def planted_sets(cs, n, seed):
    from cudasift_b200.synth import synth_descriptors
    from test_verify_cpu import planted_views
    rng = np.random.default_rng(seed)
    out = {}
    for name, planar in (("F", False), ("H", True)):
        m = n // 2
        x1, x2, F, H = planted_views(4 * m, seed, planar)
        ok = (x1 >= 0).all(1) & (x1 < [1920, 1080]).all(1) & (x2 >= 0).all(1) & (x2 < [1920, 1080]).all(1)
        x1, x2 = x1[ok][:m], x2[ok][:m] + rng.normal(0, 0.5, (m, 2))
        s1, s2 = synth_descriptors(n, seed + 1, sift_like=True), synth_descriptors(n, seed + 2, sift_like=True)
        s1["xpos"], s1["ypos"] = np.concatenate([x1, rng.uniform([0, 0], [1920, 1080], (n - m, 2))]).T.astype(np.float32)
        s2["xpos"], s2["ypos"] = np.concatenate([x2, rng.uniform([0, 0], [1920, 1080], (n - m, 2))]).T.astype(np.float32)
        s2["data"][:m] = s1["data"][:m] * 0.8 + s2["data"][:m] * 0.2
        out[name] = (s1, s2[rng.permutation(n)], H if planar else F)
    return out


def shifted_sets(cs):
    from test_verify_gpu import _shifted_views
    p1, p2 = _shifted_views(cs)
    pairs, _ = cs.match_ratio_host(p1, p2)
    Fm = cs.verify_pairs_host(p1, p2, pairs, "fundamental")[0]
    Hm = cs.verify_pairs_host(p1, p2, pairs, "homography")[0]
    return {"F": (p1, p2, Fm), "H": (p1, p2, Hm)}


def make_inputs(cs):
    inputs = {}
    for n in (2000, 10000):
        for model, v in planted_sets(cs, n, 5).items():
            inputs["planted%d_%s" % (n, model)] = v
    for model, v in shifted_sets(cs).items():
        inputs["shifted1000_%s" % model] = v
    return inputs


def split_child(iters):
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, (s1, s2, M) in make_inputs(cs).items():
        model = "fundamental" if name.endswith("F") else "homography"
        for _ in range(iters):
            cs.match_guided_host(s1, s2, model, M, 4.0)
        sys.stderr.write("input %s\n" % name)
        sys.stderr.flush()


def parse_split(text):
    """{input: {kernel: median us}} of the cross-checked guided calls at 4 px."""
    out, rows = {}, []
    for line in text.splitlines():
        m = re.match(r"guided timing \d+x\d+ \[us\]:(.*)", line)
        if m:
            toks = m.group(1).split()
            rows.append({toks[i]: float(toks[i + 1]) for i in range(0, len(toks), 2)})
        m = re.match(r"input (\S+)", line)
        if m:
            out[m.group(1)] = {k: float(np.median([r[k] for r in rows if k in r])) for k in rows[0]} if rows else {}
            rows = []
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--split-child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.split_child:
        split_child(args.iters)
        return
    import cudasift_b200 as cs
    import guided_oracle
    cs.InitCuda(0)
    L = cs.lib()
    inputs = make_inputs(cs)
    result = {"card": card(), "iters": args.iters, "warmup": args.warmup, "inputs": {}}
    for name, (s1, s2, M) in inputs.items():
        model = 2 if name.endswith("F") else 1
        n1, n2 = len(s1), len(s2)
        d1, d2 = cs.DeviceBuffer(s1.nbytes), cs.DeviceBuffer(s2.nbytes)
        d1.upload(s1)
        d2.upload(s2)
        idx, sc, pairs = cs.DeviceBuffer(8 * n1), cs.DeviceBuffer(8 * n1), cs.DeviceBuffer(8 * n1)
        m = np.ascontiguousarray(np.asarray(M, np.float64).reshape(9))
        entry = {}
        for t in THRESHOLDS:
            def call(arm):
                ms = ctypes.c_double(0.0)
                if arm == "ratio_cc":
                    r = L.cs_match_ratio(d1.ptr, n1, d2.ptr, n2, 0.8, 0.7, 1, pairs.ptr, n1, 0, ctypes.byref(ms))
                elif arm == "guided_cc":
                    r = L.cs_match_guided(d1.ptr, n1, d2.ptr, n2, model, m.ctypes.data, t, 0.8, 0.7, 1, pairs.ptr, n1,
                                          ctypes.byref(ms))
                elif arm == "knn2":
                    r = L.cs_match_knn2(d1.ptr, n1, d2.ptr, n2, idx.ptr, sc.ptr, 0, ctypes.byref(ms))
                else:
                    r = L.cs_match_knn2_guided(d1.ptr, n1, d2.ptr, n2, model, m.ctypes.data, t, idx.ptr, sc.ptr,
                                               ctypes.byref(ms))
                assert r >= 0, L.cs_last_error()
                return ms.value, r
            e = {}
            if n1 <= 2000:
                call("knn2_guided")
                gi = idx.download(np.int32, 2 * n1).reshape(-1, 2)
                gs = sc.download(np.float32, 2 * n1).reshape(-1, 2)
                wi, ws = guided_oracle.match_knn2_guided(s1, s2, model, M, t)
                assert np.array_equal(gi, wi) and gs.tobytes() == ws.tobytes(), (name, t)
                e["check"] = "knn2_guided equals the CPU statement"
            _, e["pairs_guided_cc"] = call("guided_cc")
            e["guided_stats_cc"] = cs.guided_stats()
            _, e["pairs_ratio_cc"] = call("ratio_cc")
            for _ in range(args.warmup):
                for arm in ARMS:
                    call(arm)
            times = {a: [] for a in ARMS}
            for _ in range(args.iters):
                for arm in ARMS:
                    times[arm].append(call(arm)[0])
            e["median_ms"] = {a: float(np.median(v)) for a, v in times.items()}
            entry["t%g" % t] = e
        result["inputs"][name] = entry
        for b in (d1, d2, idx, sc, pairs):
            b.free()
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    child = subprocess.run([sys.executable, os.path.abspath(__file__), "--split-child", "--iters", "10"], env=env,
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=1200)
    result["kernel_split_us_4px_cc"] = parse_split(child.stderr)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
