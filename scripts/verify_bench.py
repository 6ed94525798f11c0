"""Geometric verification (cs_verify_pairs): call time over pair counts and trial counts, for both models.

Inputs: planted two-view correspondences (1920x1080, sigma 0.5 px, 40 % uniform outliers; a general scene for F, a
plane for H) at numPairs 1000, 5000 and 20000, each at numLoops 1024, 4096 and 16384, and the real pair list of two
synthetic 1920x1080 views rolled by (7, 11) px (ranked extraction N = 1000 -> cross-checked ratio matching) at 4096
trials.  Times are the medians of the call's own CUDA events (whole call: eight kernels and the result copy), every
configuration timed in alternation with the others.  The kernel split comes from the library's CUDASIFT_MATCH_TIMING
events, in a child process.  When cv2 imports, the same inputs go through cv2.findFundamentalMat / cv2.findHomography
(RANSAC, same threshold, maxIters = numLoops; OpenCV stops early once its confidence is reached) as a CPU comparison.
The card's name and power limit are read in the same run.  One JSON line on stdout.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from mutual_bench import card  # noqa: E402

PAIRS = (1000, 5000, 20000)
LOOPS = (1024, 4096, 16384)
MODELS = {"F": 2, "H": 1}
THRESH = 2.0


def make_inputs(cs):
    """{name: (model code, numLoops, s1, s2, pairs)}"""
    from test_verify_gpu import planted, _records, _shifted_views
    out = {}
    for mname, code in MODELS.items():
        for n in PAIRS:
            x1, x2, pairs, _, _, _ = planted(n, 7 + n, code == 1)
            for loops in LOOPS:
                out["%s_%d_%d" % (mname, n, loops)] = (code, loops, _records(cs, x1), _records(cs, x2), pairs)
    p1, p2 = _shifted_views(cs)
    pairs, _ = cs.match_ratio_host(p1, p2)
    for mname, code in MODELS.items():
        out["%s_ranked1000_4096" % mname] = (code, 4096, p1, p2, pairs)
    return out


def split_child(iters):
    """Runs with CUDASIFT_MATCH_TIMING=1: a few calls per input; the library prints the kernel split."""
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, (code, loops, s1, s2, pairs) in make_inputs(cs).items():
        for _ in range(iters):
            cs.verify_pairs_host(s1, s2, pairs, code, loops, THRESH, 0)
        sys.stderr.write("input %s\n" % name)
        sys.stderr.flush()


def parse_split(text):
    """{input: {kernel: median us}} from the child's stderr (the second half of each input's calls)."""
    out, rows = {}, []
    for line in text.splitlines():
        if line.startswith("verify timing"):
            toks = line.split("[us]:")[1].split()
            rows.append({toks[i]: float(toks[i + 1]) for i in range(0, len(toks), 2)})
        elif line.startswith("input "):
            keep = rows[len(rows) // 2:]
            out[line[6:].strip()] = {k: round(float(np.median([r[k] for r in keep])), 1) for k in keep[0]} if keep else {}
            rows = []
    return out


def cpu_comparison(inputs, reps):
    try:
        import cv2
    except ImportError:
        return {"skipped": "cv2 does not import"}
    res = {"threads": cv2.getNumThreads(), "opencv": cv2.__version__}
    for name, (code, loops, s1, s2, pairs) in inputs.items():
        a = np.column_stack([s1["xpos"][pairs[:, 0]], s1["ypos"][pairs[:, 0]]]).astype(np.float64)
        b = np.column_stack([s2["xpos"][pairs[:, 1]], s2["ypos"][pairs[:, 1]]]).astype(np.float64)
        ts, k = [], 0
        for _ in range(reps):
            t0 = time.perf_counter()
            if code == 2:
                _, mask = cv2.findFundamentalMat(a, b, cv2.FM_RANSAC, THRESH, 0.999, loops)
            else:
                _, mask = cv2.findHomography(a, b, cv2.RANSAC, THRESH, maxIters=loops, confidence=0.999)
            ts.append(1000.0 * (time.perf_counter() - t0))
            k = int(mask.sum()) if mask is not None else 0
        res[name] = {"ms": round(float(np.median(ts)), 3), "inliers": k}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--split-child", action="store_true")
    args = ap.parse_args()
    if args.split_child:
        split_child(args.iters)
        return
    import cudasift_b200 as cs
    cs.InitCuda(0)
    L = cs.lib()
    inputs = make_inputs(cs)
    dev = {}
    for name, (code, loops, s1, s2, pairs) in inputs.items():
        bufs = [cs.DeviceBuffer(s1.nbytes), cs.DeviceBuffer(s2.nbytes), cs.DeviceBuffer(pairs.nbytes),
                cs.DeviceBuffer(pairs.nbytes)]
        bufs[0].upload(s1)
        bufs[1].upload(s2)
        bufs[2].upload(np.ascontiguousarray(pairs, np.int32))
        dev[name] = bufs

    model = np.zeros(9)

    def call(name):
        code, loops, s1, s2, pairs = inputs[name]
        b = dev[name]
        ms = ctypes.c_double(0.0)
        k = L.cs_verify_pairs(b[0].ptr, len(s1), b[1].ptr, len(s2), b[2].ptr, len(pairs), code, loops, THRESH, 0,
                              model.ctypes.data, b[3].ptr, len(pairs), ctypes.byref(ms))
        assert k >= 0, L.cs_last_error()
        return ms.value, k

    found = {name: call(name)[1] for name in inputs}
    stats = {}
    for name in inputs:
        call(name)
        stats[name] = cs.verify_stats()
    for _ in range(args.warmup):
        for name in inputs:
            call(name)
    times = {name: [] for name in inputs}
    for _ in range(args.iters):
        for name in inputs:
            times[name].append(call(name)[0])

    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    child = subprocess.run([sys.executable, os.path.abspath(__file__), "--split-child", "--iters", "6"], env=env,
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=1800)
    split = parse_split(child.stderr) if child.returncode == 0 else {"error": child.stderr[-300:]}
    cpu = cpu_comparison(inputs, 3)

    out = {"metric": "cs_verify_pairs call time (ms, median of the call's CUDA events)", "card": card(),
           "thresh_px": THRESH, "iters": args.iters, "warmup": args.warmup, "inputs": {}}
    for name, (code, loops, s1, s2, pairs) in inputs.items():
        out["inputs"][name] = {"model": "F" if code == 2 else "H", "numPairs": len(pairs), "numLoops": loops,
                               "ms": round(float(np.median(times[name])), 4),
                               "ms_min": round(float(np.min(times[name])), 4), "inliers": found[name],
                               "stats": stats[name], "kernel_split_us": split.get(name, split),
                               "cpu_cv2": cpu.get(name, cpu)}
    out["cpu_cv2_threads"] = cpu.get("threads")
    for bufs in dev.values():
        for b in bufs:
            b.free()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
