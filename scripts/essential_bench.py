"""Calibrated verification (cs_verify_essential): call time over pair counts and trial counts.

Inputs: planted calibrated two-view correspondences (1920x1080, the intrinsics of tests/test_essential_cpu.py, sideways
motion, sigma 0.5 px, 40 % uniform outliers) at numPairs 1000, 5000 and 20000, each at numLoops 1024, 4096 and 16384,
and the real pair list of two synthetic 1920x1080 views rolled by (7, 11) px (ranked extraction N = 1000 ->
cross-checked ratio matching) at 4096 trials, with K1 = K2 = [1400 0 960; 0 1400 540; 0 0 1].  Times are the medians
of the call's own CUDA events (whole call: eight kernels and the result copy), every configuration timed in alternation
with the others.  For comparison the same call to cs_verify_pairs with F is timed on the planted inputs.  The kernel
split comes from the library's CUDASIFT_MATCH_TIMING events, in a child process.  When cv2 imports, the same inputs go
through cv2.findEssentialMat (RANSAC, same threshold, maxIters = numLoops; OpenCV stops early once its confidence is
reached) + cv2.recoverPose as a CPU comparison.  The card's name and power limit are read in the same run.  Before
anything else the process measures the first essential call: the device memory it takes (cudaMemGetInfo through
torch, when torch imports) and its time against the second call, which shows the local memory the driver reserves for
the hypothesis kernel's per-thread stack and whether later calls pay for it again.  One JSON line on stdout.
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
from verify_bench import parse_split  # noqa: E402

PAIRS = (1000, 5000, 20000)
LOOPS = (1024, 4096, 16384)
THRESH = 2.0
K_SHIFTED = np.array([[1400.0, 0, 960], [0, 1400.0, 540], [0, 0, 1]])


def make_inputs(cs):
    """{name: (numLoops, s1, s2, pairs, K1, K2)}"""
    from test_essential_cpu import K1, K2
    from test_essential_gpu import planted, _recs
    from test_verify_gpu import _shifted_views
    out = {}
    for n in PAIRS:
        x1, x2, pairs, _, _, _, _ = planted(n, 7 + n)
        for loops in LOOPS:
            out["E_%d_%d" % (n, loops)] = (loops, _recs(cs, x1), _recs(cs, x2), pairs, K1, K2)
    p1, p2 = _shifted_views(cs)
    pairs, _ = cs.match_ratio_host(p1, p2)
    out["E_ranked1000_4096"] = (4096, p1, p2, pairs, K_SHIFTED, K_SHIFTED)
    return out


def split_child(iters):
    """Runs with CUDASIFT_MATCH_TIMING=1: a few calls per input; the library prints the kernel split."""
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, (loops, s1, s2, pairs, K1, K2) in make_inputs(cs).items():
        for _ in range(iters):
            cs.verify_essential_host(s1, s2, pairs, K1, K2, loops, THRESH, 0)
        sys.stderr.write("input %s\n" % name)
        sys.stderr.flush()


def cpu_comparison(inputs, reps):
    try:
        import cv2
    except ImportError:
        return {"skipped": "cv2 does not import"}
    res = {"threads": cv2.getNumThreads(), "opencv": cv2.__version__}
    for name, (loops, s1, s2, pairs, K1, K2) in inputs.items():
        a = np.column_stack([s1["xpos"][pairs[:, 0]], s1["ypos"][pairs[:, 0]]]).astype(np.float64)
        b = np.column_stack([s2["xpos"][pairs[:, 1]], s2["ypos"][pairs[:, 1]]]).astype(np.float64)
        a = cv2.undistortPoints(a.reshape(-1, 1, 2), K1, None, P=K2).reshape(-1, 2)   # one camera matrix for both views
        ts, k = [], 0
        for _ in range(reps):
            t0 = time.perf_counter()
            E, mask = cv2.findEssentialMat(a, b, K2, cv2.RANSAC, 0.999, THRESH, loops)
            if E is not None and E.shape == (3, 3):
                cv2.recoverPose(E, a, b, K2, mask=mask)
            ts.append(1000.0 * (time.perf_counter() - t0))
            k = int(mask.sum()) if mask is not None else 0
        res[name] = {"ms": round(float(np.median(ts)), 3), "inliers": k}
    return res


def first_call(cs, call, inputs):
    """Free device memory before and after the process's first essential call (after an F call has set up the
    verifier's scratch), and that call's time against the next three."""
    try:
        import torch
        free = lambda: torch.cuda.mem_get_info(0)[0]                     # noqa: E731
    except Exception:
        free = lambda: None                                              # noqa: E731
    name = min(inputs, key=lambda k: (len(inputs[k][3]), inputs[k][0]))
    call(name, False)
    call(name, False)
    cs.lib().cs_device_sync()
    before = free()
    t0 = call(name)[0]
    cs.lib().cs_device_sync()
    after = free()
    again = [call(name)[0] for _ in range(3)]
    cs.lib().cs_device_sync()
    return {"input": name, "first_ms": round(t0, 4), "next_ms": [round(t, 4) for t in again],
            "device_bytes_taken": (before - after) if before is not None else None,
            "device_bytes_after_next": (before - free()) if before is not None else None}


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
    for name, (loops, s1, s2, pairs, K1, K2) in inputs.items():
        bufs = [cs.DeviceBuffer(s1.nbytes), cs.DeviceBuffer(s2.nbytes), cs.DeviceBuffer(pairs.nbytes),
                cs.DeviceBuffer(pairs.nbytes)]
        bufs[0].upload(s1)
        bufs[1].upload(s2)
        bufs[2].upload(np.ascontiguousarray(pairs, np.int32))
        dev[name] = bufs
    E, R, t, model = np.zeros(9), np.zeros(9), np.zeros(3), np.zeros(9)

    def call(name, essential=True):
        loops, s1, s2, pairs, K1, K2 = inputs[name]
        b = dev[name]
        k1, k2 = np.ascontiguousarray(K1), np.ascontiguousarray(K2)
        ms = ctypes.c_double(0.0)
        if essential:
            k = L.cs_verify_essential(b[0].ptr, len(s1), b[1].ptr, len(s2), b[2].ptr, len(pairs), k1.ctypes.data,
                                      k2.ctypes.data, loops, THRESH, 0, E.ctypes.data, R.ctypes.data, t.ctypes.data,
                                      b[3].ptr, len(pairs), ctypes.byref(ms))
        else:
            k = L.cs_verify_pairs(b[0].ptr, len(s1), b[1].ptr, len(s2), b[2].ptr, len(pairs), 2, loops, THRESH, 0,
                                  model.ctypes.data, b[3].ptr, len(pairs), ctypes.byref(ms))
        assert k >= 0, L.cs_last_error()
        return ms.value, k

    first = first_call(cs, call, inputs)
    found = {name: call(name)[1] for name in inputs}
    stats = {}
    for name in inputs:
        call(name)
        stats[name] = cs.essential_stats()
    for _ in range(args.warmup):
        for name in inputs:
            call(name)
            call(name, False)
    times = {name: [] for name in inputs}
    ftimes = {name: [] for name in inputs}
    for _ in range(args.iters):
        for name in inputs:
            times[name].append(call(name)[0])
            ftimes[name].append(call(name, False)[0])

    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    child = subprocess.run([sys.executable, os.path.abspath(__file__), "--split-child", "--iters", "6"], env=env,
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=1800)
    split = parse_split(child.stderr) if child.returncode == 0 else {"error": child.stderr[-300:]}
    cpu = cpu_comparison(inputs, 3)

    out = {"metric": "cs_verify_essential call time (ms, median of the call's CUDA events)", "card": card(),
           "thresh_px": THRESH, "iters": args.iters, "warmup": args.warmup, "first_call": first, "inputs": {}}
    for name, (loops, s1, s2, pairs, K1, K2) in inputs.items():
        out["inputs"][name] = {"numPairs": len(pairs), "numLoops": loops,
                               "ms": round(float(np.median(times[name])), 4),
                               "ms_min": round(float(np.min(times[name])), 4),
                               "f_ms": round(float(np.median(ftimes[name])), 4), "inliers": found[name],
                               "stats": stats[name], "kernel_split_us": split.get(name, split),
                               "cpu_cv2": cpu.get(name, cpu)}
    out["cpu_cv2_threads"] = cpu.get("threads")
    for bufs in dev.values():
        for b in bufs:
            b.free()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
