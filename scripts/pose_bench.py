#!/usr/bin/env python
"""Camera registration (cs_absolute_pose_batch) on the GPU: call time and images/s, the kernel split, a host arm and
the pose agreement with it, on synthetic scenes (tests/pose_cases.py: skewed, unequal K, 0.5 px noise).

  (a) 64 images x 2 000 correspondences, 30 % outliers, numLoops 1 024
  (b) 1 000 images x 500 correspondences, 30 % outliers, numLoops 1 024 (a localization batch)
  (c) one image of 1 000 correspondences, 30 % outliers, numLoops 1 024 (the latency of registering one new view)

The median of the call's event time over `--reps` calls after warm-up; the card's name and power limit are read in the
same run.  --profile runs a child process under torch.profiler for the kernel split.  The host arm is
cv2.solvePnPRansac (same maxError, 1 024 iterations, confidence 0.999999) when OpenCV is importable, else the float64
statement on a timed subset, extrapolated and labelled as such.  Writes one JSON line (and --out FILE)."""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

WORKLOADS = {"a": (64, 2000, 0.3), "b": (1000, 500, 0.3), "c": (1, 1000, 0.3)}
LOOPS, MAXERR = 1024, 4.0


def scene(name):
    import pose_cases as pc
    J, V, out = WORKLOADS[name]
    return pc.batch(100 + ord(name), [V] * J, noise=0.5, outliers=(out, out))


class Data:
    def __init__(self, cs, xy):
        import pose_cases as pc
        self.buf = cs.DeviceBuffer(len(xy) * 576)
        self.buf.upload(pc.records(xy))
        self.d_data, self.numPts = self.buf.ptr, len(xy)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception as e:
        return "unknown (%s)" % str(e)[:40]


def run_gpu(name, reps):
    import cudasift_b200 as cs
    cs.InitCuda(0)
    xys, pofs, pts, Ks, Rs, ts = scene(name)
    datas = [Data(cs, xy) for xy in xys]
    for _ in range(3):
        cs.AbsolutePoseBatch(datas, pofs, pts, Ks, LOOPS, MAXERR)
    ms = []
    for _ in range(reps):
        R, t, counts, _, _, stats, m = cs.AbsolutePoseBatch(datas, pofs, pts, Ks, LOOPS, MAXERR)
        ms.append(m)
    med = float(np.median(ms))
    J = len(xys)
    rerr = [float(np.abs(R[p] - Rs[p]).max()) for p in range(J)]
    return dict(jobs=J, correspondences=len(xys[0]), ms_median=round(med, 4), ms_min=round(min(ms), 4),
                images_per_s=round(J / (med * 1e-3), 1), posed=int((counts > 0).sum()),
                rot_err_vs_truth_median=float(np.median(rerr)), R=R, t=t, counts=counts)


def host_arm(name, sub=8):
    xys, pofs, pts, Ks, Rs, ts = scene(name)
    J = len(xys)
    try:
        import cv2
        t0 = time.perf_counter()
        out = []
        for p in range(J):
            ok = pofs[p] >= 0
            r = cv2.solvePnPRansac(pts[pofs[p][ok]], xys[p][ok].astype(np.float64), Ks[p], None,
                                   iterationsCount=LOOPS, reprojectionError=MAXERR, confidence=0.999999,
                                   flags=cv2.SOLVEPNP_P3P)
            out.append((cv2.Rodrigues(r[1])[0], r[2].reshape(3)) if r[0] else (np.zeros((3, 3)), np.zeros(3)))
        dt = time.perf_counter() - t0
        return dict(kind="cv2.solvePnPRansac (P3P, %d iterations, 1 thread of the host)" % LOOPS, ms=round(dt * 1e3, 2),
                    images_per_s=round(J / dt, 1)), out
    except ImportError:
        import pose_oracle as po
        k = min(J, sub)
        t0 = time.perf_counter()
        out = [po.pose_job(xys[p], pofs[p], pts, Ks[p], LOOPS, MAXERR, p) for p in range(k)]
        dt = (time.perf_counter() - t0) * J / k
        return dict(kind="float64 statement (numpy), %d of %d images timed and extrapolated" % (k, J),
                    ms=round(dt * 1e3, 2), images_per_s=round(J / dt, 2)), [(o["R"], o["t"]) for o in out]


def profile_child(name):
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cudasift_b200 as cs
    cs.InitCuda(0)
    xys, pofs, pts, Ks, _, _ = scene(name)
    datas = [Data(cs, xy) for xy in xys]
    cs.AbsolutePoseBatch(datas, pofs, pts, Ks, LOOPS, MAXERR)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            cs.AbsolutePoseBatch(datas, pofs, pts, Ks, LOOPS, MAXERR)
        torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        if "pose_" in e.key:
            k = e.key.split("pose_")[1].split("_kernel")[0]
            split[k] = round(e.device_time_total / 5 / 1e3, 4) if hasattr(e, "device_time_total") else \
                round(e.cuda_time_total / 5 / 1e3, 4)
    print(json.dumps(split))


def ptxas():
    from cudasift_b200 import build
    out = subprocess.run([build.nvcc_path()] + [f for f in build.NVCC_FLAGS if f != "-shared"] +
                         ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "pose.cu"), "-o", os.devnull],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"pose_(gather|hyp|score|argmax|refine)_kernel", line)
        if "Compiling entry function" in line and m:
            cur = m.group(1)
        elif cur and "bytes stack frame" in line:
            res[cur] = line.strip()
        elif cur and "Used" in line and "registers" in line:
            res[cur] = res.get(cur, "") + "; " + line.split(":", 1)[1].strip()
            cur = None
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--workloads", default="abc")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--child", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.child:
        profile_child(args.child)
        return
    res = {"card": card(), "numLoops": LOOPS, "maxError": MAXERR}
    for name in args.workloads:
        g = run_gpu(name, args.reps)
        h, poses = host_arm(name)
        agree = [float(np.abs(g["R"][p] - R).max()) for p, (R, t) in enumerate(poses) if g["counts"][p] > 0 and R.any()]
        for k in ("R", "t", "counts"):
            g.pop(k)
        g["host"] = h
        g["speedup_vs_host"] = round(h["ms"] / (g["ms_median"] * len(poses) / g["jobs"]), 1) if poses else None
        g["rot_diff_vs_host_median"] = float(np.median(agree)) if agree else None
        if args.profile:
            out = subprocess.run([sys.executable, __file__, "--child", name], stdout=subprocess.PIPE, text=True).stdout
            g["kernel_ms_per_call"] = json.loads(out.strip().splitlines()[-1]) if out.strip() else None
        res[name] = g
    # (a)'s scoring bound: 64 x 1024 x <= 4 x 2000 FP64 reprojections of about 30 FP64 operations at 34 TFLOP/s
    res["a_scoring_bound_ms"] = round(64 * LOOPS * 4 * 2000 * 30 / 34e12 * 1e3, 3)
    try:
        res["ptxas"] = ptxas()
    except Exception as e:
        res["ptxas"] = str(e)[:80]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        open(args.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
