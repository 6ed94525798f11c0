"""Dense reconstruction timings: PatchMatch depth maps, fusion and undistortion on one GPU, plus the float64 oracle's
per-pixel rate on the CPU (the host arm).  Workload: --maps reference images of --width x --height, each with
--sources sources (the others of a ring), window radius 5 at step 1 and radius 4 at step 2 (the radius must be a
multiple of the step), --iterations iterations; medians of
--calls calls after one warm-up call.  Then the geometric-consistency pass on the same workload (radius 5, step 1,
--iterations iterations) from the step-1 photometric maps, and its time over the photometric one's.  Times are device
events.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import cudasift_b200 as cs  # noqa: E402
from cudasift_b200 import synth  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True).stdout.strip()
    except OSError:
        return "unknown"


def cameras(n, W, H):
    from triangulate_cases import look_at
    Ks, Rs, ts = [], [], []
    for a in range(n):
        ang = 2 * np.pi * a / n
        C = np.array([0.6 * np.sin(ang), 0.3 * np.cos(ang), -6.0])
        R = look_at(C, np.zeros(3), 0.0)
        Ks.append(np.array([[0.9 * W, 0, W / 2], [0, 0.9 * W, H / 2], [0, 0, 1.0]]))
        Rs.append(R)
        ts.append(-R @ C)
    return np.array(Ks), np.array(Rs), np.array(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--maps", type=int, default=16)
    ap.add_argument("--sources", type=int, default=8)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--iterations", type=int, default=5)
    ap.add_argument("--calls", type=int, default=3)
    a = ap.parse_args()
    n = max(a.maps, a.sources + 1)
    W, H = a.width, a.height
    Ks, Rs, ts = cameras(n, W, H)
    images = [synth.synth_image(W, H, seed=100 + k) for k in range(n)]
    jobs = [(r, [(r + 1 + k) % n for k in range(a.sources)], 4.0, 9.0) for r in range(a.maps)]
    out = dict(gpu=gpu_info(), maps=a.maps, sources=a.sources, width=W, height=H, iterations=a.iterations)
    maps = None
    for r, step in ((5, 1), (4, 2)):
        cs.PatchMatchStereo(images, Ks, Rs, ts, jobs, windowRadius=r, windowStep=step, numIterations=1)
        runs = [cs.PatchMatchStereo(images, Ks, Rs, ts, jobs, windowRadius=r, windowStep=step,
                                    numIterations=a.iterations) for _ in range(a.calls)]
        maps = maps or runs[-1]
        t = float(np.median([run[4] for run in runs]))
        side = 2 * r // step + 1
        # window samples: per pixel and iteration 12 candidates (fewer at the border), each over every source
        samples = a.maps * W * H * (1 + 12 * a.iterations) * a.sources * side * side
        out["ms_per_map_step%d" % step] = t / a.maps
        out["samples_per_s_step%d" % step] = samples / (t * 1e-3)
    cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, maps[0], maps[1], windowRadius=5, numIterations=1)
    geo = [cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, maps[0], maps[1], windowRadius=5,
                                        numIterations=a.iterations)[4] for _ in range(a.calls)]
    out["ms_per_map_geometric"] = float(np.median(geo)) / a.maps
    out["geometric_over_photometric"] = out["ms_per_map_geometric"] / out["ms_per_map_step1"]
    d, nrm, c, _, _ = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs, windowRadius=4, windowStep=2, numIterations=2)
    fus = [cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, d, nrm, c, maxPoints=1 << 20)[5] for _ in range(a.calls)]
    out["fusion_ms"] = float(np.median(fus))
    und = [cs.UndistortImages(images, Ks, np.array([-0.1, 0.02]))[2] for _ in range(a.calls)]
    out["undistort_GBps"] = 2 * 4 * n * W * H / (float(np.median(und)) * 1e6)
    import stereo_oracle as so
    small = [im[:60, :80] for im in images[:3]]
    Ks2 = Ks.copy()
    Ks2[:, 0, 2], Ks2[:, 1, 2] = 40, 30
    job = so.Job(Ks2, Rs, ts, 0, [1, 2], 4.0, 9.0)
    t0 = time.perf_counter()
    st = so.start(small, job, 0, 5, 1, 2)
    so.half_step(small, job, st, 1, 0, 0, 5, 1, 2)
    out["oracle_cpu_pixels_per_s"] = (80 * 60 * 1.5) / (time.perf_counter() - t0)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
