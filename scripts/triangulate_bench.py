"""Triangulation of feature tracks (cs_triangulate_tracks) against the host statement of the same rules.

Workloads:
  chain32      the tracks of scripts/tracks_bench.py's chain32 (32 shifted 1920x1080 views at 1 000 ranked features,
               ratio batch, verify batch, guided batch, BuildTracks), with the cameras of the shifts: a fronto-parallel
               plane at Z0 = 10, K = [400 0 960; 0 400 540; 0 0 1], R = I, C_k = -(dx, dy, 0) Z0 / 400
  synthetic    10^6 tracks of 2-12 views over 1 000 cameras (tests/triangulate_cases.collection: skewed, unequal
               intrinsics, arbitrary rolls, 0.5 px noise, 10 % outliers)
Both at numTrials = 256, maxError = 4 px, minTriAngle = 1.5 degrees (0.5 for chain32, whose baselines are short).
Arms: the call on device-resident tracks (the median of its own CUDA events over --reps calls after a warm-up), and the
host arm: tests/triangulate_oracle.py (numpy, vectorised per track) timed on --host-tracks seeded tracks and
extrapolated to all of them (labelled as such).  Agreement: on those tracks, counts, inlier masks and point presence
equal, and the largest point difference.  The kernel split comes from torch.profiler in a child process.  The card's
name and power limit are read in the same run.  One JSON line on stdout; a table on stderr.
"""
import argparse
import ctypes
import itertools
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mutual_bench import card  # noqa: E402

import triangulate_cases as tc  # noqa: E402
import triangulate_oracle as to  # noqa: E402


def chain32(cs):
    from guided_batch_bench import verified
    from match_batch_bench import H, W, extract_views
    from cudasift_b200.records import SIFT_DTYPE
    datas, _ = extract_views(cs, 32, 1000)
    jobs, Ms = verified(cs, datas, list(itertools.combinations(range(32), 2)), "fundamental")
    guided, _, _ = cs.MatchSiftDataGuidedBatch(datas, jobs, "fundamental", Ms, 4.0)
    offsets, members, _, _, _ = cs.BuildTracks([d.numPts for d in datas], [(a, b, g) for (a, b), g in zip(jobs, guided)])
    xy = []
    for d in datas:
        r = d._buf.download(SIFT_DTYPE, d.numPts)
        xy.append(np.stack([r["xpos"], r["ypos"]], 1))
        cs.FreeSiftData(d)
    f, Z0 = 400.0, 10.0
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])
    ts = np.array([[(5 * k - 70) * Z0 / f, (3 * k - 40) * Z0 / f, 0.0] for k in range(32)])
    return dict(xy=xy, Ks=np.stack([K] * 32), Rs=np.stack([np.eye(3)] * 32), ts=ts, offsets=offsets, members=members,
                minTriAngle=0.5)


def synthetic(cs):
    xy, Ks, Rs, ts, offsets, members, _ = tc.collection(0, 10 ** 6)
    return dict(xy=xy, Ks=Ks, Rs=Rs, ts=ts, offsets=offsets, members=members, minTriAngle=1.5)


WORKLOADS = {"chain32": chain32, "synthetic": synthetic}


class Call:
    """Record sets, tracks and outputs in device memory; run() is one call."""

    def __init__(self, cs, w):
        from cudasift_b200.records import SIFT_DTYPE
        self.cs, self.w, self.bufs, sets = cs, w, [], []
        for p in w["xy"]:
            rec = np.zeros(len(p), SIFT_DTYPE)
            rec["xpos"], rec["ypos"] = p[:, 0], p[:, 1]
            b = cs.DeviceBuffer(max(rec.nbytes, 8))
            if len(p):
                b.upload(rec)
            self.bufs.append(b)
            sets.append(cs.MatchSet(b.ptr if len(p) else None, len(p)))
        self.sets = (cs.MatchSet * len(sets))(*sets)
        self.K, self.R, self.t = (np.ascontiguousarray(w[k], np.float64) for k in ("Ks", "Rs", "ts"))
        off, mem = np.asarray(w["offsets"], np.int32), np.asarray(w["members"], np.int32).reshape(-1, 2)
        self.T, self.M = len(off) - 1, len(mem)
        self.io = [cs.DeviceBuffer(off.nbytes), cs.DeviceBuffer(mem.nbytes), cs.DeviceBuffer(24 * self.T),
                   cs.DeviceBuffer(4 * self.T), cs.DeviceBuffer(4 * self.M), cs.DeviceBuffer(self.M)]
        self.io[0].upload(off)
        self.io[1].upload(mem)
        self.stats = np.zeros(8, np.int64)

    def run(self):
        ms = ctypes.c_double(0.0)
        io = self.io
        r = self.cs.lib().cs_triangulate_tracks(self.sets, len(self.w["xy"]), self.K.ctypes.data, self.R.ctypes.data,
                                                self.t.ctypes.data, io[0].ptr, self.T, io[1].ptr, self.M, 256, 4.0,
                                                self.w["minTriAngle"], 0, io[2].ptr, io[3].ptr, io[4].ptr, io[5].ptr,
                                                self.stats.ctypes.data, ctypes.byref(ms))
        assert r >= 0, self.cs.lib().cs_last_error()
        return ms.value

    def outputs(self):
        return (self.io[2].download(np.float64, 3 * self.T).reshape(-1, 3), self.io[3].download(np.int32, self.T),
                self.io[5].download(np.uint8, self.M).astype(bool))

    def free(self):
        for b in self.bufs + self.io:
            b.free()


def split_child(args):
    """Kernel times per call (torch.profiler), one JSON object per workload on stdout."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cudasift_b200 as cs
    cs.InitCuda(0)
    torch.cuda.init()
    out = {}
    for name in args.workloads:
        c = Call(cs, WORKLOADS[name](cs))
        c.run()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                c.run()
        split = {}
        for e in prof.key_averages():
            if e.device_type.name != "CUDA":
                continue
            m = re.search(r"triangulate_kernel", e.key)
            key = "triangulate_kernel" if m else "memcpy" if "Memcpy" in e.key else "memset" if "Memset" in e.key \
                else e.key[:40]
            split[key] = split.get(key, 0.0) + e.device_time_total / args.reps
        out[name] = {k: round(v, 1) for k, v in split.items()}
        c.free()
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-tracks", type=int, default=2000)
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS))
    ap.add_argument("--split-child", action="store_true")
    args = ap.parse_args()
    if args.split_child:
        split_child(args)
        return
    import cudasift_b200 as cs
    cs.InitCuda(0)
    res = {}
    for name in args.workloads:
        w = WORKLOADS[name](cs)
        c = Call(cs, w)
        c.run()
        times = [c.run() for _ in range(args.reps)]
        pts, cnt, inl = c.outputs()
        sub = np.sort(np.random.default_rng(1).choice(c.T, min(args.host_tracks, c.T), replace=False))
        t0 = time.perf_counter()
        want = to.triangulate(w["xy"], w["Ks"], w["Rs"], w["ts"], w["offsets"], w["members"], 256, 4.0,
                              w["minTriAngle"], 0, tracks=sub)
        host = 1000 * (time.perf_counter() - t0) * c.T / len(sub)
        off = np.asarray(w["offsets"], np.int64)
        mem = np.concatenate([np.arange(off[k], off[k + 1]) for k in sub])
        has = ~np.isnan(want["points"][:, 0])
        agree = (cnt[sub].tolist() == want["counts"].tolist() and np.array_equal(inl[mem], want["inlier"][mem]) and
                 np.array_equal(~np.isnan(pts[sub, 0]), has))
        dev = float(np.abs(pts[sub][has] - want["points"][has]).max(initial=0.0))
        ms = float(np.median(times))
        res[name] = {"images": len(w["xy"]), "tracks": c.T, "members": c.M, "call_ms": round(ms, 3),
                     "tracks_per_s": float("%.4g" % (c.T / ms * 1000)),
                     "host_oracle_ms_extrapolated": round(host, 1), "host_tracks_timed": int(len(sub)),
                     "speedup": round(host / ms, 1), "subset_agrees": bool(agree), "subset_max_point_diff": dev,
                     "stats": c.stats.tolist()}
        c.free()
    cmd = [sys.executable, os.path.abspath(__file__), "--split-child", "--reps", str(args.reps), "--workloads",
           *args.workloads]
    child = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    try:
        split = json.loads(child.stdout.strip().splitlines()[-1])
    except Exception:
        split = {"error": child.stderr[-300:]}
    for name, r in res.items():
        r["kernel_split_us"] = split.get(name, split if "error" in split else {})
    out = {"metric": "cs_triangulate_tracks against the float64 host statement (ms; call: median of its CUDA events, "
                     "host: oracle on a seeded subset, extrapolated)", "card": card(), "reps": args.reps,
           "workloads": res}
    for name, r in res.items():
        sys.stderr.write("%-10s tracks %8d call %9.3f ms host(extrap.) %10.1f ms x%8.1f %s %s\n" % (
            name, r["tracks"], r["call_ms"], r["host_oracle_ms_extrapolated"], r["speedup"],
            "agree" if r["subset_agrees"] else "DIFFER", r["kernel_split_us"]))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
