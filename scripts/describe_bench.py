#!/usr/bin/env python
"""describe_bench.py -- describe-stage time of two or more builds of the library, loaded in one process.

  python scripts/describe_bench.py --lib parent=PATH --lib new=PATH [--lib ...] [--rounds R] [--warmup W]

Every library gets its own extractors (batch 16 and batch 1) over the 16 synthetic 1920x1080 images that bench.py
uses, resident in HBM.  A round profiles one batch of 16 and one batch of one with every library in turn
(cs_extractor_profile_batch: CUDA events at the stage boundaries), so the libraries alternate call by call.  Reported
per library and batch size: the medians over the rounds of the describe stage and of the whole pipeline per image (us),
the describe stage's ratio to the first library's, and the keypoints found (equal in every library, or the run fails).
The card's name and power limit are read in the same run.  One JSON line on stdout.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (image size, parameters, synthetic images)

BATCHES = (16, 1)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:
        return {"error": str(e)[:80]}


class Lib:
    """The C ABI calls this benchmark needs, bound on one library file (each file keeps its own state)."""

    def __init__(self, name, path):
        c = ctypes
        vp, ip, fp = c.c_void_p, c.c_int, c.c_float
        self.name, self.path = name, path
        L = self.L = c.CDLL(os.path.abspath(path), mode=os.RTLD_LOCAL)
        for f, (res, args) in {"cs_last_error": (c.c_char_p, []), "cs_init": (ip, [ip]),
                               "cs_device_alloc": (vp, [c.c_size_t]), "cs_memcpy_h2d": (ip, [vp, vp, c.c_size_t]),
                               "cs_extractor_create_batch": (vp, [ip, ip, ip, ip, ip, ip]),
                               "cs_extractor_destroy": (ip, [vp]),
                               "cs_extractor_profile_batch": (ip, [vp, ip, vp, ip, c.c_double, fp, fp, c.POINTER(fp)])}.items():
            getattr(L, f).restype, getattr(L, f).argtypes = res, args
        self.check(L.cs_init(0), "cs_init")

    def check(self, r, what):
        if r is None or (isinstance(r, int) and r < 0):
            raise RuntimeError("%s: %s failed: %s" % (self.name, what, self.L.cs_last_error().decode()))
        return r

    def profile(self, ex, ptrs, pitch):
        arr = (ctypes.c_void_p * len(ptrs))(*ptrs)
        out = (ctypes.c_float * 5)()
        n = self.check(self.L.cs_extractor_profile_batch(ex, len(ptrs), arr, pitch, bench.INIT_BLUR, bench.THRESH, 0.0, out),
                       "profile")
        return n, list(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, metavar="NAME=PATH", help="a library to time (repeat)")
    ap.add_argument("--rounds", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    libs = [Lib(*spec.split("=", 1)) for spec in args.lib]
    W, H = bench.W, bench.H
    pitch = (W + 127) // 128 * 128
    imgs = bench.make_images(0, max(BATCHES))
    ptrs = []
    for im in imgs:                                   # device images of the first library, read by every library
        padded = np.zeros((H, pitch), np.float32)
        padded[:, :W] = im
        d = libs[0].check(libs[0].L.cs_device_alloc(padded.nbytes), "alloc")
        libs[0].check(libs[0].L.cs_memcpy_h2d(d, padded.ctypes.data, padded.nbytes), "h2d")
        ptrs.append(d)
    exs = {(lb.name, b): lb.check(lb.L.cs_extractor_create_batch(W, H, bench.OCTAVES, bench.MAX_PTS, 0, b), "create")
           for lb in libs for b in BATCHES}
    times = {(lb.name, b): [] for lb in libs for b in BATCHES}
    found = {}
    for r in range(args.warmup + args.rounds):
        for b in BATCHES:
            for lb in libs:                           # the libraries alternate call by call
                n, ms = lb.profile(exs[(lb.name, b)], ptrs[:b], pitch)
                found.setdefault(b, {})[lb.name] = n
                if r >= args.warmup:
                    times[(lb.name, b)].append(ms)
    for b in BATCHES:
        assert len(set(found[b].values())) == 1, ("keypoints differ", b, found[b])
    res = {}
    for b in BATCHES:
        base = None
        for lb in libs:
            t = np.array(times[(lb.name, b)]) / b * 1e3        # us per image
            d = float(np.median(t[:, 3]))
            base = d if base is None else base
            res["%s_batch%d" % (lb.name, b)] = {"describe_us": round(d, 3), "pipeline_us": round(float(np.median(t[:, 4])), 3),
                                                "describe_ratio": round(d / base, 3),
                                                "describe_us_p10_p90": [round(float(np.percentile(t[:, 3], q)), 3) for q in (10, 90)],
                                                "keypoints": found[b][lb.name]}
    for lb in libs:
        for b in BATCHES:
            lb.L.cs_extractor_destroy(exs[(lb.name, b)])
    print(json.dumps({"metric": "describe stage, us per image (median of %d alternating rounds)" % args.rounds,
                      "card": card(), "libs": {lb.name: lb.path for lb in libs}, "results": res}), flush=True)


if __name__ == "__main__":
    main()
