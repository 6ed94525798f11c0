"""Batched ratio matching (cs_match_ratio_batch) against the loop of single cs_match_ratio calls it replaces.

Workloads: every pair of N = 8, 16 and 32 synthetic 1920x1080 views (distinct shifts of synth_image) through the
batched ranked extractor at 1 000 and 4 000 features, and 64 pairs among 16 sets of 10 000 synth_descriptors; each with
crossCheck on and off.  Arms: one batch call against the loop of single calls in auto mode, alternating call by call;
the times are the medians of the calls' own CUDA events (the loop's time is the sum over its calls), and every job's
count and pair bytes are compared in every round.  The kernel split of the batch call (summed over its waves) comes
from CUDASIFT_MATCH_TIMING in a child process.  The collection chain (batch extraction, matching, cs_verify_pairs_batch
for F) is timed on the host clock with either matcher.  The card's name and power limit are read in the same run.
One JSON line on stdout; a table on stderr.
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

from mutual_bench import card  # noqa: E402

VIEWS = (8, 16, 32)
FEATURES = (1000, 4000)
W, H = 1920, 1080


def extract_views(cs, n, feats):
    """n shifted views through one batched ranked extractor: (SiftData list, extractor call in ms on the host clock)."""
    from cudasift_b200.synth import synth_image
    img = synth_image(W, H, seed=5)
    pitch = cs.iAlignUp(W, 128)
    cis = []
    for k in range(n):
        ci = cs.CudaImage().Allocate(W, H, pitch, False, None,
                                     np.ascontiguousarray(np.roll(img, (3 * k - 40, 5 * k - 70), axis=(0, 1))))
        ci.Download()
        cis.append(ci)
    ex = cs.Extractor(W, H, 5, feats, False, batch=n, maxCandidates=32768)
    try:
        ex.submit_device_batch([ci.d_data for ci in cis], pitch, 1.0, 3.0, 0.0)
        ex.wait_batch(n)
        t0 = time.perf_counter()
        ex.submit_device_batch([ci.d_data for ci in cis], pitch, 1.0, 3.0, 0.0)
        counts = ex.wait_batch(n)
        t_ext = 1000 * (time.perf_counter() - t0)
        datas = []
        for i in range(n):
            d = cs.SiftData()
            cs.InitSiftData(d, int(counts[i]))
            d._buf.upload(ex.device_points_at(i, int(counts[i])))
            d.numPts = int(counts[i])
            datas.append(d)
    finally:
        ex.close()
    return datas, t_ext


def descriptor_sets(cs, k, n):
    from cudasift_b200.synth import synth_descriptors
    datas = []
    for s in range(k):
        d = cs.SiftData()
        cs.InitSiftData(d, n)
        d._buf.upload(synth_descriptors(n, 300 + s, sift_like=True))
        d.numPts = n
        datas.append(d)
    return datas


def workloads(cs, args):
    for n in args.views:
        for f in args.features:
            datas, t_ext = extract_views(cs, n, f)
            yield "views%d_f%d" % (n, f), datas, list(itertools.combinations(range(n), 2)), t_ext
    if args.large:
        datas = descriptor_sets(cs, 16, 10000)
        yield "desc10000_j64", datas, list(itertools.combinations(range(16), 2))[:64], None


class Arms:
    """The batch call and the loop of single calls on one workload, into the same pair-buffer layout."""

    def __init__(self, cs, datas, jobs, cross):
        self.cs, self.datas, self.jobs, self.cross = cs, datas, jobs, cross
        self.rooms = [min(datas[a].numPts, datas[b].numPts) if cross else datas[a].numPts for a, b in jobs]
        self.off = np.concatenate([[0], np.cumsum(self.rooms)]).astype(np.int64)
        total = max(int(self.off[-1]), 1)
        self.bufs = [cs.DeviceBuffer(8 * total), cs.DeviceBuffer(8 * total)]
        self.sets = (cs.MatchSet * len(datas))(*[cs.MatchSet(d.d_data, d.numPts) for d in datas])
        self.table = (cs.MatchJob * len(jobs))(*[cs.MatchJob(a, b, self.bufs[0].ptr + 8 * int(self.off[q]), self.rooms[q])
                                                 for q, (a, b) in enumerate(jobs)])

    def batch(self):
        J = len(self.jobs)
        counts, stats, ms = np.zeros(J, np.int32), np.zeros((J, 4), np.uint64), ctypes.c_double(0.0)
        r = self.cs.lib().cs_match_ratio_batch(self.sets, len(self.datas), self.table, J, 0.8, 0.7, self.cross,
                                               counts.ctypes.data, stats.ctypes.data, ctypes.byref(ms))
        assert r == 0, self.cs.lib().cs_last_error()
        return ms.value, counts

    def loop(self):
        L = self.cs.lib()
        total, counts = 0.0, np.zeros(len(self.jobs), np.int32)
        for q, (a, b) in enumerate(self.jobs):
            d1, d2, ms = self.datas[a], self.datas[b], ctypes.c_double(0.0)
            counts[q] = L.cs_match_ratio(d1.d_data, d1.numPts, d2.d_data, d2.numPts, 0.8, 0.7, self.cross,
                                         self.bufs[1].ptr + 8 * int(self.off[q]), self.rooms[q], 0, ctypes.byref(ms))
            assert counts[q] >= 0, L.cs_last_error()
            total += ms.value
        return total, counts

    def pairs(self, k, counts):
        flat = self.bufs[k].download(np.int32, 2 * int(self.off[-1])).reshape(-1, 2)
        return [flat[self.off[q]:self.off[q] + counts[q]].tobytes() for q in range(len(self.jobs))]

    def free(self):
        for b in self.bufs:
            b.free()


def chain(cs, datas, jobs, cross, batched, t_ext):
    """Extraction (the measured batch call) + matching + batched F verification, host clock, in ms."""
    t0 = time.perf_counter()
    if batched:
        pairs = cs.MatchSiftDataRatioBatch(datas, jobs, crossCheck=cross)[0]
    else:
        pairs = [cs.MatchSiftDataRatio(datas[a], datas[b], crossCheck=cross)[0] for a, b in jobs]
    cs.VerifyPairsBatch([(datas[a], datas[b], p, q) for q, ((a, b), p) in enumerate(zip(jobs, pairs))],
                        "fundamental", 1024, 4.0)
    return t_ext + 1000 * (time.perf_counter() - t0)


def split_child(args):
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, datas, jobs, _ in workloads(cs, args):
        for cross in (1, 0):
            arms = Arms(cs, datas, jobs, cross)
            for _ in range(2):
                sys.stderr.write("call\n")
                arms.batch()
            sys.stderr.write("setting %s_cross%d\n" % (name, cross))
            sys.stderr.flush()
            arms.free()
        for d in datas:
            cs.FreeSiftData(d)


def parse_split(text):
    out, rows = {}, []
    for line in text.splitlines():
        if line.startswith("call"):
            rows = []
        elif line.startswith("ratio-batch timing"):
            rows.append({k: float(v) for k, v in re.findall(r" ([a-z-]+) ([0-9.]+)", line.split("[us]:")[1])})
        elif line.startswith("setting "):
            split = {k: round(sum(r[k] for r in rows), 1) for k in rows[0]} if rows else {}
            split["waves"] = len(rows)
            out[line[8:].strip()] = split
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--views", nargs="+", type=int, default=list(VIEWS))
    ap.add_argument("--features", nargs="+", type=int, default=list(FEATURES))
    ap.add_argument("--no-large", dest="large", action="store_false")
    ap.add_argument("--split-child", action="store_true")
    args = ap.parse_args()
    if args.split_child:
        split_child(args)
        return
    import cudasift_b200 as cs
    cs.InitCuda(0)
    res = {}
    for name, datas, jobs, t_ext in workloads(cs, args):
        for cross in (1, 0):
            arms = Arms(cs, datas, jobs, cross)
            tb, tl, same = [], [], True
            for rep in range(args.reps + 1):                       # the first round warms up
                b, l = arms.batch(), arms.loop()
                same = same and np.array_equal(b[1], l[1]) and arms.pairs(0, b[1]) == arms.pairs(1, l[1])
                if rep:
                    tb.append(b[0])
                    tl.append(l[0])
            mb, ml = float(np.median(tb)), float(np.median(tl))
            J = len(jobs)
            r = {"jobs": J, "features": [d.numPts for d in datas[:1]][0], "crossCheck": cross,
                 "batch_ms": round(mb, 3), "loop_ms": round(ml, 3), "batch_us_per_pair": round(1000 * mb / J, 2),
                 "loop_us_per_pair": round(1000 * ml / J, 2), "speedup": round(ml / mb, 2), "identical": bool(same),
                 "pairs": int(b[1].sum())}
            if t_ext is not None:
                cb = [chain(cs, datas, jobs, cross, True, t_ext) for _ in range(3)]
                cl = [chain(cs, datas, jobs, cross, False, t_ext) for _ in range(3)]
                r.update(chain_batched_ms=round(float(np.median(cb)), 2), chain_loop_ms=round(float(np.median(cl)), 2),
                         extraction_ms=round(t_ext, 2))
            res["%s_cross%d" % (name, cross)] = r
            arms.free()
        for d in datas:
            cs.FreeSiftData(d)
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    cmd = [sys.executable, os.path.abspath(__file__), "--split-child", "--views", *map(str, args.views),
           "--features", *map(str, args.features)] + ([] if args.large else ["--no-large"])
    child = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    split = parse_split(child.stderr) if child.returncode == 0 else {"error": child.stderr[-300:]}
    for name, r in res.items():
        r["kernel_split_us"] = split.get(name, split if "error" in split else {})
    out = {"metric": "batched ratio matching against the loop of single calls (ms, medians of the calls' CUDA events)",
           "card": card(), "maxRatio": 0.8, "maxDistance": 0.7, "reps": args.reps, "settings": res}
    for name, r in res.items():
        sys.stderr.write("%-22s J %4d batch %9.3f ms loop %9.3f ms  per pair %8.2f / %8.2f us  x%6.2f  %s  %s\n" % (
            name, r["jobs"], r["batch_ms"], r["loop_ms"], r["batch_us_per_pair"], r["loop_us_per_pair"], r["speedup"],
            "identical" if r["identical"] else "DIFFERENT",
            ("chain %.1f / %.1f ms" % (r["chain_batched_ms"], r["chain_loop_ms"])) if "chain_loop_ms" in r else ""))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
