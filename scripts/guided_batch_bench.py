"""Batched guided matching (cs_match_guided_batch) against the loop of single cs_match_guided calls it replaces.

Workloads: every pair of N = 8, 16 and 32 shifted 1920x1080 views through the batched ranked extractor at 1 000
features (scripts/match_batch_bench.py), each pair's model from VerifyPairsBatch on its ratio pairs (F and H; pairs
whose verification found no model are left out), at 2 and 4 px; and 64 jobs over the planted 10 000 x 10 000 F and H
views of scripts/guided_bench.py.  Each with crossCheck on and off.  Arms: one batch call against the loop of single
calls, alternating call by call; the times are the medians of the calls' own CUDA events (the loop's time is the sum
over its calls), and every job's count and pair bytes are compared in every round.  The kernel split of the batch call
(summed over its waves) comes from CUDASIFT_MATCH_TIMING in a child process.  The collection chain (batch extraction,
ratio batch, verify batch, guided batch) is timed on the host clock.  The card's name and power limit are read in the
same run.  One JSON line on stdout; a table on stderr.
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

from guided_bench import planted_sets  # noqa: E402
from match_batch_bench import extract_views  # noqa: E402
from mutual_bench import card  # noqa: E402

VIEWS = (8, 16, 32)
THRESHOLDS = (2.0, 4.0)


def verified(cs, datas, pairs_idx, model):
    """The ratio batch and VerifyPairsBatch for one model: (jobs with a model, their models)."""
    ratio, _, _ = cs.MatchSiftDataRatioBatch(datas, pairs_idx)
    M, inl, _, _ = cs.VerifyPairsBatch([(datas[a], datas[b], ratio[k], k) for k, (a, b) in enumerate(pairs_idx)],
                                       model, 1024, 4.0)
    keep = [k for k in range(len(pairs_idx)) if len(inl[k]) > 0]
    return [pairs_idx[k] for k in keep], M[keep]


def planted_datas(cs):
    """Four planted 10 000 x 10 000 view pairs per model as SiftData: (datas, {model: [(a, b, M)]})."""
    datas, out = [], {"fundamental": [], "homography": []}
    for seed in range(4):
        for name, (s1, s2, M) in planted_sets(cs, 10000, 40 + seed).items():
            for s in (s1, s2):
                d = cs.SiftData()
                cs.InitSiftData(d, len(s))
                d._buf.upload(s)
                d.numPts = len(s)
                datas.append(d)
            out["fundamental" if name == "F" else "homography"].append((len(datas) - 2, len(datas) - 1, M))
    return datas, out


def workloads(cs, args):
    for n in args.views:
        datas, t_ext = extract_views(cs, n, 1000)
        pairs_idx = list(itertools.combinations(range(n), 2))
        for model in ("fundamental", "homography"):
            jobs, Ms = verified(cs, datas, pairs_idx, model)
            for t in args.thresholds:
                yield "views%d_%s_t%g" % (n, model[0].upper(), t), datas, jobs, model, Ms, t, (t_ext, pairs_idx)
        for d in datas:
            cs.FreeSiftData(d)
    if args.large:
        datas, planted = planted_datas(cs)
        for model, v in planted.items():
            jobs = [(a, b) for a, b, _ in v] * 16
            Ms = np.array([M for _, _, M in v] * 16)
            yield "planted10000_j64_%s_t4" % model[0].upper(), datas, jobs, model, Ms, 4.0, None
        for d in datas:
            cs.FreeSiftData(d)


class Arms:
    """The batch call and the loop of single calls on one workload, into the same pair-buffer layout."""

    def __init__(self, cs, datas, jobs, model, Ms, t, cross):
        self.cs, self.datas, self.jobs, self.t, self.cross = cs, datas, jobs, t, cross
        self.code = cs.GEOM_MODELS[model]
        self.codes = np.full(len(jobs), self.code, np.int32)
        self.Ms = np.ascontiguousarray(np.asarray(Ms, np.float64).reshape(len(jobs), 9))
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
        r = self.cs.lib().cs_match_guided_batch(self.sets, len(self.datas), self.table, J, self.codes.ctypes.data,
                                                self.Ms.ctypes.data, self.t, 0.8, 0.7, self.cross, counts.ctypes.data,
                                                stats.ctypes.data, ctypes.byref(ms))
        assert r == 0, self.cs.lib().cs_last_error()
        return ms.value, counts

    def loop(self):
        L = self.cs.lib()
        total, counts = 0.0, np.zeros(len(self.jobs), np.int32)
        for q, (a, b) in enumerate(self.jobs):
            d1, d2, ms = self.datas[a], self.datas[b], ctypes.c_double(0.0)
            counts[q] = L.cs_match_guided(d1.d_data, d1.numPts, d2.d_data, d2.numPts, self.code,
                                          self.Ms[q].ctypes.data, self.t, 0.8, 0.7, self.cross,
                                          self.bufs[1].ptr + 8 * int(self.off[q]), self.rooms[q], ctypes.byref(ms))
            assert counts[q] >= 0, L.cs_last_error()
            total += ms.value
        return total, counts

    def pairs(self, k, counts):
        flat = self.bufs[k].download(np.int32, 2 * int(self.off[-1])).reshape(-1, 2)
        return [flat[self.off[q]:self.off[q] + counts[q]].tobytes() for q in range(len(self.jobs))]

    def free(self):
        for b in self.bufs:
            b.free()


def chain(cs, datas, pairs_idx, model, t, t_ext):
    """Extraction (the measured batch call) + ratio batch + verify batch + guided batch, host clock, in ms."""
    t0 = time.perf_counter()
    jobs, Ms = verified(cs, datas, pairs_idx, model)
    cs.MatchSiftDataGuidedBatch(datas, jobs, model, Ms, t)
    return t_ext + 1000 * (time.perf_counter() - t0)


def split_child(args):
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, datas, jobs, model, Ms, t, _ in workloads(cs, args):
        for cross in (1, 0):
            arms = Arms(cs, datas, jobs, model, Ms, t, cross)
            for _ in range(2):
                sys.stderr.write("call\n")
                arms.batch()
            sys.stderr.write("setting %s_cross%d\n" % (name, cross))
            sys.stderr.flush()
            arms.free()


def parse_split(text):
    out, rows = {}, []
    for line in text.splitlines():
        if line.startswith("call"):
            rows = []
        elif line.startswith("guided-batch timing"):
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
    ap.add_argument("--thresholds", nargs="+", type=float, default=list(THRESHOLDS))
    ap.add_argument("--no-large", dest="large", action="store_false")
    ap.add_argument("--split-child", action="store_true")
    args = ap.parse_args()
    if args.split_child:
        split_child(args)
        return
    import cudasift_b200 as cs
    cs.InitCuda(0)
    res = {}
    for name, datas, jobs, model, Ms, t, ext in workloads(cs, args):
        for cross in (1, 0):
            arms = Arms(cs, datas, jobs, model, Ms, t, cross)
            tb, tl, same = [], [], True
            for rep in range(args.reps + 1):                       # the first round warms up
                b, l = arms.batch(), arms.loop()
                same = same and np.array_equal(b[1], l[1]) and arms.pairs(0, b[1]) == arms.pairs(1, l[1])
                if rep:
                    tb.append(b[0])
                    tl.append(l[0])
            mb, ml = float(np.median(tb)), float(np.median(tl))
            J = len(jobs)
            r = {"jobs": J, "crossCheck": cross, "batch_ms": round(mb, 3), "loop_ms": round(ml, 3),
                 "batch_us_per_pair": round(1000 * mb / J, 2), "loop_us_per_pair": round(1000 * ml / J, 2),
                 "speedup": round(ml / mb, 2), "identical": bool(same), "pairs": int(b[1].sum())}
            if ext is not None and cross:
                r["chain_ms"] = round(float(np.median([chain(cs, datas, ext[1], model, t, ext[0]) for _ in range(3)])), 2)
            res["%s_cross%d" % (name, cross)] = r
            arms.free()
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    cmd = [sys.executable, os.path.abspath(__file__), "--split-child", "--views", *map(str, args.views),
           "--thresholds", *map(str, args.thresholds)] + ([] if args.large else ["--no-large"])
    child = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    split = parse_split(child.stderr) if child.returncode == 0 else {"error": child.stderr[-300:]}
    for name, r in res.items():
        r["kernel_split_us"] = split.get(name, split if "error" in split else {})
    out = {"metric": "batched guided matching against the loop of single calls (ms, medians of the calls' CUDA events)",
           "card": card(), "maxRatio": 0.8, "maxDistance": 0.7, "reps": args.reps, "settings": res}
    for name, r in res.items():
        sys.stderr.write("%-30s J %4d batch %9.3f ms loop %9.3f ms  per pair %8.2f / %8.2f us  x%6.2f  %s %s %s\n" % (
            name, r["jobs"], r["batch_ms"], r["loop_ms"], r["batch_us_per_pair"], r["loop_us_per_pair"], r["speedup"],
            "identical" if r["identical"] else "DIFFERENT", r["kernel_split_us"],
            ("chain %.1f ms" % r["chain_ms"]) if "chain_ms" in r else ""))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
