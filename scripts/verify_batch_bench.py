"""Batched verification (cs_verify_pairs_batch, cs_verify_essential_batch) against the same jobs as sequential single
calls.

Jobs: J in {16, 64, 256, 1024}, every job a planted two-view scene of 588 (the ranked-pair size of DESIGN section 8),
1000 or 5000 pairs with 40 % uniform outliers: `planted` of tests/test_verify_gpu.py for F (a general scene) and H (a
plane), the sideways-motion scenes of scripts/essential_bench.py (tests/test_essential_gpu.py) for E.  Eight scenes per
size and model are generated and shared by the jobs, each job with its own seed.  Settings: numLoops 1024 and 4096,
thresh 2 px.  For each setting the batch call and the J single calls are timed in alternation, each as the medians of
the calls' own CUDA events (a single call's time is the sum over its J calls), and every job's outputs (model, count,
inliers, statistics; E, R, t for E) are checked for bit equality.  The per-kernel split of the batch call (summed over
its waves) comes from CUDASIFT_MATCH_TIMING in a child process.  The card's name and power limit are read in the same
run.  One JSON line on stdout; a table on stderr.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from mutual_bench import card  # noqa: E402

JOBS = (16, 64, 256, 1024)
SIZES = (588, 1000, 5000)
LOOPS = (1024, 4096)
MODELS = {"F": 2, "H": 1, "E": 3}
THRESH = 2.0
SCENES = 8


class Scenes:
    """Device records and pair lists of SCENES planted scenes per (model, size)."""

    def __init__(self, cs, models, sizes):
        from test_essential_cpu import K1, K2
        from test_essential_gpu import planted as planted_e
        from test_verify_gpu import planted, _records
        self.cs, self.K1, self.K2, self.bufs, self.scenes = cs, np.ascontiguousarray(K1), np.ascontiguousarray(K2), [], {}
        for m in models:
            for n in sizes:
                for k in range(SCENES):
                    if m == "E":
                        x1, x2, pairs = planted_e(n, 7 + n + 1000 * k)[:3]
                    else:
                        x1, x2, pairs = planted(n, 7 + n + 1000 * k, m == "H")[:3]
                    self.scenes[m, n, k] = (self._put(_records(cs, x1)), len(x1), self._put(_records(cs, x2)), len(x2),
                                            self._put(np.ascontiguousarray(pairs, np.int32)), len(pairs))

    def _put(self, a):
        b = self.cs.DeviceBuffer(a.nbytes)
        b.upload(a)
        self.bufs.append(b)
        return b.ptr

    def free(self):
        for b in self.bufs:
            b.free()


def make_jobs(cs, scenes, m, n, J):
    """The job table of J jobs (job p on scene p % SCENES, seed p), and the inlier buffers of the batch and the singles."""
    table = (cs.VerifyJob * J)()
    inl_b, inl_s = cs.DeviceBuffer(8 * n * J), cs.DeviceBuffer(8 * n * J)
    inl_b.zero()                                     # past each job's count the buffers keep these zeros
    inl_s.zero()
    for p in range(J):
        s1, n1, s2, n2, pairs, k = scenes.scenes[m, n, p % SCENES]
        table[p] = cs.VerifyJob(s1, n1, s2, n2, pairs, k, p, inl_b.ptr + 8 * n * p, k)
    return table, inl_b, inl_s


def run_batch(cs, scenes, m, J, table, loops):
    L = cs.lib()
    ms = ctypes.c_double(0.0)
    counts = np.zeros(J, np.int32)
    if m == "E":
        k1 = np.ascontiguousarray(np.broadcast_to(scenes.K1.reshape(9), (J, 9)))
        k2 = np.ascontiguousarray(np.broadcast_to(scenes.K2.reshape(9), (J, 9)))
        E, R, t, st = np.zeros((J, 9)), np.zeros((J, 9)), np.zeros((J, 3)), np.zeros((J, 10), np.int64)
        r = L.cs_verify_essential_batch(ctypes.addressof(table), J, k1.ctypes.data, k2.ctypes.data, loops, THRESH,
                                        E.ctypes.data, R.ctypes.data, t.ctypes.data, counts.ctypes.data, st.ctypes.data,
                                        ctypes.byref(ms))
        out = (np.concatenate([E, R, t], 1), st)
    else:
        M, st = np.zeros((J, 9)), np.zeros((J, 8), np.int64)
        r = L.cs_verify_pairs_batch(ctypes.addressof(table), J, MODELS[m], loops, THRESH, M.ctypes.data,
                                    counts.ctypes.data, st.ctypes.data, ctypes.byref(ms))
        out = (M, st)
    assert r == 0, L.cs_last_error()
    return ms.value, counts, out


def run_singles(cs, scenes, m, J, table, inl_s, n, loops):
    L = cs.lib()
    total, counts, models, stats = 0.0, np.zeros(J, np.int32), [], []
    for p in range(J):
        j = table[p]
        ms = ctypes.c_double(0.0)
        dst = inl_s.ptr + 8 * n * p
        if m == "E":
            E, R, t = np.zeros(9), np.zeros(9), np.zeros(3)
            k = L.cs_verify_essential(j.s1, j.n1, j.s2, j.n2, j.pairs, j.numPairs, scenes.K1.ctypes.data,
                                      scenes.K2.ctypes.data, loops, THRESH, j.seed, E.ctypes.data, R.ctypes.data,
                                      t.ctypes.data, dst, j.maxInliers, ctypes.byref(ms))
            models.append(np.concatenate([E, R, t]))
            stats.append(cs.essential_stats())
        else:
            M = np.zeros(9)
            k = L.cs_verify_pairs(j.s1, j.n1, j.s2, j.n2, j.pairs, j.numPairs, MODELS[m], loops, THRESH, j.seed,
                                  M.ctypes.data, dst, j.maxInliers, ctypes.byref(ms))
            models.append(M)
            stats.append(cs.verify_stats())
        assert k >= 0, L.cs_last_error()
        counts[p] = k
        total += ms.value
    return total, counts, (np.array(models), np.array(stats, np.int64))


def settings(args):
    for m in args.models:
        for loops in args.loops:
            for n in args.sizes:
                for J in args.jobs:
                    yield m, loops, n, J


def split_child(args):
    """Runs with CUDASIFT_MATCH_TIMING=1: two batch calls per setting; the library prints each wave's kernel times."""
    import cudasift_b200 as cs
    cs.InitCuda(0)
    scenes = Scenes(cs, args.models, args.sizes)
    for m, loops, n, J in settings(args):
        table, inl_b, inl_s = make_jobs(cs, scenes, m, n, J)
        for _ in range(2):
            sys.stderr.write("call\n")
            run_batch(cs, scenes, m, J, table, loops)
        sys.stderr.write("setting %s_%d_%d_%d\n" % (m, n, loops, J))
        sys.stderr.flush()
        inl_b.free()
        inl_s.free()
    scenes.free()


def parse_split(text):
    """{setting: {kernel: us summed over the last call's waves}, with "waves"}"""
    out, rows = {}, []
    for line in text.splitlines():
        if line.startswith("call"):
            rows = []
        elif line.startswith("verify timing"):
            toks = line.split("[us]:")[1].split()
            rows.append({toks[i]: float(toks[i + 1]) for i in range(0, len(toks), 2)})
        elif line.startswith("setting "):
            split = {k: round(sum(r[k] for r in rows), 1) for k in rows[0]} if rows else {}
            split["waves"] = len(rows)
            out[line[8:].strip()] = split
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--models", nargs="+", default=list(MODELS))
    ap.add_argument("--jobs", nargs="+", type=int, default=list(JOBS))
    ap.add_argument("--sizes", nargs="+", type=int, default=list(SIZES))
    ap.add_argument("--loops", nargs="+", type=int, default=list(LOOPS))
    ap.add_argument("--split-child", action="store_true")
    args = ap.parse_args()
    if args.split_child:
        split_child(args)
        return
    import cudasift_b200 as cs
    cs.InitCuda(0)
    scenes = Scenes(cs, args.models, args.sizes)
    res = {}
    for m, loops, n, J in settings(args):
        table, inl_b, inl_s = make_jobs(cs, scenes, m, n, J)
        tb, ts = [], []
        for rep in range(args.reps + 1):                           # the first round warms up and checks the outputs
            b = run_batch(cs, scenes, m, J, table, loops)
            s = run_singles(cs, scenes, m, J, table, inl_s, n, loops)
            if rep == 0:
                same = {"counts": np.array_equal(b[1], s[1]), "models": b[2][0].tobytes() == s[2][0].tobytes(),
                        "stats": np.array_equal(b[2][1], s[2][1]),
                        "inliers": inl_b.download(np.int32, 2 * n * J).tobytes() == inl_s.download(np.int32, 2 * n * J).tobytes()}
                inliers = int(b[1].sum())
            else:
                tb.append(b[0])
                ts.append(s[0])
        mb, msg = float(np.median(tb)), float(np.median(ts))
        res["%s_%d_%d_%d" % (m, n, loops, J)] = {
            "model": m, "numPairs": n, "numLoops": loops, "jobs": J, "batch_ms": round(mb, 4),
            "singles_ms": round(msg, 4), "batch_us_per_job": round(1000 * mb / J, 2),
            "single_us_per_job": round(1000 * msg / J, 2), "speedup": round(msg / mb, 2), "identical": all(same.values()),
            "differs": [k for k, v in same.items() if not v],
            "inliers": inliers}
        inl_b.free()
        inl_s.free()
    scenes.free()
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    cmd = [sys.executable, os.path.abspath(__file__), "--split-child", "--models", *args.models,
           "--jobs", *map(str, args.jobs), "--sizes", *map(str, args.sizes), "--loops", *map(str, args.loops)]
    child = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    split = parse_split(child.stderr) if child.returncode == 0 else {"error": child.stderr[-300:]}
    for name, r in res.items():
        r["kernel_split_us"] = split.get(name, split if "error" in split else {})
    out = {"metric": "batched verification against sequential single calls (ms, medians of the calls' CUDA events)",
           "card": card(), "thresh_px": THRESH, "reps": args.reps, "settings": res}
    for name, r in res.items():
        sys.stderr.write("%-20s batch %9.3f ms  singles %9.3f ms  per job %8.2f / %8.2f us  x%6.2f  %s\n" % (
            name, r["batch_ms"], r["singles_ms"], r["batch_us_per_job"], r["single_us_per_job"], r["speedup"],
            "identical" if r["identical"] else "DIFFERENT: " + " ".join(r["differs"])))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
