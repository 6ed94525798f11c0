"""Feature tracks (cs_build_tracks) against the host path a caller has without it.

Workloads:
  chain32      the guided-batch output of 32 shifted 1920x1080 views at 1 000 ranked features (F at 4 px, cross-checked,
               every verified pair of the 496), as scripts/guided_batch_bench.py builds it
  synthetic    1 000 images x 8 000 features, about 20 000 lists x 1 000 pairs: image a sees points a * 300 ... a * 300 +
               5 999 (tracks of 20 views) through its own feature permutation, lists between images 1 to 19 apart,
               950 planted pairs and 50 random pairs (5 %) per list
  path         2^22 features of one image paired with itself, 0 - 1 - ... in descending order
  star         one feature against 10^5 features of another image
Arms: the call on device-resident lists (the median of its own CUDA events over --reps calls after a warm-up), and the
host path on the same lists (download them, renumber globally, scipy.sparse.csgraph.connected_components, component
minima, numpy lexsort, runs, conflicts and the same output), host clock.  Both outputs are compared byte for byte.  The
kernel split (a mean per call over --reps calls) comes from torch.profiler in a child process.  The card's name and
power limit are read in the same run.  One JSON line on stdout; a table on stderr.
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


def chain32(cs):
    from guided_batch_bench import verified
    from match_batch_bench import extract_views
    datas, _ = extract_views(cs, 32, 1000)
    jobs, Ms = verified(cs, datas, list(itertools.combinations(range(32), 2)), "fundamental")
    guided, _, _ = cs.MatchSiftDataGuidedBatch(datas, jobs, "fundamental", Ms, 4.0)
    sizes = [d.numPts for d in datas]
    for d in datas:
        cs.FreeSiftData(d)
    return sizes, [(a, b, g) for (a, b), g in zip(jobs, guided)]


def synthetic(seed=0, n=1000, feats=8000, step=300, seen=6000, per=1000, rand=50):
    rng = np.random.default_rng(seed)
    perms = [rng.permutation(feats).astype(np.int32) for _ in range(n)]   # feature of point a * step + i in image a
    lists = []
    for a in range(n):
        for d in range(1, 21):
            b = a + d
            if b >= n or len(lists) >= 20000:
                continue
            shared = seen - step * d                                       # points b * step ... a * step + seen - 1
            if shared <= 0:
                continue
            p = b * step + rng.integers(0, shared, per - rand)
            planted = np.stack([perms[a][p - a * step], perms[b][p - b * step]], 1)
            lists.append((a, b, np.concatenate([planted, rng.integers(0, feats, (rand, 2), dtype=np.int32)])))
    return [feats] * n, lists


def path():
    n = 1 << 22
    k = np.arange(n - 2, -1, -1, dtype=np.int32)
    return [n], [(0, 0, np.stack([k + 1, k], 1))]


def star():
    n = 100000
    return [1, n], [(1, 0, np.stack([np.arange(n, dtype=np.int32), np.zeros(n, np.int32)], 1))]


WORKLOADS = {"chain32": chain32, "synthetic": lambda cs: synthetic(), "path": lambda cs: path(),
             "star": lambda cs: star()}


class Call:
    """Device-resident lists and outputs sized as BuildTracks sizes them; run() is one call."""

    def __init__(self, cs, sizes, lists):
        self.cs = cs
        self.sizes = np.asarray(sizes, np.int32)
        self.lists = [(a, b, np.ascontiguousarray(np.asarray(p, np.int32).reshape(-1, 2))) for a, b, p in lists]
        counts = [len(p) for _, _, p in self.lists]
        self.off = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int64)
        self.P, self.N = int(self.off[-1]), int(self.sizes.sum(dtype=np.int64))
        self.mm = min(self.N, 2 * self.P)
        self.mt = self.mm // 2
        self.bufs = [cs.DeviceBuffer(max(self.P, 1) * 8), cs.DeviceBuffer(4 * self.N), cs.DeviceBuffer(4 * (self.mt + 1)),
                     cs.DeviceBuffer(8 * max(self.mm, 1))]
        self.bufs[0].upload(np.concatenate([p for _, _, p in self.lists]))
        self.table = (cs.TrackList * len(self.lists))(*[
            cs.TrackList(a, b, self.bufs[0].ptr + 8 * int(self.off[q]) if len(p) else None, len(p))
            for q, (a, b, p) in enumerate(self.lists)])
        self.stats = np.zeros(8, np.int64)

    def run(self):
        ms = ctypes.c_double(0.0)
        T = self.cs.lib().cs_build_tracks(self.sizes.ctypes.data, len(self.sizes), self.table, len(self.lists), 2, 1,
                                          self.bufs[1].ptr, self.bufs[2].ptr, self.mt, self.bufs[3].ptr, self.mm,
                                          self.stats.ctypes.data, ctypes.byref(ms))
        assert T >= 0, self.cs.lib().cs_last_error()
        return ms.value, T

    def outputs(self, T):
        M = int(self.stats[7])
        return (self.bufs[2].download(np.int32, T + 1), self.bufs[3].download(np.int32, 2 * M).reshape(M, 2),
                self.bufs[1].download(np.int32, self.N))

    def host_path(self):
        """What a caller does today, from the device-resident lists to the same three arrays (ms, outputs)."""
        import scipy.sparse
        import scipy.sparse.csgraph
        t0 = time.perf_counter()
        flat = self.bufs[0].download(np.int32, 2 * self.P).reshape(-1, 2)
        base = np.concatenate([[0], np.cumsum(self.sizes, dtype=np.int64)])
        la = np.repeat(np.array([a for a, _, _ in self.lists], np.int64), np.diff(self.off))
        lb = np.repeat(np.array([b for _, b, _ in self.lists], np.int64), np.diff(self.off))
        ok = (flat[:, 0] >= 0) & (flat[:, 0] < self.sizes[la]) & (flat[:, 1] >= 0) & (flat[:, 1] < self.sizes[lb])
        u, v = base[la[ok]] + flat[ok, 0], base[lb[ok]] + flat[ok, 1]
        _, comp = scipy.sparse.csgraph.connected_components(
            scipy.sparse.coo_matrix((np.ones(len(u), np.int8), (u, v)), shape=(self.N, self.N)), directed=False)
        matched = np.zeros(self.N, bool)
        matched[u] = True
        matched[v] = True
        g = np.flatnonzero(matched)
        first = np.full(int(comp.max()) + 1, self.N, np.int64)
        np.minimum.at(first, comp[g], g)
        label = first[comp[g]]
        order = np.lexsort((g, label))
        g, label = g[order], label[order]
        image = np.searchsorted(base, g, side="right") - 1
        head = np.ones(len(g), bool)
        head[1:] = label[1:] != label[:-1]
        starts = np.flatnonzero(head)
        size = np.diff(np.concatenate([starts, [len(g)]]))
        same = np.zeros(len(g), bool)
        same[1:] = ~head[1:] & (image[1:] == image[:-1])
        conflict = np.add.reduceat(same.astype(np.int64), starts) > 0
        kept = (size >= 2) & ~conflict
        run = np.repeat(np.arange(len(starts)), size)
        track = np.full(len(starts), -1, np.int64)
        track[kept] = np.arange(int(kept.sum()))
        trackOf = np.full(self.N, -1, np.int32)
        trackOf[g] = track[run]
        sel = kept[run]
        members = np.stack([image[sel], g[sel] - base[image[sel]]], 1).astype(np.int32)
        offsets = np.concatenate([[0], np.cumsum(size[kept])]).astype(np.int32)
        return 1000 * (time.perf_counter() - t0), (offsets, members, trackOf)

    def free(self):
        for b in self.bufs:
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
        c = Call(cs, *WORKLOADS[name](cs))
        c.run()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                c.run()
        split = {}
        for e in prof.key_averages():
            if e.device_type.name != "CUDA" or "Memcpy" in e.key or "Memset" in e.key:
                continue
            m = re.search(r"tracks_([a-z]+)_kernel", e.key)
            key = m.group(1) if m else "cub_sort" if "Radix" in e.key else e.key[:40]
            split[key] = split.get(key, 0.0) + e.device_time_total / args.reps
        out[name] = {k: round(v, 1) for k, v in split.items()}
        c.free()
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=3)
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
        c = Call(cs, *WORKLOADS[name](cs))
        c.run()
        times = [c.run()[0] for _ in range(args.reps)]
        T = c.run()[1]
        got = c.outputs(T)
        host = [c.host_path() for _ in range(args.host_reps)]
        ms, hms = float(np.median(times)), float(np.median([h[0] for h in host]))
        same = all(x.tobytes() == y.tobytes() for x, y in zip(got, host[0][1]))
        res[name] = {"images": len(c.sizes), "features": c.N, "lists": len(c.lists), "pairs": c.P,
                     "call_ms": round(ms, 3), "pairs_per_s": float("%.4g" % (c.P / ms * 1000)),
                     "host_path_ms": round(hms, 1), "speedup": round(hms / ms, 1), "identical": bool(same),
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
    out = {"metric": "cs_build_tracks against the host path (ms; call: median of its CUDA events, host path: host clock)",
           "card": card(), "reps": args.reps, "workloads": res}
    for name, r in res.items():
        sys.stderr.write("%-10s pairs %9d call %9.3f ms (%.3g pairs/s) host %9.1f ms x%7.1f %s %s\n" % (
            name, r["pairs"], r["call_ms"], r["pairs_per_s"], r["host_path_ms"], r["speedup"],
            "identical" if r["identical"] else "DIFFERENT", r["kernel_split_us"]))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
