"""CPU checks of batched ratio matching (cs_match_ratio_batch): the entry point exists and is typed, every invalid argument
is rejected with the offending job or set named before any CUDA call, empty batches return 0 without a device, shared
and self-paired sets pass the overlap sweep, and the Python wrapper builds its tables as documented."""
import ctypes
import os
import re
import subprocess

import numpy as np

import cudasift_b200 as cs
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_E_ARG = -2
REC = 576


def test_symbol_declared_exported_and_typed():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert "cs_match_ratio_batch" in declared and "cs_match_ratio_batch" in exported
    f = cs.lib().cs_match_ratio_batch
    assert f.restype is ctypes.c_int and len(f.argtypes) == 10
    assert "typedef struct cs_match_set" in header and "typedef struct cs_match_job" in header
    assert ctypes.sizeof(cs.MatchSet) == 16 and ctypes.sizeof(cs.MatchJob) == 24
    assert "MatchSiftDataRatioBatch" in cs.__all__ and callable(cs.MatchSiftDataRatioBatch)


class Arena:
    """Host memory laid out as on the device: set A (6 records), set B (5 records), then three pair buffers of 4 pairs,
    8-byte aligned.  Nothing is dereferenced: every case fails its checks or has only empty jobs."""

    def __init__(self):
        self.buf = np.zeros(11 * REC + 3 * 32 + 64, np.uint8)
        base = self.buf.ctypes.data + (-self.buf.ctypes.data) % 16
        self.A, self.B = base, base + 6 * REC
        self.pairs = [base + 11 * REC + 32 * k for k in range(3)]

    def sets(self):
        return [dict(pts=self.A, n=6), dict(pts=self.B, n=5), dict(pts=self.A + REC, n=3)]   # set 2 overlaps set 0

    def jobs(self):
        return [dict(set1=0, set2=1, pairs=self.pairs[0], maxPairs=4), dict(set1=1, set2=1, pairs=self.pairs[1],
                maxPairs=4), dict(set1=2, set2=0, pairs=self.pairs[2], maxPairs=4)]


def _call(sets, jobs, common=None, counts=None, stats=None):
    common = common or {}
    st = (cs.MatchSet * max(len(sets), 1))(*[cs.MatchSet(s["pts"], s["n"]) for s in sets])
    jt = (cs.MatchJob * max(len(jobs), 1))(*[cs.MatchJob(j["set1"], j["set2"], j["pairs"], j["maxPairs"]) for j in jobs])
    if counts is None:
        counts = np.full(max(len(jobs), 1), 7, np.int32)
    ms = ctypes.c_double(-1.0)
    r = cs.lib().cs_match_ratio_batch(st if common.get("sets", 1) else None, common.get("numSets", len(sets)),
                                      jt if common.get("jobs", 1) else None, common.get("numJobs", len(jobs)),
                                      common.get("ratio", 0.8), common.get("dist", 0.7), 1,
                                      counts.ctypes.data if common.get("counts", 1) else None,
                                      stats.ctypes.data if stats is not None else None, ctypes.byref(ms))
    return r, ms.value


def _expect(r, ms, what, name):
    assert r == CS_E_ARG, (what, r)
    msg = cs.lib().cs_last_error().decode()
    assert "invalid argument" in msg and "CS_E_ARG" in msg, (what, msg)
    if name:
        assert name in msg, (what, msg)
    assert ms == 0.0, what


def test_rejects_every_invalid_argument():
    a = Arena()
    A, B = a.A, a.B
    cases = [
        ("set n < 0", {1: dict(n=-1)}, {}, {}, "sets[1]"),
        ("NULL set with records", {2: dict(pts=None)}, {}, {}, "sets[2]"),
        ("set1 out of range", {}, {1: dict(set1=3)}, {}, "jobs[1]"),
        ("set2 negative", {}, {2: dict(set2=-1)}, {}, "jobs[2]"),
        ("maxPairs < 0", {}, {0: dict(maxPairs=-1)}, {}, "jobs[0]"),
        ("NULL pairs", {}, {2: dict(pairs=None)}, {}, "jobs[2]"),
        ("pairs unaligned", {}, {1: dict(pairs=a.pairs[1] + 4)}, {}, "jobs[1]"),
        ("pairs over another job's pairs", {}, {2: dict(pairs=a.pairs[0] + 8)}, {}, "jobs[0].pairs and jobs[2].pairs"),
        ("pairs over a set's records", {}, {1: dict(pairs=B + REC)}, {}, "jobs[1].pairs and sets[1].pts"),
        ("pairs over an unused set's records", {}, {0: dict(pairs=A + 2 * REC, maxPairs=1)}, {}, "jobs[0].pairs"),
        ("maxRatio NaN", {}, {}, dict(ratio=float("nan")), None),
        ("maxDistance NaN", {}, {}, dict(dist=float("nan")), None),
        ("numJobs < 0", {}, {}, dict(numJobs=-1), "numJobs"),
        ("numJobs 65537", {}, {}, dict(numJobs=65537), "numJobs"),
        ("numSets 65537", {}, {}, dict(numSets=65537), "numSets"),
        ("numSets < 0", {}, {}, dict(numSets=-1), "numSets"),
        ("NULL jobs", {}, {}, dict(jobs=0), "jobs"),
        ("NULL sets", {}, {}, dict(sets=0), "sets"),
        ("NULL counts_out", {}, {}, dict(counts=0), "counts_out"),
    ]
    for what, sch, jch, common, name in cases:
        sets, jobs = a.sets(), a.jobs()
        for k, f in sch.items():
            sets[k].update(f)
        for k, f in jch.items():
            jobs[k].update(f)
        counts = np.full(3, 7, np.int32)
        _expect(*_call(sets, jobs, common, counts), what, name)
        assert (counts == 7).all(), what
    assert not a.buf.any()


def test_empty_batches_return_zero_before_any_cuda_call():
    a = Arena()
    ms = ctypes.c_double(-1.0)
    assert cs.lib().cs_match_ratio_batch(None, 0, None, 0, 0.8, 0.7, 1, None, None, ctypes.byref(ms)) == 0
    assert ms.value == 0.0
    sets = a.sets() + [dict(pts=None, n=0)]
    jobs = [dict(set1=3, set2=0, pairs=a.pairs[0], maxPairs=4), dict(set1=1, set2=3, pairs=None, maxPairs=0),
            dict(set1=3, set2=3, pairs=a.pairs[2], maxPairs=4)]
    counts, stats = np.full(3, 7, np.int32), np.full((3, 4), 7, np.uint64)
    r, ms = _call(sets, jobs, {}, counts, stats)
    assert r == 0 and ms == 0.0 and not counts.any() and not stats.any()
    r, _ = _call(sets, jobs, {}, counts)                                 # stats_out may be NULL
    assert r == 0


def test_overlap_sweep_accepts_shared_and_self_paired_sets():
    """Overlapping record sets, sets shared by several jobs, (a, a) jobs and pair buffers that touch records or each
    other without overlapping pass the sweep.  Every job names the empty set 3, so the call then needs no device."""
    a = Arena()
    sets = a.sets() + [dict(pts=None, n=0)]                              # set 2 overlaps set 0
    jobs = [dict(set1=3, set2=0, pairs=a.B + 5 * REC, maxPairs=4),      # right after set B's last record
            dict(set1=1, set2=3, pairs=a.B + 5 * REC + 32, maxPairs=4),  # right after job 0's buffer
            dict(set1=3, set2=3, pairs=a.pairs[2], maxPairs=4), dict(set1=3, set2=2, pairs=None, maxPairs=0)]
    counts = np.full(len(jobs), 7, np.int32)
    assert _call(sets, jobs, {}, counts)[0] == 0 and not counts.any()
    jobs[0]["pairs"] = a.B + 5 * REC - 8                                 # one pair over set B's last record
    _expect(*_call(sets, jobs), "pairs over set B's last record", "jobs[0].pairs and sets[1].pts")


class _FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            if name == "cs_match_ratio_batch":
                S, J = args[1], args[3]
                sets = [cs.MatchSet.from_address(args[0] + k * ctypes.sizeof(cs.MatchSet)) for k in range(S)]
                jobs = [cs.MatchJob.from_address(args[2] + k * ctypes.sizeof(cs.MatchJob)) for k in range(J)]
                c = (ctypes.c_int * J).from_address(args[7].value)
                for k in range(J):
                    c[k] = min(jobs[k].maxPairs, 2)
                self.calls.append((name, args, [(s.pts, s.n) for s in sets],
                                   [(j.set1, j.set2, j.pairs, j.maxPairs) for j in jobs]))
                return 0
            self.calls.append((name, args, None, None))
            if name == "cs_device_alloc":
                return 4096 * (1 + len(self.calls))
            return 0
        return f


def _data(n, ptr):
    d = cs.SiftData()
    d.numPts = n
    d._buf = type("B", (), {"ptr": ptr})()
    return d


def test_wrapper_maps_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    datas = [_data(7, 1 << 20), _data(5, 1 << 21), _data(0, 1 << 22)]
    jobs = [(0, 1), (1, 1), (2, 0), (1, 0)]
    pairs, stats, ms = cs.MatchSiftDataRatioBatch(datas, jobs, maxRatio=0.6, maxDistance=0.5, crossCheck=True)
    (name, a, sets, table), = [c for c in fake.calls if c[0] == "cs_match_ratio_batch"]
    assert sets == [(1 << 20, 7), (1 << 21, 5), (1 << 22, 0)]
    assert a[1] == 3 and a[3] == 4 and a[4] == 0.6 and a[5] == 0.5 and a[6] == 1
    rooms = [5, 5, 0, 5]                                                 # min(n1, n2) with the cross-check
    assert [t[3] for t in table] == rooms and [t[:2] for t in table] == jobs
    (alloc,) = [c for c in fake.calls if c[0] == "cs_device_alloc"]
    assert alloc[1][0] == 8 * sum(rooms)                                 # one device buffer for every pair list
    base = table[0][2]
    assert table[1][2] - base == 40 and table[2][2] is None and table[3][2] - base == 80
    assert [p.shape for p in pairs] == [(2, 2), (2, 2), (0, 2), (2, 2)] and all(p.dtype == np.int32 for p in pairs)
    assert stats.shape == (4, 4) and stats.dtype == np.uint64
    fake.calls.clear()
    cs.MatchSiftDataRatioBatch(datas, [(0, 1)], crossCheck=False)       # without the cross-check: n1 rows of room
    (name, a, sets, table), = [c for c in fake.calls if c[0] == "cs_match_ratio_batch"]
    assert table[0][3] == 7 and a[6] == 0 and a[4] == 0.8 and a[5] == 0.7
    fake.calls.clear()
    pairs, stats, _ = cs.MatchSiftDataRatioBatch(datas, [])
    assert pairs == [] and stats.shape == (0, 4)
