"""CPU checks of batched verification (cs_verify_pairs_batch, cs_verify_essential_batch): the entry points exist and are
typed, every invalid argument is rejected with the offending job's index before any CUDA call, empty batches return 0
without a device, and the Python wrappers pass their arguments through."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("cs_verify_pairs_batch", "cs_verify_essential_batch")
CS_E_ARG = -2
REC = 576
K = np.array([[1200.0, 0, 960], [0, 1200.0, 540], [0, 0, 1]])


def test_symbols_declared_exported_and_typed():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for name in NEW:
        assert name in declared and name in exported, name
        f = getattr(cs.lib(), name)
        assert f.restype is ctypes.c_int and f.argtypes, name
    assert len(cs.lib().cs_verify_pairs_batch.argtypes) == 9
    assert len(cs.lib().cs_verify_essential_batch.argtypes) == 12
    assert "typedef struct cs_verify_job" in header
    assert ctypes.sizeof(cs.VerifyJob) == 72               # 4 x (pointer, int) padded to 16, and the seed
    for name in ("VerifyPairsBatch", "VerifyEssentialBatch"):
        assert name in cs.__all__ and callable(getattr(cs, name)), name


class Arena:
    """Host memory laid out as a batch would be on the device: set A (6 records), set B (5 records), then room for three
    jobs' pairs (4 each) and inliers (4 each), 8-byte aligned.  Nothing is ever dereferenced: every case fails its
    argument checks, or has no pairs."""

    def __init__(self):
        self.buf = np.zeros(11 * REC + 6 * 32 + 64, np.uint8)
        base = self.buf.ctypes.data + (-self.buf.ctypes.data) % 16
        self.A, self.B = base, base + 6 * REC
        self.pairs = [base + 11 * REC + 32 * k for k in range(3)]
        self.inl = [base + 11 * REC + 96 + 32 * k for k in range(3)]

    def jobs(self):
        """Three valid jobs: A-B, B-A and A paired with itself (shared sets are allowed: they are only read)."""
        sets = [(self.A, 6, self.B, 5), (self.B, 5, self.A, 6), (self.A, 6, self.A, 6)]
        return [dict(s1=s1, n1=n1, s2=s2, n2=n2, pairs=self.pairs[k], numPairs=4, seed=k, inliers=self.inl[k],
                     maxInliers=4) for k, (s1, n1, s2, n2) in enumerate(sets)]


def _table(jobs):
    t = (cs.VerifyJob * max(len(jobs), 1))()
    for k, j in enumerate(jobs):
        t[k] = cs.VerifyJob(j["s1"], j["n1"], j["s2"], j["n2"], j["pairs"], j["numPairs"], j["seed"], j["inliers"],
                            j["maxInliers"])
    return t


def _cases(a):
    """(what, job changes {index: fields}, common changes, the job index the message must name or None)"""
    A, B = a.A, a.B
    return [
        ("n1 < 0", {1: dict(n1=-1)}, {}, 1), ("NULL set 2", {2: dict(s2=None)}, {}, 2),
        ("numPairs < 0", {0: dict(numPairs=-3)}, {}, 0), ("NULL pairs", {2: dict(pairs=None)}, {}, 2),
        ("maxInliers < 0", {1: dict(maxInliers=-1)}, {}, 1), ("NULL inliers", {1: dict(inliers=None)}, {}, 1),
        ("pairs unaligned", {2: dict(pairs=a.pairs[2] + 4)}, {}, 2),
        ("inliers unaligned", {0: dict(inliers=a.inl[0] + 4)}, {}, 0),
        ("inliers inside its own set", {1: dict(inliers=B + REC)}, {}, 1),
        ("inliers over its own pairs", {2: dict(inliers=a.pairs[2] + 8)}, {}, 2),
        ("numLoops 0", {}, dict(loops=0), 0), ("numLoops 65537", {}, dict(loops=65537), 0),
        ("thresh NaN", {}, dict(thresh=float("nan")), 0), ("thresh 0", {}, dict(thresh=0.0), 0),
        # across jobs: an inlier buffer against another job's inliers, records and pairs
        ("inliers over another job's inliers", {2: dict(inliers=a.inl[0] + 8, maxInliers=2)}, {}, 0),
        ("inliers over another job's records", {1: dict(inliers=A + 2 * REC)}, {}, 1),
        ("inliers over another job's pairs", {0: dict(inliers=a.pairs[2], maxInliers=1)}, {}, 0),
        ("numJobs < 0", {}, dict(numJobs=-1), None), ("numJobs 65537", {}, dict(numJobs=65537), None),
        ("NULL jobs", {}, dict(table=None), None),
    ]


def _call_pairs(a, jobs, common, outs):
    t = _table(jobs)
    J = common.get("numJobs", len(jobs))
    ms = ctypes.c_double(-1.0)
    r = cs.lib().cs_verify_pairs_batch(ctypes.addressof(t) if common.get("table", 1) else None, J,
                                       common.get("model", 2), common.get("loops", 64), common.get("thresh", 2.0),
                                       outs.get("models"), outs.get("counts"), outs.get("stats"), ctypes.byref(ms))
    return r, ms.value


def _call_essential(a, jobs, common, outs, k1=None, k2=None):
    t = _table(jobs)
    J = common.get("numJobs", len(jobs))
    ms = ctypes.c_double(-1.0)
    r = cs.lib().cs_verify_essential_batch(ctypes.addressof(t) if common.get("table", 1) else None, J, k1, k2,
                                           common.get("loops", 64), common.get("thresh", 2.0), outs.get("E"),
                                           outs.get("R"), outs.get("t"), outs.get("counts"), outs.get("stats"),
                                           ctypes.byref(ms))
    return r, ms.value


def _expect_arg(r, ms, what, job):
    assert r == CS_E_ARG, (what, r)
    msg = cs.lib().cs_last_error().decode()
    assert "invalid argument" in msg and "CS_E_ARG" in msg, (what, msg)
    if job is not None:
        assert "jobs[%d]" % job in msg, (what, msg)
    assert ms == 0.0, what


def _apply(a, change):
    jobs = a.jobs()
    for k, f in change.items():
        jobs[k].update(f)
    return jobs


def test_pairs_batch_rejects_every_invalid_argument():
    a = Arena()
    models, counts, stats = np.full(27, 7.0), np.full(3, 7, np.int32), np.full(24, 7, np.int64)
    outs = dict(models=models.ctypes.data, counts=counts.ctypes.data, stats=stats.ctypes.data)
    for what, change, common, job in _cases(a) + [("model 3", {}, dict(model=3), 0)]:
        _expect_arg(*_call_pairs(a, _apply(a, change), common, outs), what, job)
    for drop in ("models", "counts"):
        _expect_arg(*_call_pairs(a, a.jobs(), {}, dict(outs, **{drop: None})), "NULL " + drop, None)
    assert not a.buf.any() and (models == 7.0).all() and (counts == 7).all() and (stats == 7).all()


def test_essential_batch_rejects_every_invalid_argument():
    a = Arena()
    Ks = np.ascontiguousarray(np.broadcast_to(K.reshape(9), (3, 9)))
    bad = Ks.copy()
    bad[1, 8] = 2.0
    nan = Ks.copy()
    nan[2, 0] = np.nan
    E, R, t = np.full(27, 7.0), np.full(27, 7.0), np.full(9, 7.0)
    counts, stats = np.full(3, 7, np.int32), np.full(30, 7, np.int64)
    outs = dict(E=E.ctypes.data, R=R.ctypes.data, t=t.ctypes.data, counts=counts.ctypes.data, stats=stats.ctypes.data)
    k = Ks.ctypes.data
    for what, change, common, job in _cases(a):
        _expect_arg(*_call_essential(a, _apply(a, change), common, outs, k, k), what, job)
    _expect_arg(*_call_essential(a, a.jobs(), {}, outs, None, k), "NULL K1s", None)
    _expect_arg(*_call_essential(a, a.jobs(), {}, outs, k, None), "NULL K2s", None)
    _expect_arg(*_call_essential(a, a.jobs(), {}, outs, k, bad.ctypes.data), "K2s[1][8] = 2", 1)
    _expect_arg(*_call_essential(a, a.jobs(), {}, outs, nan.ctypes.data, k), "K1s[2] NaN", 2)
    for drop in ("E", "R", "t", "counts"):
        _expect_arg(*_call_essential(a, a.jobs(), {}, dict(outs, **{drop: None}), k, k), "NULL " + drop, None)
    assert not a.buf.any() and (E == 7.0).all() and (counts == 7).all() and (stats == 7).all()


def test_total_pair_count_above_int_max():
    """Three jobs of 2^30 pairs each (addresses that are never read): the running total passes INT_MAX at job 1."""
    base = 1 << 44
    jobs = [dict(s1=None, n1=0, s2=None, n2=0, pairs=base + (k << 34), numPairs=1 << 30, seed=0, inliers=None,
                 maxInliers=0) for k in range(3)]
    models, counts = np.zeros(27), np.zeros(3, np.int32)
    r, ms = _call_pairs(None, jobs, {}, dict(models=models.ctypes.data, counts=counts.ctypes.data))
    _expect_arg(r, ms, "total > INT_MAX", 1)
    assert "INT_MAX" in cs.lib().cs_last_error().decode()
    Ks = np.ascontiguousarray(np.broadcast_to(K.reshape(9), (3, 9)))
    E, counts = np.zeros(27), np.zeros(3, np.int32)
    r, ms = _call_essential(None, jobs, {}, dict(E=E.ctypes.data, R=E.ctypes.data, t=E.ctypes.data,
                                                 counts=counts.ctypes.data), Ks.ctypes.data, Ks.ctypes.data)
    _expect_arg(r, ms, "total > INT_MAX (E)", 1)


def test_empty_batches_return_zero_before_any_cuda_call():
    """numJobs == 0 (NULL outputs allowed), and jobs that all have no pairs: zero models, counts and statistics, and no
    device is needed.  Shared and self-paired record sets are accepted."""
    a = Arena()
    ms = ctypes.c_double(-1.0)
    assert cs.lib().cs_verify_pairs_batch(None, 0, 2, 64, 2.0, None, None, None, ctypes.byref(ms)) == 0
    assert ms.value == 0.0
    assert cs.lib().cs_verify_essential_batch(None, 0, None, None, 64, 2.0, None, None, None, None, None, None) == 0
    jobs = a.jobs()
    for j in jobs:
        j.update(numPairs=0, pairs=None)
    models, counts, stats = np.full(27, 7.0), np.full(3, 7, np.int32), np.full(24, 7, np.int64)
    r, ms = _call_pairs(a, jobs, {}, dict(models=models.ctypes.data, counts=counts.ctypes.data, stats=stats.ctypes.data))
    assert r == 0 and ms == 0.0 and not models.any() and not counts.any() and not stats.any()
    Ks = np.ascontiguousarray(np.broadcast_to(K.reshape(9), (3, 9)))
    E, R, t = np.full(27, 7.0), np.full(27, 7.0), np.full(9, 7.0)
    counts, stats = np.full(3, 7, np.int32), np.full(30, 7, np.int64)
    r, ms = _call_essential(a, jobs, {}, dict(E=E.ctypes.data, R=R.ctypes.data, t=t.ctypes.data,
                                              counts=counts.ctypes.data, stats=stats.ctypes.data),
                            Ks.ctypes.data, Ks.ctypes.data)
    assert r == 0 and not E.any() and not R.any() and not t.any() and not counts.any() and not stats.any()
    # stats_out may be NULL
    r, _ = _call_pairs(a, jobs, {}, dict(models=models.ctypes.data, counts=counts.ctypes.data))
    assert r == 0


class _FakeLib:
    """Records the calls the wrappers make (the job table decoded at call time) instead of reaching the library."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            if name in ("cs_verify_pairs_batch", "cs_verify_essential_batch"):
                J = args[1]
                table = [cs.VerifyJob.from_address(args[0] + k * ctypes.sizeof(cs.VerifyJob)) for k in range(J)]
                jobs = [(j.s1, j.n1, j.s2, j.n2, j.pairs, j.numPairs, j.seed, j.inliers, j.maxInliers) for j in table]
                counts = args[6] if name == "cs_verify_pairs_batch" else args[9]
                c = (ctypes.c_int * J).from_address(counts.value)
                for k in range(J):
                    c[k] = min(jobs[k][5], 2)
                self.calls.append((name, args, jobs))
                return 0
            self.calls.append((name, args, None))
            if name == "cs_device_alloc":
                return 4096 * (1 + len(self.calls))
            return 0
        return f


def _data(n, ptr):
    d = cs.SiftData()
    d.numPts = n
    d._buf = type("B", (), {"ptr": ptr})()
    return d


def test_wrappers_map_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    d1, d2 = _data(7, 1 << 20), _data(5, 1 << 21)
    p0 = np.array([[0, 1], [2, 3], [4, 4]], np.int64)
    p2 = np.array([[1, 1], [3, 0], [5, 2], [6, 4], [0, 0]], np.int32)
    jobs = [(d1, d2, p0, 11), (d2, d2, np.zeros((0, 2), np.int32)), (d1, d1, p2, 2 ** 63 + 5)]
    models, inl, stats, ms = cs.VerifyPairsBatch(jobs, model="homography", numLoops=100, thresh=1.5)
    (name, a, table), = [c for c in fake.calls if c[0] == "cs_verify_pairs_batch"]
    assert a[1] == 3 and a[2] == 1 and a[3] == 100 and a[4] == pytest.approx(1.5)
    # one pair buffer and one inlier buffer, each job's pointers at its offset in them
    uploads = [c for c in fake.calls if c[0] == "cs_memcpy_h2d"]
    assert len(uploads) == 1 and uploads[0][1][2] == 8 * 8
    (s1, n1, s2, n2, pp0, k0, seed0, ii0, m0), j1, (_, _, _, _, pp2, k2, seed2, ii2, m2) = table
    assert (s1, n1, s2, n2) == (1 << 20, 7, 1 << 21, 5) and j1[:4] == (1 << 21, 5, 1 << 21, 5)
    assert (k0, m0, seed0) == (3, 3, 11) and (k2, m2, seed2) == (5, 5, 2 ** 63 + 5)
    assert j1[4] is None and j1[5] == 0 and j1[6] == 0 and j1[7] is None and j1[8] == 0
    assert pp2 - pp0 == 24 and ii2 - ii0 == 24 and ii0 != pp0
    assert models.shape == (3, 3, 3) and models.dtype == np.float64 and stats.shape == (3, 8)
    assert [x.shape for x in inl] == [(2, 2), (0, 2), (2, 2)] and all(x.dtype == np.int32 for x in inl)
    fake.calls.clear()
    cs.VerifyPairsBatch([(d1, d2, p0)])                                  # defaults: F, 4096 trials, 4 px, seed 0
    (name, a, table), = [c for c in fake.calls if c[0] == "cs_verify_pairs_batch"]
    assert a[2] == 2 and a[3] == 4096 and a[4] == pytest.approx(4.0) and table[0][6] == 0
    with pytest.raises(ValueError):
        cs.VerifyPairsBatch([(d1, d2, p0)], model="essential")
    with pytest.raises(ValueError):
        cs.VerifyPairsBatch([(d1, d2)])
    fake.calls.clear()
    k2s = np.stack([K, 2 * K, 3 * K])
    E, R, t, inl, stats, ms = cs.VerifyEssentialBatch(jobs, K, k2s, numLoops=77, thresh=2.5)
    (name, a, table), = [c for c in fake.calls if c[0] == "cs_verify_essential_batch"]
    assert a[1] == 3 and a[4] == 77 and a[5] == pytest.approx(2.5)
    k1 = np.ctypeslib.as_array((ctypes.c_double * 27).from_address(a[2].value)).reshape(3, 9)
    assert k1.shape == (3, 9) and len(table) == 3 and table[2][6] == 2 ** 63 + 5
    assert E.shape == (3, 3, 3) and R.shape == (3, 3, 3) and t.shape == (3, 3) and stats.shape == (3, 10)
    assert [x.shape for x in inl] == [(2, 2), (0, 2), (2, 2)]
    fake.calls.clear()
    out = cs.VerifyPairsBatch([])
    assert out[0].shape == (0, 3, 3) and out[1] == [] and out[2].shape == (0, 8)
