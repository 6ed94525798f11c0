"""CPU checks of batched guided matching (cs_match_guided_batch): the entry point exists and is typed, every invalid
argument is rejected with the offending job or set named before any CUDA call, empty batches return 0 without a
device, shared and self-paired sets pass the overlap sweep, and the Python wrapper builds its tables and broadcasts
its model as documented."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
from cudasift_b200 import build
from test_match_batch_cpu import REC, Arena, _data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_E_ARG = -2
H, F = 1, 2


def test_symbol_declared_exported_and_typed():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert "cs_match_guided_batch" in declared and "cs_match_guided_batch" in exported
    f = cs.lib().cs_match_guided_batch
    assert f.restype is ctypes.c_int and len(f.argtypes) == 13
    assert "MatchSiftDataGuidedBatch" in cs.__all__ and callable(cs.MatchSiftDataGuidedBatch)


def _call(sets, jobs, common=None, models=None, Ms=None, counts=None, stats=None):
    common = common or {}
    J = len(jobs)
    st = (cs.MatchSet * max(len(sets), 1))(*[cs.MatchSet(s["pts"], s["n"]) for s in sets])
    jt = (cs.MatchJob * max(J, 1))(*[cs.MatchJob(j["set1"], j["set2"], j["pairs"], j["maxPairs"]) for j in jobs])
    models = np.array(models if models is not None else [F] * max(J, 1), np.int32)
    Ms = np.array(Ms if Ms is not None else [np.eye(3).ravel()] * max(J, 1), np.float64)
    if counts is None:
        counts = np.full(max(J, 1), 7, np.int32)
    ms = ctypes.c_double(-1.0)
    r = cs.lib().cs_match_guided_batch(st if common.get("sets", 1) else None, common.get("numSets", len(sets)),
                                       jt if common.get("jobs", 1) else None, common.get("numJobs", J),
                                       models.ctypes.data if common.get("models", 1) else None,
                                       Ms.ctypes.data if common.get("models_in", 1) else None,
                                       common.get("thresh", 4.0), common.get("ratio", 0.8), common.get("dist", 0.7), 1,
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
    eye = np.eye(3).ravel()
    nan = eye.copy()
    nan[4] = np.nan
    big = eye * 1e200                                                     # entries finite, the norm is not
    cases = [
        # the rules of cs_match_ratio_batch
        ("set n < 0", {1: dict(n=-1)}, {}, {}, {}, "sets[1]"),
        ("NULL set with records", {2: dict(pts=None)}, {}, {}, {}, "sets[2]"),
        ("set1 out of range", {}, {1: dict(set1=3)}, {}, {}, "jobs[1]"),
        ("set2 negative", {}, {2: dict(set2=-1)}, {}, {}, "jobs[2]"),
        ("maxPairs < 0", {}, {0: dict(maxPairs=-1)}, {}, {}, "jobs[0]"),
        ("NULL pairs", {}, {2: dict(pairs=None)}, {}, {}, "jobs[2]"),
        ("pairs unaligned", {}, {1: dict(pairs=a.pairs[1] + 4)}, {}, {}, "jobs[1]"),
        ("pairs over another job's pairs", {}, {2: dict(pairs=a.pairs[0] + 8)}, {}, {}, "jobs[0].pairs and jobs[2].pairs"),
        ("pairs over a set's records", {}, {1: dict(pairs=B + REC)}, {}, {}, "jobs[1].pairs and sets[1].pts"),
        ("pairs over an unused set's records", {}, {0: dict(pairs=A + 2 * REC, maxPairs=1)}, {}, {}, "jobs[0].pairs"),
        ("maxRatio NaN", {}, {}, dict(ratio=float("nan")), {}, None),
        ("maxDistance NaN", {}, {}, dict(dist=float("nan")), {}, None),
        ("numJobs < 0", {}, {}, dict(numJobs=-1), {}, "numJobs"),
        ("numJobs 65537", {}, {}, dict(numJobs=65537), {}, "numJobs"),
        ("numSets 65537", {}, {}, dict(numSets=65537), {}, "numSets"),
        ("numSets < 0", {}, {}, dict(numSets=-1), {}, "numSets"),
        ("NULL jobs", {}, {}, dict(jobs=0), {}, "jobs"),
        ("NULL sets", {}, {}, dict(sets=0), {}, "sets"),
        ("NULL counts_out", {}, {}, dict(counts=0), {}, "counts_out"),
        # the model rules
        ("NULL models", {}, {}, dict(models=0), {}, "models"),
        ("NULL models_in", {}, {}, dict(models_in=0), {}, "models_in"),
        ("model 0", {}, {}, {}, dict(models={1: 0}), "jobs[1]"),
        ("model 3", {}, {}, {}, dict(models={2: 3}), "jobs[2]"),
        ("zero model", {}, {}, {}, dict(Ms={1: np.zeros(9)}), "jobs[1]"),
        ("NaN model", {}, {}, {}, dict(Ms={2: nan}), "jobs[2]"),
        ("infinite model", {}, {}, {}, dict(Ms={0: np.where(eye > 0, np.inf, 0.0)}), "jobs[0]"),
        ("model norm not finite", {}, {}, {}, dict(Ms={1: big}), "jobs[1]"),
        ("thresh 0", {}, {}, dict(thresh=0.0), {}, "jobs[0]"),
        ("thresh NaN", {}, {}, dict(thresh=float("nan")), {}, "jobs[0]"),
        ("thresh inf", {}, {}, dict(thresh=float("inf")), {}, "jobs[0]"),
    ]
    for what, sch, jch, common, mch, name in cases:
        sets, jobs = a.sets(), a.jobs()
        for k, f in sch.items():
            sets[k].update(f)
        for k, f in jch.items():
            jobs[k].update(f)
        models, Ms = [F, H, F], [eye, eye, eye]
        for k, v in mch.get("models", {}).items():
            models[k] = v
        for k, v in mch.get("Ms", {}).items():
            Ms[k] = v
        counts = np.full(3, 7, np.int32)
        _expect(*_call(sets, jobs, common, models, Ms, counts), what, name)
        assert (counts == 7).all(), what
    assert not a.buf.any()


def test_empty_batches_return_zero_before_any_cuda_call():
    a = Arena()
    ms = ctypes.c_double(-1.0)
    assert cs.lib().cs_match_guided_batch(None, 0, None, 0, None, None, 4.0, 0.8, 0.7, 1, None, None,
                                          ctypes.byref(ms)) == 0
    assert ms.value == 0.0
    sets = a.sets() + [dict(pts=None, n=0)]
    jobs = [dict(set1=3, set2=0, pairs=a.pairs[0], maxPairs=4), dict(set1=1, set2=3, pairs=None, maxPairs=0),
            dict(set1=3, set2=3, pairs=a.pairs[2], maxPairs=4)]
    counts, stats = np.full(3, 7, np.int32), np.full((3, 4), 7, np.uint64)
    r, ms = _call(sets, jobs, {}, [F, H, F], None, counts, stats)
    assert r == 0 and ms == 0.0 and not counts.any() and not stats.any()
    r, _ = _call(sets, jobs, {}, [F, H, F], None, counts)                # stats_out may be NULL
    assert r == 0
    # the model of an empty job is still checked, as the single call checks it before returning 0
    _expect(*_call(sets, jobs, {}, [F, H, F], [np.eye(3).ravel(), np.zeros(9), np.eye(3).ravel()]), "zero model",
            "jobs[1]")


def test_overlap_sweep_accepts_shared_and_self_paired_sets():
    """Overlapping record sets, sets shared by several jobs, (a, a) jobs and pair buffers that touch records or each
    other without overlapping pass the sweep.  Every job names the empty set 3, so the call then needs no device."""
    a = Arena()
    sets = a.sets() + [dict(pts=None, n=0)]
    jobs = [dict(set1=3, set2=0, pairs=a.B + 5 * REC, maxPairs=4),
            dict(set1=1, set2=3, pairs=a.B + 5 * REC + 32, maxPairs=4),
            dict(set1=3, set2=3, pairs=a.pairs[2], maxPairs=4), dict(set1=3, set2=2, pairs=None, maxPairs=0)]
    counts = np.full(len(jobs), 7, np.int32)
    assert _call(sets, jobs, {}, [F, H, F, H], None, counts)[0] == 0 and not counts.any()
    jobs[0]["pairs"] = a.B + 5 * REC - 8
    _expect(*_call(sets, jobs, {}, [F, H, F, H]), "pairs over set B's last record", "jobs[0].pairs and sets[1].pts")


class _FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            if name == "cs_match_guided_batch":
                S, J = args[1], args[3]
                sets = [cs.MatchSet.from_address(args[0] + k * ctypes.sizeof(cs.MatchSet)) for k in range(S)]
                jobs = [cs.MatchJob.from_address(args[2] + k * ctypes.sizeof(cs.MatchJob)) for k in range(J)]
                models = list((ctypes.c_int * J).from_address(args[4].value)) if J else []
                Ms = np.array((ctypes.c_double * (9 * J)).from_address(args[5].value)) if J else np.zeros(0)
                c = (ctypes.c_int * J).from_address(args[10].value)
                for k in range(J):
                    c[k] = min(jobs[k].maxPairs, 2)
                self.calls.append((name, args, [(s.pts, s.n) for s in sets],
                                   [(j.set1, j.set2, j.pairs, j.maxPairs) for j in jobs], models, Ms))
                return 0
            self.calls.append((name, args, None, None, None, None))
            if name == "cs_device_alloc":
                return 4096 * (1 + len(self.calls))
            return 0
        return f


def test_wrapper_maps_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    datas = [_data(7, 1 << 20), _data(5, 1 << 21), _data(0, 1 << 22)]
    jobs = [(0, 1), (1, 1), (2, 0), (1, 0)]
    Ms = np.arange(36, dtype=np.float64).reshape(4, 3, 3) + 1
    pairs, stats, ms = cs.MatchSiftDataGuidedBatch(datas, jobs, ["fundamental", "homography", 2, 1], Ms, thresh=3.0,
                                                   maxRatio=0.6, maxDistance=0.5, crossCheck=True)
    (name, a, sets, table, models, M), = [c for c in fake.calls if c[0] == "cs_match_guided_batch"]
    assert sets == [(1 << 20, 7), (1 << 21, 5), (1 << 22, 0)]
    assert a[1] == 3 and a[3] == 4 and a[6] == 3.0 and a[7] == pytest.approx(0.6) and a[8] == 0.5 and a[9] == 1
    assert models == [F, H, F, H] and np.array_equal(M, Ms.ravel())
    rooms = [5, 5, 0, 5]                                                 # min(n1, n2) with the cross-check
    assert [t[3] for t in table] == rooms and [t[:2] for t in table] == jobs
    (alloc,) = [c for c in fake.calls if c[0] == "cs_device_alloc"]
    assert alloc[1][0] == 8 * sum(rooms)                                 # one device buffer for every pair list
    base = table[0][2]
    assert table[1][2] - base == 40 and table[2][2] is None and table[3][2] - base == 80
    assert [p.shape for p in pairs] == [(2, 2), (2, 2), (0, 2), (2, 2)] and all(p.dtype == np.int32 for p in pairs)
    assert stats.shape == (4, 4) and stats.dtype == np.uint64
    fake.calls.clear()
    cs.MatchSiftDataGuidedBatch(datas, [(0, 1), (1, 0)], "homography", Ms[:2], crossCheck=False)   # one model for all
    (name, a, sets, table, models, M), = [c for c in fake.calls if c[0] == "cs_match_guided_batch"]
    assert models == [H, H] and [t[3] for t in table] == [7, 5] and a[9] == 0 and a[6] == 4.0
    assert a[7] == pytest.approx(0.8) and a[8] == pytest.approx(0.7)
    fake.calls.clear()
    pairs, stats, _ = cs.MatchSiftDataGuidedBatch(datas, [], "fundamental", np.zeros((0, 3, 3)))
    assert pairs == [] and stats.shape == (0, 4)
    with pytest.raises(ValueError):
        cs.MatchSiftDataGuidedBatch(datas, [(0, 1)], ["fundamental", "homography"], Ms[:1])
    with pytest.raises(ValueError):
        cs.MatchSiftDataGuidedBatch(datas, [(0, 1)], "affine", Ms[:1])
