"""GPU checks of the tensor matcher (csrc/match_tc.cu) over the case families of tests/tc_cases.py at the schedule
shapes derived from the device's SM count: every rule that runs on it against the CPU oracles, the fallback row count
against the interval the restatement of tests/tc_model.py gives, and the tensor cores' accumulation error measured by a
standalone probe (tests/tc_accum_probe.cu) against the budget the error bound gives it."""
import ctypes
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import knn_oracle
import oracle
import tc_cases as tc
import tc_model as tm
from cudasift_b200.synth import synth_descriptors
from test_mutual_gpu import cross_check

pytestmark = pytest.mark.gpu
ALL_EXACT = (1 << 64) - 1
FIELDS = ("score", "ambiguity", "match", "match_xpos", "match_ypos")
H100_SMS = 132            # the shapes are listed for it; the tests derive them from the device's count


@functools.lru_cache(maxsize=None)
def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _shapes():
    return tc.shapes(H100_SMS)


def _eq(a, b, what):
    for f in FIELDS:
        assert a[f].tobytes() == b[f].tobytes(), "%s: field %s differs in %d rows" % (what, f, int((a[f] != b[f]).sum()))


def _stats_ok(st, family, d, what):
    """The certification decision itself: gated sets go the exact way, the others list a number of fallback rows
    inside the restatement's interval, and the ordinary family lists fewer than 1 %."""
    assert st[3] == 2, (what, st)
    if family == "gated":
        assert st[2] == ALL_EXACT, (what, st)
        return
    lo, hi = d.fallback_bounds()
    assert lo <= st[2] <= hi, (what, st[2], lo, hi)
    if family == "ordinary" and d.n1 >= 100 and d.ncand >= 128:    # fewer candidates: no second neighbour to certify
        assert st[2] < 0.01 * d.n1, (what, st)


SHAPE_IDS = [s[2] for s in tc.shapes(H100_SMS)]


def test_shapes_are_this_devices():
    """The listed shapes hit the seams on this device: its SM count gives the same facts as the H100's."""
    sms = _sms()
    for n1, n2, _ in _shapes():
        if sms != H100_SMS:
            pytest.skip("%d SMs: the shapes are the H100's" % sms)
        assert tc.shape_facts(n1, n2, sms) == tc.shape_facts(n1, n2, H100_SMS)


@pytest.mark.parametrize("shape", SHAPE_IDS)
@pytest.mark.parametrize("family", tc.FAMILIES)
def test_match_equals_oracle(cs, family, shape):
    """MatchSiftData (match_host) on the tensor path equals the oracle in all five fields and the exact path."""
    n1, n2 = map(int, shape.split("x"))
    s1, s2, _ = tc.make(family, n1, n2)
    got, _ = cs.match_host(s1, s2, mode=2)
    st = cs.match_stats()
    want = oracle.match(s1, s2, threads=8)
    _eq(got, want, "%s %s mode 2 vs oracle" % (family, shape))
    _stats_ok(st, family, tm.Direction(s1["data"], s2["data"], knn=False), "%s %s" % (family, shape))
    exact, _ = cs.match_host(s1, s2, mode=1)
    _eq(got, exact, "%s %s mode 2 vs mode 1" % (family, shape))


@pytest.mark.parametrize("shape", SHAPE_IDS)
@pytest.mark.parametrize("family", tc.FAMILIES)
def test_knn2_equals_oracle(cs, family, shape):
    """cs_match_knn2 on the tensor path equals the CPU statement in both directions."""
    n1, n2 = map(int, shape.split("x"))
    s1, s2, _ = tc.make(family, n1, n2)
    for x, y, what in ((s1, s2, "forward"), (s2, s1, "reverse")):
        gi, gs, _ = cs.match_knn2(x, y, mode=2)
        st = cs.match_stats()
        wi, ws = knn_oracle.match_knn2(x, y)
        assert gi.tobytes() == wi.tobytes(), (family, shape, what, int((gi != wi).any(1).sum()))
        assert gs.tobytes() == ws.tobytes(), (family, shape, what)
        _stats_ok(st, family, tm.Direction(x["data"], y["data"], knn=True), "%s %s %s" % (family, shape, what))


def _mutual_sets(family, n1, n2):
    """The family's sets with their tail rows [32 floor(n / 32), n) copies of rows of the other set: a tail row that
    wrongly became a candidate would be the best match of the row it copies."""
    s1, s2, _ = tc.make(family, n1, n2)
    s1, s2 = s1.copy(), s2.copy()
    for x, y in ((s1, s2), (s2, s1)):
        nv = (len(x) // 32) * 32
        for k, r in enumerate(range(nv, len(x))):
            x["data"][r] = y["data"][k]
    return s1, s2


@pytest.mark.parametrize("n1,n2", tc.MUTUAL_SHAPES)
@pytest.mark.parametrize("family", tc.FAMILIES)
def test_mutual_equals_two_oracle_matches(cs, family, n1, n2):
    """MatchSiftDataMutual equals two one-way oracle matches and their cross-check; the shapes give the B-role copy to
    neither, one or both sets."""
    s1, s2 = _mutual_sets(family, n1, n2)
    g1, g2, pairs, _ = cs.match_mutual_host(s1, s2, mode=2)
    st = cs.match_stats()
    w1, w2 = oracle.match(s1, s2, threads=8), oracle.match(s2, s1, threads=8)
    _eq(g1, w1, "%s %dx%d set 1" % (family, n1, n2))
    _eq(g2, w2, "%s %dx%d set 2" % (family, n1, n2))
    assert np.array_equal(pairs, cross_check(w1, w2)), (family, n1, n2)
    assert st[3] == 2
    if family == "gated":
        assert st[2] == ALL_EXACT
    else:
        b1 = tm.Direction(s1["data"], s2["data"], knn=False).fallback_bounds()
        b2 = tm.Direction(s2["data"], s1["data"], knn=False).fallback_bounds()
        assert b1[0] + b2[0] <= st[2] <= b1[1] + b2[1], (st, b1, b2)


class _Sets:
    def __init__(self, cs, arrays):
        self.datas = []
        for a in arrays:
            d = cs.InitSiftData(cs.SiftData(), max(len(a), 1))
            d._buf.upload(a)
            d.numPts = len(a)
            self.datas.append(d)

    def free(self, cs):
        for d in self.datas:
            cs.FreeSiftData(d)


BATCH_SHAPES = [(127, 255), (128, 673), (129, 896), (257, 4095)]


@pytest.mark.parametrize("family", [f for f in tc.FAMILIES if f != "ordinary"])
def test_ratio_batch_mixed_jobs(cs, family):
    """MatchSiftDataRatioBatch with the family's jobs among ordinary ones: every job equals its single call and the
    ratio test on the CPU statement's lists (rows a last-bit arccos difference could flip excepted); per job stats."""
    arrays, jobs, kinds = [], [], []
    for q, (n1, n2) in enumerate(BATCH_SHAPES):
        o1, o2 = synth_descriptors(n1 + 7, 50 + q), synth_descriptors(n2 - 5, 60 + q)
        s1, s2, _ = tc.make(family, n1, n2)
        base = len(arrays)
        arrays += [o1, s1, s2, o2]
        jobs += [(base, base + 3), (base + 1, base + 2), (base + 2, base + 1)]
        kinds += ["ordinary", family, family]
    S = _Sets(cs, arrays)
    try:
        pairs, stats, _ = cs.MatchSiftDataRatioBatch(S.datas, jobs)
        for q, ((a, b), kind) in enumerate(zip(jobs, kinds)):
            single, _ = cs.MatchSiftDataRatio(S.datas[a], S.datas[b])
            assert pairs[q].tobytes() == single.tobytes(), (family, q)
            i1, sc1 = knn_oracle.match_knn2(arrays[a], arrays[b])
            i2, sc2 = knn_oracle.match_knn2(arrays[b], arrays[a])
            want, margin = knn_oracle.ratio_pairs(i1, sc1, i2, sc2, 0.8, 0.7, True)
            if margin > 1e-6:
                assert np.array_equal(pairs[q], want), (family, q)
            gated = kind == "gated" and (tm.gated(arrays[a]["data"]) or tm.gated(arrays[b]["data"]))
            if gated:
                assert stats[q][2] == ALL_EXACT, (q, stats[q])
    finally:
        S.free(cs)


@pytest.mark.parametrize("family", tc.FAMILIES)
def test_assign_words_adversarial_vocabulary(cs, family):
    """AssignWords with the family's set 2 as the vocabulary equals j1 of the CPU statement for every feature."""
    feats, vocab = [], None
    for n1, n2 in ((127, 4095), (257, 4095)):
        s1, s2, _ = tc.make(family, n1, 4095)
        feats.append(s1)
        vocab = s2
    feats.append(synth_descriptors(300, 77))
    S, V = _Sets(cs, feats), _Sets(cs, [vocab])
    try:
        wordOf, stats, _ = cs.AssignWords(S.datas, V.datas[0])
    finally:
        S.free(cs)
        V.free(cs)
    want = np.concatenate([knn_oracle.match_knn2(f, vocab)[0][:, 0] for f in feats])
    assert wordOf.tobytes() == want.tobytes(), (family, int((wordOf != want).sum()))


# ------------------------------------------------------------------------------------------ accumulation probe
def _pack(x):
    """Rows [128][128] -> one operand tile as prep writes it: [hi | lo][chunk][128 rows][8 halves]."""
    hi, lo = tm.split(x)
    part = lambda h: np.ascontiguousarray(h.reshape(128, 16, 8).transpose(1, 0, 2)).view(np.uint16)
    return np.concatenate([part(hi).ravel(), part(lo).ravel()])


@pytest.fixture(scope="module")
def probe(cs):
    from cudasift_b200 import build
    nvcc = build.nvcc_path()
    assert nvcc, "nvcc is needed to build the accumulation probe"
    d = tempfile.mkdtemp(prefix="tc_probe_")
    try:
        so = os.path.join(d, "probe.so")
        subprocess.run([nvcc] + build.ARCH + ["-O3", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                                              os.path.join(os.path.dirname(__file__), "tc_accum_probe.cu")],
                       check=True, capture_output=True)
        L = ctypes.CDLL(so)
        L.probe_run.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        yield L
    finally:
        shutil.rmtree(d, ignore_errors=True)


def test_accumulation_within_budget(cs, probe, record_property):
    """The MMA sequence of t3_gemm_kernel on split-FP16 operands of every ungated family: |accumulator - float64 sum of
    hi*hi + hi*lo + lo*hi| / (|a||b| 2^24) <= 2^-15, the share of T3_C1 the error bound gives the tensor cores."""
    tiles_a, tiles_b, rows_a, rows_b = [], [], [], []
    for family in [f for f in tc.FAMILIES if f != "gated"]:
        s1, s2, _ = tc.make(family, 128, 673)
        for a, b in ((s1["data"][:128], s2["data"][:128]), (s1["data"][:128], s2["data"][128:256])):
            tiles_a.append(_pack(a)); tiles_b.append(_pack(b))
            rows_a.append(a); rows_b.append(b)
    n = len(tiles_a)
    A, B = np.concatenate(tiles_a), np.concatenate(tiles_b)
    bufs = [cs.DeviceBuffer(A.nbytes), cs.DeviceBuffer(B.nbytes), cs.DeviceBuffer(n * 128 * 128 * 4)]
    try:
        bufs[0].upload(A); bufs[1].upload(B)
        assert probe.probe_run(bufs[0].ptr, bufs[1].ptr, bufs[2].ptr, n) == 0
        acc = bufs[2].download(np.float32, n * 128 * 128).reshape(n, 128, 128)
    finally:
        for b in bufs:
            b.free()
    worst = 0.0
    for t in range(n):
        want = tm.approx_scaled(rows_a[t], rows_b[t])
        na = np.sqrt((rows_a[t].astype(np.float64) ** 2).sum(1))[:, None]
        nb = np.sqrt((rows_b[t].astype(np.float64) ** 2).sum(1))[None, :]
        norm = na * nb * 2.0 ** 24
        rel = np.abs(acc[t].astype(np.float64) - want) / np.where(norm > 0, norm, 1.0)
        rel[norm == 0] = np.abs(acc[t][norm == 0])
        worst = max(worst, float(rel.max()))
    record_property("accumulation_rel_error_max", worst)
    print("tensor-core accumulation: max |acc - exact| / (|a||b|) = %.3g (2^%.2f); budget 2^-15" % (worst, np.log2(max(worst, 1e-300))))
    assert worst <= tm.ACCUM_BUDGET, worst
