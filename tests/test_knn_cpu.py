"""CPU checks of two-nearest-neighbour matching (cs_match_knn2, cs_match_ratio, cs_match_ratio_host): the entry points
exist, they reject bad arguments before any CUDA call, the Python wrappers pass their arguments through, the CPU
statement (tests/knn_oracle.c) equals a brute-force numpy chain, and a numpy restatement of the tensor path's top-2
certification rule (the top-2 rule of t3_resolve_kernel in csrc/match_tc.cu) reproduces the oracle on every row it certifies."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
import knn_oracle
from cudasift_b200 import build
from cudasift_b200.synth import synth_descriptors
from test_match_logic_cpu import T3_C1, T3_C2, SCALE, exact_scores, split

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("cs_match_knn2", "cs_match_ratio", "cs_match_ratio_host")
CS_E_ARG = -2
REC = 576


def test_symbols_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for name in NEW:
        assert name in declared and name in exported, name
        assert hasattr(cs.lib(), name)
    for name in ("match_knn2", "MatchSiftDataRatio", "match_ratio_host"):
        assert name in cs.__all__ and callable(getattr(cs, name)), name
    assert build.SOURCES.count("match_knn.cu") == 1


def _layout(base):
    """Two sets of 4 records, then 8-byte aligned room for idx, score and pairs."""
    s1, s2 = base, base + 4 * REC
    out = base + 8 * REC
    return s1, s2, out, out + 64, out + 128


def _knn_bad(base):
    s1, s2, idx, sc, _ = _layout(base)
    return [
        ("n1 < 0", (s1, -1, s2, 4, idx, sc, 0)),
        ("n2 < 0", (s1, 4, s2, -3, idx, sc, 0)),
        ("NULL set 1", (None, 4, s2, 4, idx, sc, 0)),
        ("NULL set 2", (s1, 4, None, 4, idx, sc, 0)),
        ("NULL idx", (s1, 4, s2, 4, None, sc, 0)),
        ("NULL score", (s1, 4, s2, 4, idx, None, 0)),
        ("mode -1", (s1, 4, s2, 4, idx, sc, -1)),
        ("mode 3", (s1, 4, s2, 4, idx, sc, 3)),
        ("idx unaligned", (s1, 4, s2, 4, idx + 4, sc, 0)),
        ("score unaligned", (s1, 4, s2, 4, idx, sc + 4, 0)),
        ("idx inside set 1", (s1, 4, s2, 4, s1 + 64, sc, 0)),
        ("score inside set 2", (s1, 4, s2, 4, idx, s2 + 3 * REC, 0)),
        ("idx ends inside set 1", (s1 + 8, 4, s2, 4, s1, sc, 0)),
        ("idx and score overlap", (s1, 4, s2, 4, idx, idx + 16, 0)),
    ]


def _ratio_bad(base):
    s1, s2, _, _, pairs = _layout(base)
    nan = float("nan")
    return [
        ("n1 < 0", (s1, -1, s2, 4, 0.8, 0.7, 1, pairs, 4, 0)),
        ("n2 < 0", (s1, 4, s2, -3, 0.8, 0.7, 1, pairs, 4, 0)),
        ("NULL set 1", (None, 4, s2, 4, 0.8, 0.7, 1, pairs, 4, 0)),
        ("NULL set 2", (s1, 4, None, 4, 0.8, 0.7, 0, pairs, 4, 0)),
        ("maxPairs < 0", (s1, 4, s2, 4, 0.8, 0.7, 1, pairs, -1, 0)),
        ("NULL pairs", (s1, 4, s2, 4, 0.8, 0.7, 1, None, 4, 0)),
        ("mode -1", (s1, 4, s2, 4, 0.8, 0.7, 1, pairs, 4, -1)),
        ("mode 3", (s1, 4, s2, 4, 0.8, 0.7, 0, pairs, 4, 3)),
        ("NaN maxRatio", (s1, 4, s2, 4, nan, 0.7, 1, pairs, 4, 0)),
        ("NaN maxDistance", (s1, 4, s2, 4, 0.8, nan, 1, pairs, 4, 0)),
        ("pairs unaligned", (s1, 4, s2, 4, 0.8, 0.7, 1, pairs + 4, 4, 0)),
        ("pairs inside set 1", (s1, 4, s2, 4, 0.8, 0.7, 1, s1 + 2 * REC, 4, 0)),
        ("pairs inside set 2", (s1, 4, s2, 4, 0.8, 0.7, 0, s2 + 8, 4, 0)),
    ]


@pytest.mark.parametrize("entry", NEW)
def test_invalid_arguments_return_cs_e_arg(entry):
    """Every invalid argument fails with CS_E_ARG, and *ms is reset, whether or not a device is present."""
    buf = np.zeros(8 * REC + 256 + 16, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    f = getattr(cs.lib(), entry)
    cases = _knn_bad(base) if entry == "cs_match_knn2" else _ratio_bad(base)
    for what, args in cases:
        ms = ctypes.c_double(-1.0)
        assert f(*args, ctypes.byref(ms)) == CS_E_ARG, (entry, what)
        msg = cs.lib().cs_last_error().decode()
        assert "invalid argument" in msg and "CS_E_ARG" in msg, (entry, what, msg)
        assert ms.value == 0.0, (entry, what)
    assert not buf.any()


@pytest.mark.parametrize("entry", NEW)
def test_empty_sets_write_nothing(entry):
    """n1 == 0 or n2 == 0 returns 0 before any CUDA call; an empty set may be NULL, and so may the outputs of an empty
    set 1.  Sets may overlap: they are only read."""
    buf = np.zeros(8 * REC + 256 + 16, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    s1, s2, idx, sc, pairs = _layout(base)
    f = getattr(cs.lib(), entry)
    ms = ctypes.c_double(-1.0)
    if entry == "cs_match_knn2":
        assert f(s1, 0, s2, 4, None, None, 0, ctypes.byref(ms)) == 0 and ms.value == 0.0
        assert f(s1, 4, None, 0, idx, sc, 1, None) == 0
        assert f(None, 0, None, 0, None, None, 2, None) == 0
        assert f(s1, 4, s1, 0, idx, sc, 2, None) == 0                # the same set twice is allowed
    else:
        assert f(s1, 0, s2, 4, 0.8, 0.7, 1, None, 0, 0, ctypes.byref(ms)) == 0 and ms.value == 0.0
        assert f(s1, 4, None, 0, 0.8, 0.7, 0, pairs, 4, 1, None) == 0
        assert f(None, 0, None, 0, 0.8, 0.7, 1, None, 0, 2, None) == 0
        assert f(s1, 0, s1, 4, 0.8, 0.7, 1, pairs, 4, 2, None) == 0
    assert not buf.any()


class _FakeLib:
    """Records the calls the wrappers make instead of reaching the library."""

    def __init__(self, pairs=3):
        self.calls = []
        self.pairs = pairs

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            if name == "cs_device_alloc":
                return 4096 + 1024 * len(self.calls)
            if name in ("cs_match_ratio", "cs_match_ratio_host"):
                return self.pairs
            return 0
        return f


def test_knn_wrapper_maps_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    s1, s2 = np.zeros(7, cs.SIFT_DTYPE), np.zeros(5, cs.SIFT_DTYPE)
    idx, score, ms = cs.match_knn2(s1, s2, mode=2)
    (name, a), = [c for c in fake.calls if c[0] == "cs_match_knn2"]
    allocs = [c[1][0] for c in fake.calls if c[0] == "cs_device_alloc"]
    assert allocs == [7 * REC, 5 * REC, 7 * 8, 7 * 8]
    assert a[1] == 7 and a[3] == 5 and a[6] == 2 and len({a[0], a[2], a[4], a[5]}) == 4
    assert idx.shape == (7, 2) and idx.dtype == np.int32 and score.shape == (7, 2) and score.dtype == np.float32
    fake.calls.clear()
    idx, score, ms = cs.match_knn2(s1[:0], s2)
    assert not [c for c in fake.calls if c[0] == "cs_match_knn2"] and idx.shape == (0, 2)


def test_ratio_wrappers_map_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    d1, d2 = cs.SiftData(), cs.SiftData()
    d1._buf, d2._buf = cs.DeviceBuffer(64), cs.DeviceBuffer(64)
    d1.numPts, d2.numPts = 7, 5
    pairs, ms = cs.MatchSiftDataRatio(d1, d2, maxRatio=0.6, maxDistance=0.5, crossCheck=False, mode=1)
    (name, a), = [c for c in fake.calls if c[0] == "cs_match_ratio"]
    assert a[0] == d1.d_data and a[1] == 7 and a[2] == d2.d_data and a[3] == 5
    assert a[4] == pytest.approx(0.6) and a[5] == pytest.approx(0.5) and a[6] == 0
    assert a[8] == 7 and a[9] == 1                      # one pair per row of set 1 at most
    assert pairs.shape == (3, 2) and pairs.dtype == np.int32
    fake.calls.clear()
    cs.MatchSiftDataRatio(d1, d2)                       # COLMAP's defaults, cross-checked, auto mode
    (name, a), = [c for c in fake.calls if c[0] == "cs_match_ratio"]
    assert a[4] == pytest.approx(0.8) and a[5] == pytest.approx(0.7) and a[6] == 1 and a[8] == 5 and a[9] == 0
    d1._buf = d2._buf = None
    fake.calls.clear()
    fake.pairs = 2
    pairs, ms = cs.match_ratio_host(np.zeros(9, cs.SIFT_DTYPE), np.zeros(4, cs.SIFT_DTYPE), 0.9, 0.4, False, 2)
    (name, a), = fake.calls
    assert name == "cs_match_ratio_host" and a[1] == 9 and a[3] == 4
    assert a[4] == pytest.approx(0.9) and a[5] == pytest.approx(0.4) and a[6] == 0 and a[8] == 9 and a[9] == 2
    assert pairs.shape == (2, 2)
    fake.calls.clear()
    cs.match_ratio_host(np.zeros(9, cs.SIFT_DTYPE), np.zeros(4, cs.SIFT_DTYPE))
    (name, a), = fake.calls
    assert a[6] == 1 and a[8] == 4 and a[9] == 0


def test_python_wrapper_raises_on_rejection():
    with pytest.raises(cs.CudaSiftError, match="invalid argument"):
        cs.match_ratio_host(np.zeros(3, cs.SIFT_DTYPE), np.zeros(3, cs.SIFT_DTYPE), mode=5)
    with pytest.raises(cs.CudaSiftError, match="invalid argument"):
        cs.match_ratio_host(np.zeros(3, cs.SIFT_DTYPE), np.zeros(3, cs.SIFT_DTYPE), maxRatio=float("nan"))


def numpy_knn2(a, b):
    """Brute force on the numpy chain: the first two candidates in (score descending, index ascending), scores > 0."""
    ex = exact_scores(a, b)
    n1 = len(a)
    idx, score = np.full((n1, 2), -1, np.int32), np.zeros((n1, 2), np.float32)
    for r in range(n1):
        pos = np.nonzero(ex[r] > 0)[0]
        order = pos[np.lexsort((pos, -ex[r, pos]))][:2]
        idx[r, :len(order)] = order
        score[r, :len(order)] = ex[r, order]
    return idx, score


def test_oracle_equals_numpy_chain():
    cases = [(synth_descriptors(40, 1), synth_descriptors(75, 2)), (synth_descriptors(33, 3), synth_descriptors(1, 4)),
             (synth_descriptors(50, 5, sift_like=True), synth_descriptors(97, 6, sift_like=True))]
    s1, s2 = synth_descriptors(20, 7), synth_descriptors(64, 8)
    s2["data"][9] = s2["data"][3]                       # a tied best: the lower index first, equal scores
    s1["data"][0] = s2["data"][3]
    s1["data"][1] = 0                                   # no positive score
    cases.append((s1, s2))
    for a, b in cases:
        gi, gs = knn_oracle.match_knn2(a, b, threads=3)
        wi, ws = numpy_knn2(a["data"], b["data"])
        assert np.array_equal(gi, wi) and gs.tobytes() == ws.tobytes()
    gi, gs = knn_oracle.match_knn2(s1, s2)
    assert tuple(gi[0]) == (3, 9) and gs[0, 0] == gs[0, 1]
    assert tuple(gi[1]) == (-1, -1) and tuple(gs[1]) == (0.0, 0.0)


def emulate_knn(s1, s2):
    """The tensor path's rule for every row: the per-(row, partition) top-3 of the 4-candidate group maxima of the
    split-FP16 scores, T = second largest of {G[0..7], S[0..7]}, the row decidable if 2 delta < T, each partition
    certified if Th <= 0 or Th < T - delta, and the exact top two of the groups I1 (G >= T - delta) and I2
    (S >= T - delta).  Returns (idx, score, undecided rows, exact chains)."""
    a, b = s1["data"], s2["data"]
    n1, n2 = len(a), len(b)
    ng = -(-n2 // 4)
    bp = np.zeros((4 * ng, 128), np.float32)
    bp[:n2] = b
    ex = exact_scores(a, b)
    ah, al = split(a)
    bh, bl = split(bp)
    approx = ((ah @ bh.T) + (ah @ bl.T) + (al @ bh.T)) / (SCALE * SCALE)
    na = np.sqrt((a.astype(np.float64) ** 2).sum(1)) * 1.0001
    bmax = (np.sqrt((b.astype(np.float64) ** 2).sum(1)) * 1.0001).max()
    gm = approx.reshape(n1, ng, 4).max(-1)                       # group g lies in partition g % 8
    idx, score = np.full((n1, 2), -1, np.int32), np.zeros((n1, 2), np.float32)
    undecided = np.zeros(n1, bool)
    chains = 0
    for r in range(n1):
        delta = 2.0 * (T3_C1 * na[r] * bmax + T3_C2 * (na[r] + bmax))
        G, S, Th, I1, I2 = np.zeros(8), np.zeros(8), np.zeros(8), [-1] * 8, [-1] * 8
        for p in range(8):
            ids = np.arange(p, ng, 8)
            v = gm[r, ids]
            order = np.argsort(-v, kind="stable")[:3]
            top = [(v[o], ids[o]) for o in order if v[o] > 0.0]
            if len(top) > 0: G[p], I1[p] = top[0]
            if len(top) > 1: S[p], I2[p] = top[1]
            if len(top) > 2: Th[p] = top[2][0]
        T = sorted(list(G) + list(S))[-2]
        low = T - delta
        if not (T > 2.0 * delta) or not all(Th[p] <= 0.0 or Th[p] < low for p in range(8)):
            undecided[r] = True
            continue
        groups = [I1[p] for p in range(8) if I1[p] >= 0 and G[p] >= low] + \
                 [I2[p] for p in range(8) if I2[p] >= 0 and S[p] >= low]
        cand = np.array([4 * g + c for g in groups for c in range(4)])
        chains += len(cand)
        cand = cand[cand < n2]
        cand = cand[ex[r, cand] > 0]
        order = cand[np.lexsort((cand, -ex[r, cand]))][:2]
        idx[r, :len(order)] = order
        score[r, :len(order)] = ex[r, order]
    return idx, score, undecided, chains


def _check(s1, s2):
    gi, gs, und, chains = emulate_knn(s1, s2)
    wi, ws = knn_oracle.match_knn2(s1, s2, threads=4)
    ok = ~und
    assert np.array_equal(gi[ok], wi[ok]) and gs[ok].tobytes() == ws[ok].tobytes()
    return und, chains


@pytest.mark.parametrize("n2,sift_like", [(1000, False), (1003, True), (1984, False)])
def test_certification_random_sets(n2, sift_like):
    """Every row is decided with a handful of exact chains, including a tail of n2 % 4 != 0 candidates."""
    s1, s2 = synth_descriptors(256, 1, sift_like=sift_like), synth_descriptors(n2, 2, sift_like=sift_like)
    und, chains = _check(s1, s2)
    assert not und.any()
    assert chains < 16 * len(s1)


def test_certification_flags_what_it_cannot_decide():
    s1, s2 = synth_descriptors(128, 21), synth_descriptors(640, 22)
    s2["data"][32] = s2["data"][0]; s2["data"][64] = s2["data"][0]     # three equal group maxima in partition 0
    s1["data"][:16] = s2["data"][0] * 0.999 + s1["data"][:16] * 0.001
    s1["data"][20] *= -1                                               # no positive score at all
    s1["data"][21] = s2["data"][40]; s2["data"][7] = s2["data"][40]; s2["data"][33] = s2["data"][40]   # partitions 2, 1, 0
    und, _ = _check(s1, s2)
    assert und[:16].all() and und[20]
    assert not und[21]                                                 # duplicates in different partitions are decidable
    gi, gs = knn_oracle.match_knn2(s1[21:22], s2)
    assert tuple(gi[0]) == (7, 33) and gs[0, 0] == gs[0, 1]
