"""CPU checks of the tensor matcher's certification argument (csrc/match_tc.cu) over the case families of
tests/tc_cases.py, through the restatement of tests/tc_model.py: the split error stays inside eps with room for the
tensor cores' accumulation, every certified row re-scores a candidate set whose exact rule output is the oracle's under
every admissible perturbation of the accumulators, and every planted near-tie inside delta is re-scored or left to the
exact fallback."""
import functools

import numpy as np
import pytest

import knn_oracle
import oracle
import tc_cases as tc
import tc_model as tm

F32, F64 = np.float32, np.float64
CPU_SHAPES = [(1, 32), (127, 255), (129, 896)]
H100_SMS = 132


@functools.lru_cache(maxsize=None)
def _exact(family, n1, n2):
    s1, s2, _ = tc.make(family, n1, n2)
    return tm.exact_scores(s1["data"], s2["data"])


def test_fma32_is_one_rounding():
    """fma32 against the C fmaf of the oracles: every row's best chain score is the oracle's."""
    s1, s2, _ = tc.make("halfway", 127, 255)
    ex = _exact("halfway", 127, 255)
    idx, score = knn_oracle.match_knn2(s1, s2)
    best = np.where(ex > 0, ex, 0).max(1)
    assert best.tobytes() == score[:, 0].tobytes()
    rng = np.random.default_rng(5)
    a, b, c = (rng.standard_normal(100000).astype(F32) * 10.0 ** rng.uniform(-15, 15, 100000).astype(F32) for _ in range(3))
    got = tm.fma32(a, b, c)
    want = np.array([F32(float(np.longdouble(x) * np.longdouble(y) + np.longdouble(z))) for x, y, z in zip(a[:2000], b[:2000], c[:2000])])
    # long double has 64 bits: the product is exact and the sum is rounded once before the float32 rounding; where
    # that double rounding could matter the two agree with fma32 except at exact ties, which fma32 resolves
    assert (got[:2000] == want).mean() > 0.999


@pytest.mark.parametrize("family", tc.FAMILIES)
def test_families_plant_what_they_name(family):
    """make() asserts each family's property; here: no family is empty and the planted families carry every gap,
    placement and reversal over the GPU test's shapes."""
    gaps, places = set(), set()
    for n1, n2, _ in tc.shapes(H100_SMS):
        s1, s2, plan = tc.make(family, n1, n2)
        assert len(s1) == n1 and len(s2) == n2
        for p in tc.plan_of((s1, s2, plan)):
            gaps.add(p["gap"]); places.add(p["placement"])
    if family in tc.PLANTED_FAMILIES:
        assert gaps == set(tc.GAPS) | {"reversal"}, gaps
        assert places == set(tc.PLACEMENTS), places


@pytest.mark.parametrize("sms", [H100_SMS, 114, 78])
def test_shapes_cover_the_schedule_seams(sms):
    """n1 in {1, 127, 128, 129, 257}; row tiles of 1, 2, 6, 7 and many segments (the resolve unrolls T3_SEG = 6 and
    loops over the rest); n2 % 32 in {0, 1, 31} and n2 % 128 in {0, 32, 127}; a CTA boundary on a row tile's end and
    one inside a row tile with U > 1; mutual shapes with the B-role copy in neither, one and both sets."""
    sh = tc.shapes(sms)
    assert {n1 for n1, _, _ in sh} == {1, 127, 128, 129, 257}
    assert {n2 % 32 for _, n2, _ in sh} == {0, 1, 31} and {0, 32, 127} <= {n2 % 128 for _, n2, _ in sh}
    for rule in ("ref", "knn"):
        facts = [tc.shape_facts(n1, n2, sms)[rule] for n1, n2, _ in sh]
        segs = {f["maxseg"] for f in facts}
        assert {1, 2, 6, 7} <= segs and max(segs) > 2 * tm.T3_SEG, segs
        assert any(f["coincide"] for f in facts) and any(f["straddle"] for f in facts)
    copies = [sum(tm.b_role_copy(n, (n // 32) * 32) for n in (n1, n2)) for n1, n2 in tc.MUTUAL_SHAPES]
    assert set(copies) == {0, 1, 2}


@pytest.mark.parametrize("family", [f for f in tc.FAMILIES if f != "gated"])
def test_split_error_within_eps(family):
    """(a) |split-FP16 value - FP32 chain| + the accumulation budget <= eps = T3_C1 |a||b| + T3_C2 (|a| + |b|) for every
    pair (|b| <= bmax, so the bmax form the kernel uses holds too).  In the tiny-norm families it is T3_C2 that carries
    the bound: there the error exceeds what T3_C1 alone allows."""
    worst, c2_needed = 0.0, 0
    for n1, n2 in CPU_SHAPES:
        s1, s2, _ = tc.make(family, n1, n2)
        a, b = s1["data"], s2["data"]
        ex = _exact(family, n1, n2).astype(F64)
        ap = tm.approx_scaled(a, b) / 2.0 ** 24
        na = np.sqrt((a.astype(F64) ** 2).sum(1))[:, None]
        nb = np.sqrt((b.astype(F64) ** 2).sum(1))[None, :]
        err = np.abs(ap - ex) + tm.ACCUM_BUDGET * na * nb
        room = tm.eps64(na, nb)
        assert (err <= room).all(), (family, float((err / room).max()))
        worst = max(worst, float((err / room).max()))
        c2_needed += int((err > float(tm.T3_C1) * na * nb).sum())
    if family in ("subnormal16", "norms", "planted_tiny"):
        assert c2_needed > 0, "T3_C2 carries the bound for the tiny-norm rows"
    print("%s: worst (error + budget) / eps = %.3g, pairs that need T3_C2: %d" % (family, worst, c2_needed))


def _certified_equal_oracle(family, n1, n2, knn):
    s1, s2, plan = tc.make(family, n1, n2)
    ex = _exact(family, n1, n2)
    d = tm.Direction(s1["data"], s2["data"], knn)
    if knn:
        wi, ws = knn_oracle.match_knn2(s1, s2)
    else:
        want = oracle.match(s1, s2, threads=8)
    certified = 0
    for name, pert in d.perturbations(ex, seed=n1 + n2).items():
        ok, cands = d.run(pert)
        for r in np.nonzero(ok)[0]:
            if knn:
                (j1, j2), (v1, v2) = tm.rule_knn(cands[r], ex[r], d.n2)
                assert (j1, j2) == tuple(wi[r]) and F32(v1) == ws[r, 0] and F32(v2) == ws[r, 1], (name, r)
            else:
                sc, m, amb = tm.rule_ref(cands[r], ex[r], d.n2)
                assert (sc, m, amb) == (want["score"][r], want["match"][r], want["ambiguity"][r]), (name, r)
        certified += int(ok.sum())
        # (c) every planted row inside delta: uncertified, or both of its two best contenders re-scored -- except, in the
        # reference rule, a second best that shares a partition other than 0 with the best: only partition 0 supplies a
        # second best to the output (quirk Q9), so that one may be dropped once its approximate score is delta below
        for p in tc.plan_of((s1, s2, plan)):
            r = p["row"]
            if not ok[r]:
                continue
            sc = {q: F64(ex[r, q]) for q in p["pos"]}
            order = sorted(p["pos"], key=lambda q: (-sc[q], q))
            need = {q for q in order if sc[q] == sc[order[0]]}
            rest = [q for q in order if sc[q] < sc[order[0]]]
            if rest and sc[order[0]] - sc[rest[0]] < F64(d.delta[r]):
                part = (rest[0] >> 2) & 7
                if knn or part == 0 or part != (order[0] >> 2) & 7:
                    need.add(rest[0])
            assert need <= set(cands[r]), (name, p)
    lo, hi = d.fallback_bounds()
    assert 0 <= lo <= hi <= n1
    return certified, lo, hi


@pytest.mark.parametrize("knn", [False, True], ids=["ref", "knn"])
@pytest.mark.parametrize("family", [f for f in tc.FAMILIES if f != "gated"])
def test_certified_rows_equal_oracle(family, knn):
    """(b) and (c) on every CPU shape under every perturbation of Direction.perturbations."""
    for n1, n2 in CPU_SHAPES:
        certified, lo, hi = _certified_equal_oracle(family, n1, n2, knn)
        if family in ("ordinary", "planted", "halfway", "cancel"):
            assert certified > 0
        if family == "ordinary" and n1 > 100:
            assert hi <= 0.01 * n1


def test_planted_rows_inside_delta_are_present():
    """The planted cases really put rows inside delta, and some of them have contenders in different groups."""
    inside = 0
    for family in tc.PLANTED_FAMILIES:
        s1, s2, plan = tc.make(family, 129, 896)
        d = tm.Direction(s1["data"], s2["data"], False)
        ex = _exact(family, 129, 896)
        for p in tc.plan_of((s1, s2, plan)):
            sc = np.sort(ex[p["row"], list(p["pos"])].astype(F64))
            inside += int(sc[-1] - sc[-2] < F64(d.delta[p["row"]]) and p["placement"] != "group")
    assert inside >= 4


def test_rowok_term_decides_tiny_rows():
    """Rows whose every approximate score is zero (components below 2^-37 vanish in the split) have positive exact
    scores: without the m2 > 2 delta term of rowOk they would be certified with no candidate and report no match."""
    rng = np.random.default_rng(3)
    a = (np.abs(rng.standard_normal((4, 128))) * 1e-13).astype(F32)
    b = np.abs(rng.standard_normal((64, 128))).astype(F32)
    d = tm.Direction(a, b, knn=False)
    assert not d.approx.any()
    ok, _ = d.run()
    assert not ok.any()
    assert (tm.exact_scores(a, b) > 0).all()
