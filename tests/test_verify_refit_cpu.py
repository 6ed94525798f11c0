"""The preconditions of the cases of tests/test_verify_refit_gpu.py, checked in float64 without a GPU: the pair counts
the cases claim, no pair on the threshold of the planted model or of the refit over the planted inliers, the spectrum
classification, the exact-data cases (every pair an inlier of both fits), the tiny-threshold cases (each slot's
inliers are its own sample and nothing else comes near) and the keep-rule branch of the cases the GPU file also
restates whole."""
import numpy as np
import pytest

import essential_oracle as eo
import verify_oracle as vo
import test_verify_refit_gpu as rg

NAMES = rg.NAMES


def _planted_refit(c):
    ok, p = rg.valid(c)
    good = c.good[ok]
    c1, c2, s = vo.normalisation(p)
    return p, good, rg.refit(c, p, good, c1, c2, s), (c1, c2, s)


def test_case_list_covers_the_kernel_shapes():
    for kind in "FHE":
        for n in rg.SIZES + ((4, 5, 6) if kind == "H" else (5, 6) if kind == "E" else ()):
            c = rg.case(f"{kind}-n{n}")
            ok, _ = rg.valid(c)
            assert ok.sum() == n and len(c.pairs) == n + max(1, round(0.1 * n)), (kind, n)
            bad = c.pairs[~ok]                         # both kinds: indices out of range, non-finite coordinates
            inside = (bad >= 0).all(1) & (bad[:, 0] < len(c.x1)) & (bad[:, 1] < len(c.x2))
            assert len(bad) < 6 or (inside.any() and (~inside).any())
            assert n < 10 or np.nonzero(~ok)[0].min() < n            # interleaved, not appended
    assert {rg.case(n).kind for n in NAMES} == set(rg.KINDS.values())


@pytest.mark.parametrize("name", [n for n in NAMES if "tiny" not in rg.tags(n)])
def test_no_pair_on_the_threshold(name):
    """Of the planted model, and of the refit over the planted inliers where the spectrum is not clustered."""
    c = rg.case(name)
    p, good, R, (c1, c2, s) = _planted_refit(c)
    if c.truth.any():                                  # pure rotation has no E
        assert rg.band(c, rg.residuals(c, c.truth, p)) == 0
    if R is not None and rg.spectrum(c, p, good, c1, c2, s) >= rg.CLUSTERED:
        assert rg.band(c, rg.residuals(c, R, p)) == 0


@pytest.mark.parametrize("name", NAMES)
def test_spectrum_classified_as_claimed(name):
    """Clustered exactly where the case says so, the others at least 1.5 times above the cut."""
    c = rg.case(name)
    p, good, R, (c1, c2, s) = _planted_refit(c)
    if good.sum() < rg.MIN_REFIT[c.kind] or "tiny" in c.tags:
        return
    sp = rg.spectrum(c, p, good, c1, c2, s)
    if "clustered" in c.tags:
        assert sp < rg.CLUSTERED, sp
    else:
        assert sp >= 1.5 * rg.CLUSTERED, sp


@pytest.mark.parametrize("name", [n for n in NAMES if "exact" in rg.tags(n)])
def test_exact_cases_fit_every_pair(name):
    c = rg.case(name)
    p, good, R, _ = _planted_refit(c)
    assert good.all() and len(p) == len(c.pairs)
    assert rg.residuals(c, c.truth, p).max() < 0.01 * c.thresh
    assert R is not None and rg.residuals(c, R, p).max() < 0.01 * c.thresh


@pytest.mark.parametrize("kind", ["F", "H", "E"])
def test_tiny_threshold_leaves_each_slot_its_sample(kind):
    """Every live slot of the restatement fits its own sample within a tenth of the threshold, and no other pair lies
    within ten times the threshold of it."""
    c = rg.case(f"{kind}-tiny")
    ok, p = rg.valid(c)
    if c.kind == rg.ESSENTIAL:
        M, smp, _ = eo.slot_models(p, c.K1, c.K2, c.loops, c.seed)
    else:
        M, smp, _ = vo.slot_models(p, c.kind, c.loops, c.seed)
    per = rg.PER_SAMPLE[c.kind]
    live = np.nonzero(~np.isnan(M[:, 0]))[0]
    assert len(live) > 0
    for k in live:
        r = rg.residuals(c, M[k].reshape(3, 3), p)
        own = np.zeros(len(p), bool)
        own[smp[k // per]] = True
        assert (r[own] < 0.1 * c.thresh).all() and (r[~own] >= 10 * c.thresh).all(), k


@pytest.mark.parametrize("name", [n for n in NAMES if "whole" in rg.tags(n)])
def test_restated_keep_rule_branch(name):
    """The whole call restated: the refit of an exact case ties and is kept, that of a drop case loses inliers, and no
    pair lies on the threshold of either fit."""
    c = rg.case(name)
    ok, p = rg.valid(c)
    if c.kind == rg.ESSENTIAL:
        M, smp, (c1, c2, s) = eo.slot_models(p, c.K1, c.K2, c.loops, c.seed)
    else:
        M, smp, (c1, c2, s) = vo.slot_models(p, c.kind, c.loops, c.seed)
    counts = np.array([(rg.residuals(c, m.reshape(3, 3), p) < c.thresh).sum() if np.isfinite(m).all() else -1
                       for m in M])
    r0 = rg.residuals(c, M[int(np.argmax(counts))].reshape(3, 3), p)
    inl0 = r0 < c.thresh
    rR = rg.residuals(c, rg.refit(c, p, inl0, c1, c2, s), p)
    assert rg.band(c, r0) == 0 and rg.band(c, rR) == 0
    cnt0, cntR = int(inl0.sum()), int((rR < c.thresh).sum())
    if "exact" in c.tags:
        assert cnt0 == cntR == len(p)
    if "drop" in c.tags:
        assert cntR < cnt0
