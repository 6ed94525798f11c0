"""Case families for the tensor matcher (csrc/match_tc.cu): descriptor sets over the whole input range its gate admits,
planted near-ties, and the GEMM schedule's shapes.  TEST INFRASTRUCTURE ONLY.

Value families (rows of both sets):
  ordinary      synth_descriptors: unit norm, non-negative (the family the rest of the suite uses)
  cancel        signed rows; half of set 2 nearly orthogonal to a row of set 1 (score << |a||b|)
  norms         per-row norms from 1e-20 to 40 in each set, and one row of set 2 near 88 that sets bmax for every row
  subnormal16   components from 2^-46 to 2^-15, where lo, or hi and lo, of the 2^12-scaled split are FP16 subnormal
  edge          components at 7.9999995 (the largest value the gate admits) and FP32 subnormals
  halfway       every component puts lo exactly halfway between two FP16 values (the largest split error)
  gated         the edge family with one component exactly 8.0 in set 2: every row takes the exact way
Planted families (signed rows at scale 1 and at 1e-6, where T3_C2 carries the bound and lo is FP16 subnormal):
  pairs and triples of candidates whose chain scores differ by 0, 1 ulp, 0.5 eps, eps, 2 eps and 3 eps, in one
  4-group, in one partition (j >> 2) & 7 but different groups, and in different partitions; and rows where the chain's
  order of the two best candidates is the reverse of the float64 order.  make() asserts every planted relation.

shapes(sms) derives the schedule shapes from the SM count through t3_plan (tc_model)."""
import functools

import numpy as np

import tc_model as tm
from cudasift_b200.records import SIFT_DTYPE
from cudasift_b200.synth import synth_descriptors

F32, F64 = np.float32, np.float64
VALUE_FAMILIES = ("ordinary", "cancel", "norms", "subnormal16", "edge", "halfway", "gated")
PLANTED_FAMILIES = ("planted", "planted_tiny")
FAMILIES = VALUE_FAMILIES + PLANTED_FAMILIES
GAPS = ("0", "1ulp", "0.5eps", "eps", "2eps", "3eps")
PLACEMENTS = ("group", "partition", "cross")
TOP = np.nextafter(F32(8.0), F32(0.0))          # 7.9999995


def records(desc, seed):
    r = np.zeros(len(desc), SIFT_DTYPE)
    r["data"] = desc
    rng = np.random.default_rng(seed)
    r["xpos"] = rng.uniform(0, 1920, len(desc)).astype(F32)
    r["ypos"] = rng.uniform(0, 1080, len(desc)).astype(F32)
    return r


def _signed_unit(rng, n):
    """Signed directions with every |component| in [0.5, 1] before normalising: no component above 0.18."""
    d = rng.uniform(0.5, 1.0, (n, 128)) * np.where(rng.random((n, 128)) < 0.5, -1.0, 1.0)
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def _halfway(rng, shape):
    """Scaled values hi + lo with lo exactly halfway between two FP16 values; unscaled (exact) and signed."""
    n = int(np.prod(shape))
    e = rng.integers(-14, 15, n)                         # hi's exponent (2^12-scaled)
    hi = (1024 + rng.integers(0, 1024, n)) * np.exp2(e - 10.0)
    normal_lo = e >= -1
    # lo normal: lo in [2^(e-12), 2^(e-11)), an odd multiple of its half ulp 2^(e-23); lo subnormal: (j + 0.5) 2^-24
    lo = np.where(normal_lo, (2048 + 2 * rng.integers(0, 1024, n) + 1) * np.exp2(e - 23.0),
                  (rng.integers(0, np.maximum(np.exp2(e + 13.0).astype(np.int64), 1)) + 0.5) * 2.0 ** -24)
    x = (hi + lo) / tm.SCALE * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    return x.reshape(shape)


def _value_sets(family, n1, n2, rng):
    if family == "ordinary":
        return synth_descriptors(n1, int(rng.integers(1 << 30)))["data"], synth_descriptors(n2, int(rng.integers(1 << 30)))["data"]
    if family == "cancel":
        a = _signed_unit(rng, n1)
        b = _signed_unit(rng, n2)
        for j in range(0, n2, 2):                        # nearly orthogonal to row j % n1 of set 1
            u = a[j % n1]
            v = b[j] - (b[j] @ u) * u
            v /= np.linalg.norm(v)
            b[j] = v + rng.choice([-1, 1]) * 10.0 ** rng.uniform(-6, -2) * u
        return a, b
    if family == "norms":
        a = _signed_unit(rng, n1) * 10.0 ** rng.uniform(-20, np.log10(40), (n1, 1))
        b = _signed_unit(rng, n2) * 10.0 ** rng.uniform(-20, np.log10(40), (n2, 1))
        a[0] *= 1e-20 / np.linalg.norm(a[0])
        big = (n2 // 32) * 32 - 1 if n2 >= 32 else n2 - 1
        b[big] = np.minimum(rng.uniform(7.5, 8.0, 128), TOP) * np.where(rng.random(128) < 0.5, -1, 1)
        return a, b
    if family == "subnormal16":
        def rows(n):
            top = rng.uniform(-36, -15, (n, 1))           # per row: whole rows where hi is subnormal or zero
            x = np.exp2(top - rng.uniform(0, 10, (n, 128))) * np.where(rng.random((n, 128)) < 0.5, -1, 1)
            mixed = rng.random(n) < 0.3
            x[mixed, ::2] = _signed_unit(rng, int(mixed.sum()))[:, ::2]
            return x
        return rows(n1), rows(n2)
    if family in ("edge", "gated"):
        def rows(n):
            x = _signed_unit(rng, n)
            m = rng.random((n, 128))
            x[m < 0.02] = TOP * np.sign(x[m < 0.02])
            x[(m >= 0.02) & (m < 0.06)] = rng.choice([1e-40, -1e-40, 1.4e-45, -2e-39], int(((m >= 0.02) & (m < 0.06)).sum()))
            return x
        a, b = rows(n1), rows(n2)
        if family == "gated":
            b[n2 // 2, 5] = 8.0
        return a, b
    if family == "halfway":
        return _halfway(rng, (n1, 128)), _halfway(rng, (n2, 128))
    raise ValueError(family)


# ---------------------------------------------------------------------------------------------------- planting
def _positions(placement, j, arity):
    step = {"group": 1, "partition": 32, "cross": 4}[placement]
    return [j + step * k for k in range(arity)]


def _hit(a, b0, target, rng, exact_ulp):
    """A copy of b0 with one component moved so that the chain score is target (exact_ulp) or within 1 % of it."""
    order = np.argsort(-np.abs(a))
    s0 = F64(tm.chain_pairs(a[None], b0[None])[0])
    for k in order[:8]:
        if exact_ulp:
            steps = np.arange(1, 4097)
            cand = np.repeat(b0[None], len(steps), 0)
            v = b0[k]
            direction = F32(-np.inf) if (a[k] > 0) == (target < s0) else F32(np.inf)
            vals = [v]
            for _ in steps:
                vals.append(np.nextafter(vals[-1], direction))
            cand[:, k] = np.array(vals[1:], F32)
            sc = tm.chain_pairs(np.repeat(a[None], len(steps), 0), cand)
            w = np.nonzero(sc == F32(target))[0]
            if len(w):
                return cand[w[0]]
        else:
            c = b0.copy()
            c[k] = F32(F64(b0[k]) + (target - s0) / F64(a[k]))
            got = F64(tm.chain_pairs(a[None], c[None])[0])
            if abs(got - target) <= 0.01 * abs(target - s0) and np.all(np.abs(c) < 8):
                return c
    raise AssertionError("no component reaches the planted score")


def _reversal(a, b0, rng):
    """A near copy of b0 whose chain score and float64 score order against b0's are opposite (seeded search): random
    moves of b0 that change the true score by about a third of an ulp of the score."""
    a64 = a.astype(F64)
    c0 = tm.chain_pairs(a[None], b0[None])[0]
    t0 = b0.astype(F64) @ a64
    step = 0.3 * F64(np.spacing(c0)) / np.linalg.norm(a64)
    for _ in range(16):
        cand = (b0[None].astype(F64) + rng.normal(0.0, step, (2048, 128))).astype(F32)
        ch = tm.chain_pairs(np.repeat(a[None], 2048, 0), cand)
        t = cand.astype(F64) @ a64
        w = np.nonzero(((ch > c0) & (t < t0)) | ((ch < c0) & (t > t0)))[0]
        if len(w):
            return cand[w[0]]
    raise AssertionError("no reversal found")


def _plant(a, b, n2cand, rng, scale):
    """Plants contenders into b (in place) for rows of a; returns the plan: one dict per planted row."""
    n1 = len(a)
    blk = 96 if n2cand >= 96 else 12
    nrows = min(n1, n2cand // blk, 32)
    combos = [(g, p, k) for g in GAPS for p in PLACEMENTS for k in (2, 3)]
    rng.shuffle(combos)
    plan = []
    for q in range(nrows):
        r = int(rng.integers(n1)) if n1 > nrows else q
        while any(p["row"] == r for p in plan):
            r = (r + 1) % n1
        j = q * blk + 4 * int(rng.integers(0, 2 if blk == 12 else 8))
        reversal = q % 8 == 7
        if reversal:
            gap, placement, arity = "reversal", "cross", 2
        else:
            for gap, placement, arity in combos[q % len(combos):] + combos:
                if _positions(placement, j, arity)[-1] < min(j + blk, n2cand):
                    break
        pos = _positions(placement, j, arity)
        u = a[r].astype(F64) / np.linalg.norm(a[r])
        base = (u + 0.05 * _signed_unit(rng, 1)[0])
        b0 = (base / np.linalg.norm(base) * scale).astype(F32)
        s0 = F64(tm.chain_pairs(a[r][None], b0[None])[0])
        ncheck = np.sqrt((a[r].astype(F64) ** 2).sum())
        eps = tm.eps64(ncheck, scale * 1.05)
        vecs = [b0]
        for k in range(1, arity):
            if gap == "0":
                vecs.append(b0.copy())
            elif gap == "1ulp":
                t = F64(s0)
                for _ in range(k):
                    t = F64(np.nextafter(F32(t), F32(-np.inf)))
                vecs.append(_hit(a[r], b0, t, rng, True))
            elif gap == "reversal":
                vecs.append(_reversal(a[r], b0, rng))
            else:
                m = {"0.5eps": 0.5, "eps": 1.0, "2eps": 2.0, "3eps": 3.0}[gap]
                vecs.append(_hit(a[r], b0, s0 - k * m * eps, rng, False))
        perm = rng.permutation(arity)
        for i, p in enumerate(pos):
            b[p] = vecs[perm[i]]
        sc = tm.chain_pairs(np.repeat(a[r][None], arity, 0), b[pos])
        order = [pos[i] for i in np.argsort(-sc.astype(F64), kind="stable")]
        plan.append(dict(row=r, pos=pos, gap=gap, placement=placement, order=order))
    return plan


@functools.lru_cache(maxsize=None)
def make(family, n1, n2, seed=0):
    """(set 1 records, set 2 records, plan): plan lists the planted rows of the planted families (their contenders'
    positions, best first by the chain, the gap kind and the placement)."""
    rng = np.random.default_rng([seed, n1, n2, FAMILIES.index(family)])
    plan = []
    if family in PLANTED_FAMILIES:
        scale = 1.0 if family == "planted" else 1e-6
        a = (_signed_unit(rng, n1) * scale).astype(F32)
        b = (_signed_unit(rng, n2) * scale).astype(F32)
        n2v = (n2 // 32) * 32
        big = n2v - 1 if n2v else n2 - 1                 # the last candidate sets bmax; contenders lie below it
        b[big] = (_signed_unit(rng, 1)[0] * scale * 1.05).astype(F32)
        if big >= 12:
            plan = _plant(a, b, big, rng, scale)
    else:
        a, b = _value_sets(family, n1, n2, rng)
    s1, s2 = records(np.asarray(a, F32), seed * 2 + 1), records(np.asarray(b, F32), seed * 2 + 2)
    check(family, s1, s2, plan)
    return s1, s2, tuple(map(lambda p: tuple(sorted((k, tuple(v) if isinstance(v, list) else v) for k, v in p.items())),
                             plan))


def plan_of(case):
    return [dict(p) for p in case[2]]


# ---------------------------------------------------------------------------------------------------- self-checks
def check(family, s1, s2, plan):
    """Asserts that a case has what its family names."""
    a, b = s1["data"], s2["data"]
    assert len(a) and len(b)
    both = np.concatenate([a, b])
    if family == "gated":
        assert tm.gated(b) and not tm.gated(a)
        return
    assert not tm.gated(both), family
    if family == "cancel":
        na, nb = np.linalg.norm(a.astype(F64), axis=1), np.linalg.norm(b.astype(F64), axis=1)
        j = np.arange(0, len(b), 2)
        cos = np.abs((a[j % len(a)].astype(F64) * b[j].astype(F64)).sum(1)) / (na[j % len(a)] * nb[j])
        assert np.median(cos) < 1e-2 and (np.sign(both) < 0).mean() > 0.4
    elif family == "norms":
        n = np.sqrt((both.astype(F64) ** 2).sum(1))
        assert n.min() <= 1.1e-20 and n.max() > 80 and np.abs(both).max() < 8
        nb = np.sqrt((b.astype(F64) ** 2).sum(1))
        assert (nb > 80).sum() == 1
    elif family == "subnormal16":
        hi, lo = tm.split(both)
        x = np.abs(both)
        mid, low = (x >= 2.0 ** -26) & (x < 2.0 ** -15), x < 2.0 ** -26     # lo subnormal / hi subnormal or zero
        lo_sub = (lo != 0) & (np.abs(lo.astype(F64)) < 2.0 ** -14)
        hi_sub = np.abs(hi.astype(F64)) < 2.0 ** -14
        assert lo_sub[mid].mean() > 0.3 and hi_sub[low].mean() > 0.99 and hi_sub[mid].mean() < 0.01
        assert mid.sum() > 100 and low.sum() > 100
    elif family == "edge":
        assert np.abs(both).max() == TOP
        sub = (both != 0) & (np.abs(both) < np.finfo(F32).tiny)
        assert sub.sum() > 0
    elif family == "halfway":
        xs = both.astype(F64) * tm.SCALE
        hi, lo = tm.split(both)
        r = xs - hi.astype(F64)
        ulp = np.where(np.abs(r) < 2.0 ** -14, 2.0 ** -24, np.exp2(np.floor(np.log2(np.abs(r) + 1e-300)) - 10))
        assert np.all(np.abs(r - lo.astype(F64)) == ulp / 2)       # every lo was rounded from a tie
    if family in PLANTED_FAMILIES:
        _check_plan(a, b, plan)


def _check_plan(a, b, plan):
    n2v = (len(b) // 32) * 32
    dn = tm.Direction(a, b, knn=False)
    for p in plan:
        r, pos = p["row"], p["pos"]
        assert pos[-1] < n2v
        sc = tm.chain_pairs(np.repeat(a[r][None], len(pos), 0), b[pos])
        order = [pos[i] for i in np.argsort(-sc.astype(F64), kind="stable")]
        assert p["gap"] == "0" or order == list(p["order"]), "the chain order is the planted one"
        g = F64(sc.max()) - F64(np.sort(sc)[-2])
        eps = tm.eps64(np.sqrt((a[r].astype(F64) ** 2).sum()), F64(dn.bmax) / 1.0001)
        if p["gap"] == "0":
            assert g == 0
        elif p["gap"] == "1ulp":
            assert F32(np.sort(sc)[-2]) == np.nextafter(sc.max(), F32(-np.inf))
        elif p["gap"] == "reversal":
            t = b[pos].astype(F64) @ a[r].astype(F64)
            assert (np.argmax(t) != np.argmax(sc)) and t[0] != t[1] and sc[0] != sc[1]
        else:
            m = {"0.5eps": 0.5, "eps": 1.0, "2eps": 2.0, "3eps": 3.0}[p["gap"]]
            assert 0.95 * m * eps <= g <= 1.05 * m * eps, (p, g / eps)
        # placement
        grp = [q >> 2 for q in pos]
        part = [(q >> 2) & 7 for q in pos]
        if p["placement"] == "group":
            assert len(set(grp)) == 1
        elif p["placement"] == "partition":
            assert len(set(part)) == 1 and len(set(grp)) == len(pos)
        else:
            assert len(set(part)) == len(pos)
        # the contenders are the row's top candidates by far
        others = np.delete(np.arange(n2v), pos)
        rest = (b[others].astype(F64) @ a[r].astype(F64)).max() if len(others) else -np.inf
        assert rest < 0.5 * F64(sc.min()), "the planted contenders lead the row"


# ---------------------------------------------------------------------------------------------------- shapes
def shapes(sms):
    """One-way shapes (n1, n2, what) from the SM count.  n2 = 128 (tiles - 1) + r with r in {32, 33, 127, 128}: n2 % 32
    in {0, 1, 31}, n2 % 128 in {0, 32, 127}, and the same tile count for both rules (n2v = 32 floor(n2 / 32))."""
    ne = 2 * tm.idivup(sms // 3 + 1, 2)                  # three row tiles of ne units: more units than SMs, U = 2
    no = ne + 1
    spec = [(1, 1, 32), (127, 2, 127), (128, 2, 32), (128, 6, 33), (1, 7, 127), (129, 7, 128), (257, 32, 127),
            (257, ne, 33), (257, no, 128)]
    return [(n1, 128 * (t - 1) + r, "%dx%d" % (n1, 128 * (t - 1) + r)) for n1, t, r in spec]


MUTUAL_SHAPES = [(256, 512), (300, 512), (300, 1000), (1030, 256)]     # B-role copy in neither, one, both, neither


def shape_facts(n1, n2, sms):
    """Per rule the most segments a row tile spans and whether a CTA boundary coincides with / falls inside a row
    tile's end (U > 1)."""
    out = {}
    for rule, n2c in (("ref", (n2 // 32) * 32), ("knn", n2)):
        if n2c == 0:
            continue
        segs = segments(n1, n2c, sms)
        U = tm.t3_plan(n1, n2c, sms)[3]
        out[rule] = dict(maxseg=max(c1 - c0 + 1 for c0, c1, _ in segs), U=U,
                         coincide=any(e for _, _, e in segs[:-1]) and U > 1,
                         straddle=any(not e for _, _, e in segs[:-1]) and U > 1)
    return out


segments = tm.segments
