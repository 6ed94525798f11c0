"""The detector's restatement (tests/detect_ref.py) validated without a GPU, and the seam coverage of the GPU cases.

- fma32 rounds once, ties included, against exact rational arithmetic.
- The CPU oracle's records (IEEE division, libm exp2f / powf: all inside the MUFU bounds the restatement assumes) are
  exactly the restatement's kept set, every field inside its admissible set.
- The seam shapes the GPU tests use (detect_ref.SEAM_SHAPES) put the last strip and the last item of a level on every seam the detector
  has, for every row-stream height the pipeline picks (cs_detector_items)."""
import ctypes
from fractions import Fraction

import numpy as np
import pytest

import detect_ref as dr
import oracle
import refcases
from cudasift_b200.synth import synth_image
from test_describe_gpu import split_records


def _round_f32(q):
    """Round the rational q to float32, ties to even."""
    f = np.float32(float(q))
    cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
    return min(cands, key=lambda v: (abs(Fraction(float(v)) - q), int(np.float32(v).view(np.uint32)) & 1))


def test_fma32_rounds_once():
    rng = np.random.default_rng(3)
    a = rng.standard_normal(3000).astype(np.float32)
    b = rng.standard_normal(3000).astype(np.float32)
    c = rng.standard_normal(3000).astype(np.float32)
    # exact ties, rounded to even: 1 + 2^-24 -> 1, and 1 + 2^-23 + 2^-24 -> 1 + 2^-22
    one, m = np.float32(1.0), np.float32(1.0 + 2.0 ** -23)
    ta = np.array([one, m, m], np.float32)
    tb = np.array([one, one, one], np.float32)
    tc = np.array([np.float32(2.0 ** -24), np.float32(2.0 ** -24), np.float32(-2.0 ** -24)], np.float32)
    # (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24 is a float32 midpoint; +-2^-70 breaks the tie, but float64 absorbs it
    da = np.array([np.float32(1.0 + 2.0 ** -12)] * 4, np.float32)
    db = np.array([np.float32(1.0 + 2.0 ** -12)] * 4, np.float32)
    dc = np.array([np.float32(2.0 ** -70), np.float32(-2.0 ** -70), np.float32(2.0 ** -80), np.float32(0.0)],
                  np.float32)
    A, B, C = (np.concatenate(v) for v in ((a, ta, da), (b, tb, db), (c, tc, dc)))
    got = dr.fma32(A, B, C)
    for i in range(len(A)):
        q = Fraction(float(A[i])) * Fraction(float(B[i])) + Fraction(float(C[i]))
        assert got[i] == _round_f32(q), (i, A[i], B[i], C[i], got[i])
    # the naive float64 route double-rounds one of the crafted ties; fma32 does not
    naive = (da.astype(np.float64) * db + dc).astype(np.float32)
    exact = np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                      for x, y, z in zip(da, db, dc)], np.float32)
    assert not np.array_equal(naive, exact) and np.array_equal(dr.fma32(da, db, dc), exact)


def test_mufu_sets_hold_the_exact_result_within_bound():
    rng = np.random.default_rng(5)
    x = rng.standard_normal(2000).astype(np.float32)
    y = (rng.standard_normal(2000) * 10 ** rng.uniform(-5, 5, 2000)).astype(np.float32)
    c = dr.fdividef(x, y)
    q = x.astype(np.float64) / y
    assert np.all(np.abs(c.astype(np.float64) - q[:, None]) <= 2 * dr._ulp_of(q)[:, None])
    assert (c == (x / y)[:, None]).any(1).all()                       # the IEEE quotient is admissible
    assert (np.unique(c, axis=1).shape[1] >= 5)
    assert np.all(dr.fdividef(np.float32(1.0), np.float32(0.0)) == np.inf)
    assert np.all(dr.fdividef(np.float32(1.0), np.float32(2.0 ** 127)) == 0.0)
    t = dr.pow_table()
    assert np.all(t[0] == 1.0) and all((t[s] == np.float32(2.0 ** (s / 5))).any() for s in range(5))


def oracle_levels(img, octaves, up=False):
    lv = [oracle.lowpass(oracle.scaleup(img) if up else img, 1.0)]
    for _ in range(1, octaves):
        lv.append(oracle.scaledown(lv[-1]))
    return lv


ORACLE_CASES = [("synth320", lambda: synth_image(320, 240, seed=9), dict(thresh=2.0)),
                ("synth491x195_t1", lambda: synth_image(491, 195, seed=4), dict(thresh=1.0)),
                ("left_crop", lambda: refcases.left_crop(), dict(thresh=4.5)),
                ("synth320_low", lambda: synth_image(320, 240, seed=2), dict(thresh=2.0, lowest=3.0))]


@pytest.mark.parametrize("name,make,kw", ORACLE_CASES, ids=[c[0] for c in ORACLE_CASES])
def test_oracle_records_are_the_restatements_kept_set(name, make, kw):
    img = np.ascontiguousarray(make(), np.float32)
    octaves = 5
    pts, _ = oracle.extract(img, octaves, 1.0, kw["thresh"], kw.get("lowest", 0.0))
    pidx, _ = split_records(pts)
    seen = 0
    stats = dict(records=0, marginal=0)
    for l, lv in enumerate(oracle_levels(img, octaves)):
        ref = dr.Level(lv, octaves, l, kw["thresh"], kw.get("lowest", 0.0) / (1 << l))
        s = np.float32(1 << l)
        p = pts[pidx[pts["subsampling"][pidx] == s]]
        rec = dict(x=p["xpos"] / s, y=p["ypos"] / s, scale=p["scale"] / s, sharpness=p["sharpness"],
                   edgeness=p["edgeness"])
        sc, gy, gx = ref.locate(rec)
        st = ref.check(sc, gy, gx, rec)
        key = (sc.astype(np.int64) << 40) | (gy.astype(np.int64) << 20) | gx
        assert len(np.unique(key)) == len(key), "two records of one extremum"
        seen += len(p)
        stats["records"] += st["records"]
        stats["marginal"] += st["marginal"]
    assert seen == len(pidx) > 100
    print("\n%s: %s" % (name, stats))


# ----------------------------------------------------------------------------------------------------- seam coverage
def _items(w, h, octaves, up, n, hs):
    import cudasift_b200 as cs
    L = cs.lib()
    cap = 1 << 16
    out = np.zeros(4 * cap, np.uint32)
    cnt = L.cs_detector_items(w, h, octaves, int(up), n, hs, out.ctypes.data_as(ctypes.c_void_p), cap)
    assert 0 <= cnt <= cap
    return out[:4 * cnt].reshape(-1, 4)


def _level_sizes(w, h, octaves, up):
    lw, lh = [w * (2 if up else 1)], [h * (2 if up else 1)]
    for _ in range(1, octaves):
        lw.append(lw[-1] // 2)
        lh.append(lh[-1] // 2)
    return lw, lh


@pytest.mark.parametrize("batch", sorted(dr.HS_OF_BATCH))
def test_gpu_cases_cover_every_seam(batch):
    hs = dr.HS_OF_BATCH[batch]
    strips0, stripsc, lastrows, small = set(), set(), set(), set()
    for w, h, octaves in dr.SEAM_SHAPES:
        lw, lh = _level_sizes(w, h, octaves, False)
        it = _items(w, h, octaves, False, 1, hs)
        for l in range(octaves):
            if lw[l] < 1 or lh[l] < 1:
                break
            if min(lw[l], lh[l]) == 3:
                small.add("w" if lw[l] == 3 else "h")
            mine = it[(it[:, 0] & 0xff) == l]
            if len(mine) == 0:
                continue
            last_x0 = int(mine[:, 1].max())
            cols = min(dr.D2_STRIP, lw[l] - 2 - last_x0)
            (strips0 if l == 0 else stripsc).add(cols)
            last = mine[mine[:, 2] == mine[:, 2].max()][0]
            left = lh[l] - 1 - int(last[2])                     # tested rows from the last item's first to h - 2
            # the last item splits what is left between its two streams (no stream marches past the level for nothing)
            assert int(last[3]) == (hs if left >= 2 * hs else (left + 1) // 2), (w, h, l, hs, last, left)
            lastrows.add(left)
    want_cols = {1, 2, 3, 4, 243, 244}
    assert want_cols <= strips0, sorted(want_cols - strips0)
    assert want_cols <= stripsc, sorted(want_cols - stripsc)
    assert {1, 2, 2 * hs - 1, 2 * hs} <= lastrows, sorted({1, 2, 2 * hs - 1, 2 * hs} - lastrows)
    assert small == {"w", "h"}


# ------------------------------------------------------------------------------------------------- oversized levels
@pytest.mark.parametrize("w,h,up", [(8194, 64, 0), (64, 8194, 0), (4097, 64, 1), (64, 4097, 1)])
def test_levels_past_the_tag_limit_are_refused(w, h, up):
    """An extremum's tag packs gx and gy into 13 bits: a level 0 wider or taller than 8193 px would alias two
    positions, and the cap's fix-up deletes records by tag.  Such sizes are refused by name, before any CUDA call."""
    import cudasift_b200 as cs
    L = cs.lib()
    assert not L.cs_extractor_create_batch(w, h, 5, 1024, up, 1)
    assert b"size limit of 8193" in L.cs_last_error()
    r = L.cs_extract(ctypes.c_void_p(16), w, h, w, 5, 1.0, 3.0, 0.0, up, None, ctypes.c_void_p(16), None, 1024)
    assert r == -2 and b"ExtractSift" in L.cs_last_error() and b"size limit of 8193" in L.cs_last_error()
    L.cs_set_tuning(b"no such key", 0)                    # a known last error to tell a new one from
    r = L.cs_extract_host(ctypes.c_void_p(16), w, h, 5, 1.0, 3.0, 0.0, up, None, 1024)
    assert r == -2 and b"size limit of 8193" in L.cs_last_error()


def test_largest_level_within_the_tag_limit_passes_the_size_check():
    """8193 px (4096 px with scaleUp) pass the size check: with no record buffer the next check refuses the call,
    still before any CUDA call."""
    import cudasift_b200 as cs
    L = cs.lib()
    for w, h, up in ((8193, 64, 0), (64, 8193, 0), (4096, 64, 1), (64, 4096, 1)):
        r = L.cs_extract(ctypes.c_void_p(16), w, h, w, 5, 1.0, 3.0, 0.0, up, None, None, None, 1024)
        err = L.cs_last_error()
        assert r == -2 and b"missing image or SiftData" in err and b"size limit" not in err, (w, h, up, err)
