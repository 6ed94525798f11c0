"""The describe stage (describe_kernel) against its float64 restatement (tests/describe_ref.py), record by record.

(a) Every record of real extractions: the batched extractor's records and pyramid levels; each primary's
    pre-describe keypoint is recovered exactly (positions divided by powers of two).
(b) Crafted keypoints through cs_describe_points: flat windows (Q21), saturated edges (Q22), borders and large
    scales, two equal peaks, Q1 and secondary-slot overflow, run-to-run identity.

No fraction of records is exempt.  Orientation decisions within the restatement's margin (near-ties) may go either
way, but only to one of the tied candidates; descriptors must lie within the restatement's per-element bound."""
import numpy as np
import pytest

import describe_ref as dr
import refcases
from cudasift_b200.records import SIFT_DTYPE
from cudasift_b200.synth import synth_image

pytestmark = pytest.mark.gpu

WRITTEN = ("xpos", "ypos", "scale", "sharpness", "edgeness", "orientation", "subsampling", "data")


def raw(a):
    return np.ascontiguousarray(a).tobytes()


def split_records(pts):
    """(primary indices, {primary index: secondary index}): a secondary is the higher-index record of a pair sharing
    subsampling, x, y, scale, sharpness and edgeness."""
    key = {}
    sec = {}
    for i, r in enumerate(pts):
        k = tuple(np.asarray([r[f] for f in ("subsampling", "xpos", "ypos", "scale", "sharpness", "edgeness")],
                             np.float32).view(np.uint32))
        if k in key:
            assert key[k] not in sec, "three records share one keypoint"
            sec[key[k]] = i
        else:
            key[k] = i
    return np.array(sorted(key.values()), np.int64), sec


def check_level(lv, px, py, ps, prim, sec, may_have_secondary):
    """Assert the kernel's records of one level (primary records `prim`, secondaries `sec` as a list aligned with
    prim, None where absent) against the restatement.  Returns the statistics."""
    n = len(px)
    o = dr.orientations(lv, px, py, ps)
    got1 = prim["orientation"].astype(np.float64)
    flat = o["flat"]
    assert np.all(np.isnan(got1[flat])), "a window without a peak has a NaN orientation"
    ok1 = dr.match_orientation(o, got1, o["cand1"]) | flat
    assert ok1.all(), ("primary orientation", np.nonzero(~ok1)[0][:5], got1[~ok1][:5], o["ori1"][~ok1][:5])
    has2 = np.array([s is not None for s in sec], bool)
    if not may_have_secondary:
        assert not has2.any(), "quirk Q1: no secondary at the finest subsampling"
    else:
        sure = o["has2_certain"]
        bad = sure & (has2 != o["has2"])
        assert not bad.any(), ("secondary decision", np.nonzero(bad)[0][:5], o["ratio_margin"][bad][:5])
    near_tie = int((o["near_tie"] & ~flat).sum())
    recs = [prim]
    kp = [np.arange(n)]
    if has2.any():
        idx = np.nonzero(has2)[0]
        s2 = np.concatenate([sec[i] for i in idx])
        ok2 = dr.match_orientation({k: v[idx] for k, v in o.items()}, s2["orientation"].astype(np.float64),
                                   o["cand2"][idx])
        assert ok2.all(), ("secondary orientation", s2["orientation"][~ok2][:5])
        recs.append(s2)
        kp.append(idx)
    recs = np.concatenate(recs)
    kp = np.concatenate(kp)
    d = dr.descriptors(lv, px[kp], py[kp], ps[kp], recs["orientation"])
    got = recs["data"].astype(np.float64)
    fin = np.isfinite(got).all(1)
    assert np.array_equal(fin, np.isfinite(d["desc"]).all(1)), "non-finite rows where the restatement has none"
    q21 = d["q21"]
    assert np.all(np.abs(got[q21] - dr.R32) < 1e-6), "Q21 rows are constant 1/sqrt(128)"
    chk = np.nonzero(~q21)[0]
    ok, bmax, K = dr.within_bound(d, got[chk], chk)
    # a row where a perturbation within bounds could zero a gradient is either a Q21 row or within the bound
    maybe = d["q21_maybe"][chk] & np.all(np.abs(got[chk] - dr.R32) < 1e-6, 1)
    assert (ok | maybe).all(), ("descriptor outside the bound", chk[~(ok | maybe)][:5])
    loose = int((bmax >= 0.2).sum())
    err = np.abs(got - d["desc"])
    clean = np.zeros(len(recs), bool)
    clean[chk] = ~d["amb_rows"][chk] & (K == 0) & ~d["q21_maybe"][chk]
    over = clean[:, None] & ~(err <= d["round_bound"])
    assert not over.any(), "rows without a grid-ambiguous fetch differ by more than rounding"
    amb = np.zeros(len(recs), bool)
    amb[chk] = ~clean[chk]
    return dict(kp=n, records=len(recs), near_tie=near_tie, q21=int(q21.sum()), q21_maybe=int(d["q21_maybe"].sum()),
                q22=int(d["q22"].sum()), amb_rows=int(amb.sum()), clean_rows=int(clean.sum()),
                flip_rows=int((K > 0).sum()), bound_ge_002=int((bmax >= 0.02).sum()), bound_ge_02=loose,
                bound_inf=int(np.isinf(bmax).sum()),
                err_clean=float(err[clean].max(initial=0)), err_amb=float(err[amb].max(initial=0)),
                err_q21=float(np.abs(got[q21] - dr.R32).max(initial=0)),
                bound_amb=float(np.median(bmax[amb[chk]])) if amb.any() else 0.0)


def add(tot, st):
    for k, v in st.items():
        tot[k] = max(tot.get(k, 0), v) if k.startswith("err") or k.startswith("bound") else tot.get(k, 0) + v
    return tot


CASES = [("synth1920", lambda: synth_image(1920, 1080, seed=7), dict(octaves=5, thresh=3.0)),
         ("synth641_oct4_t2", lambda: synth_image(641, 479, seed=7), dict(octaves=4, thresh=2.0)),
         ("synth640_up", lambda: synth_image(640, 480, seed=7), dict(octaves=5, thresh=3.0, up=True)),
         ("synth800_oct1", lambda: synth_image(800, 600, seed=8), dict(octaves=1, thresh=2.0)),
         ("synth800_oct7", lambda: synth_image(800, 600, seed=8), dict(octaves=7, thresh=2.0)),
         ("left_crop", lambda: refcases.left_crop(), dict(octaves=5, thresh=4.5)),
         ("dense_noise", lambda: refcases.dense_cases()[0][0], dict(octaves=5, thresh=refcases.dense_cases()[0][1]))]


@pytest.mark.parametrize("name,make,kw", CASES, ids=[c[0] for c in CASES])
def test_every_record_of_real_extractions(cs, name, make, kw):
    img = np.ascontiguousarray(make(), np.float32)
    h, w = img.shape
    up = kw.get("up", False)
    ex = cs.Extractor(w, h, kw["octaves"], 32768, up)
    pitch = cs.iAlignUp(w, 128)
    ci = cs.CudaImage().Allocate(w, h, pitch, False, None, img)
    ci.Download()
    try:
        ex.submit_device(ci.d_data, pitch, 1.0, kw["thresh"], 0.0)
        n = ex.wait()
        pts = ex.device_points_at(0, n)
        levels = []
        for l in range(kw["octaves"]):
            try:
                levels.append(ex.read_level(0, l))
            except cs.CudaSiftError:
                break
    finally:
        ex.close()
    assert 0 < n < 32768
    pidx, sec = split_records(pts)
    tot = {}
    f = np.float32(0.5 if up else 1.0)
    for l, lv in enumerate(levels):
        s = np.float32(1 << l)
        sel = pidx[pts["subsampling"][pidx] == s]
        if len(sel) == 0:
            continue
        p = pts[sel]
        px, py, ps = (p[k] / f / s for k in ("xpos", "ypos", "scale"))
        # the division is exact: multiplying back gives the record
        assert np.array_equal(px * s * f, p["xpos"]) and np.array_equal(ps * s * f, p["scale"])
        secs = [pts[sec[i]:sec[i] + 1] if i in sec else None for i in sel]
        add(tot, check_level(lv, px, py, ps, p, secs, may_have_secondary=(l > 0)))
    assert tot["kp"] == len(pidx) and tot["records"] == n, "every record checked"
    # a bound of 0.2 (the clamp) leaves an element unchecked: such rows must stay under the 1 % of rows a blanket
    # allowance would exempt, which is what the bound replaces
    assert tot["bound_ge_02"] <= 0.01 * n and tot["bound_inf"] == 0, tot
    print("\n%s: %s" % (name, tot))


# ------------------------------------------------------------------------------------------------- crafted keypoints
def records(xs, ys, ss, sub=1.0):
    r = np.zeros(len(xs), SIFT_DTYPE)
    r["xpos"], r["ypos"], r["scale"], r["subsampling"] = xs, ys, ss, sub
    r["sharpness"] = np.arange(len(xs)) + 1.0
    r["edgeness"] = 0.5
    return r


def describe(cs, level, recs, maxPts=None, finest=1.0):
    """cs_describe_points on `level` with `recs` in slots 0..n-1 of a maxPts-record buffer: (count, records)."""
    level = np.ascontiguousarray(level, np.float32)
    h, w = level.shape
    n = len(recs)
    maxPts = maxPts or 2 * n + 1
    buf = np.zeros(maxPts, cs.SIFT_DTYPE)
    buf[:n] = recs
    img = cs.CudaImage().Allocate(w, h, None, False, None, level)
    img.Download()
    db = cs.DeviceBuffer(buf.nbytes)
    db.upload(buf)
    c = cs.lib().cs_describe_points(img.d_data, w, h, img.pitch, db.ptr, n, maxPts, finest)
    assert c >= 0, cs.lib().cs_last_error()
    out = db.download(cs.SIFT_DTYPE, maxPts)
    db.free()
    return c, out


def check_crafted(cs, level, recs, finest=1.0):
    c, out = describe(cs, level, recs, finest=finest)
    n = len(recs)
    secs = {}
    for j in range(n, c):
        k = [i for i in range(n) if out["xpos"][i] == out["xpos"][j] and out["ypos"][i] == out["ypos"][j]
             and out["scale"][i] == out["scale"][j] and out["sharpness"][i] == out["sharpness"][j]]
        assert len(k) == 1
        secs[k[0]] = out[j:j + 1]
    s = np.float32(recs["subsampling"][0])
    st = check_level(level, recs["xpos"], recs["ypos"], recs["scale"], out[:n], [secs.get(i) for i in range(n)],
                     may_have_secondary=(s != np.float32(finest)))
    return st, c, out


def test_flat_window_q21(cs):
    img = synth_image(160, 160, seed=3)
    img[40:120, 40:120] = 100.0                       # exactly constant, wider than any window below
    xs = np.array([80.0, 80.0, 46.0, 80.0, 114.0, 42.5], np.float32)
    ys = np.array([80.0, 75.0, 80.0, 44.0, 116.0, 42.5], np.float32)
    ss = np.array([2.0, 3.0, 2.5, 2.0, 1.7, 2.0], np.float32)
    r = records(xs, ys, ss, 2.0)               # not the finest subsampling: Q1 does not hide a secondary
    d = dr.descriptors(img, xs, ys, ss, np.full(len(xs), 30.0, np.float32))
    assert d["q21"].all(), "every window reaches the plateau"
    st, c, out = check_crafted(cs, img, r)
    assert c == len(xs), "a window without a peak has no secondary"
    assert st["q21"] >= len(xs) and np.all(np.abs(out["data"][:len(xs)] - dr.R32) < 1e-6)
    o = dr.orientations(img, xs, ys, ss)
    assert o["flat"][0] and np.isnan(out["orientation"][0])     # fully inside: no peak, NaN orientation
    print("\nQ21:", st)


def edge_image(w=96, h=96):
    """Values falling to the right (dx = -6 at orientation 0) with a tiny rise downwards (dy = 2.8e-4): the gradient
    angle is pi - 4.7e-5 rad, inside (3.1415, pi], so angf >= 8 and angi == 8 (quirk Q22) for every sample, with
    margins to both discontinuities (angf = 8 and the wrap at pi) far above the texture rounding."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    return (200.0 - 3.0 * xx + 1.4e-4 * yy).astype(np.float32)


def test_saturated_edge_q22(cs):
    """Every vote goes through Q22.  The kernel matches the restatement that carries those votes into bin 0 of the
    next cell, and not the variant that drops them."""
    img = edge_image()
    xs = np.array([48.0, 44.0, 52.5, 47.25], np.float32)
    ys = np.array([48.0, 30.0, 60.0, 47.0], np.float32)
    ss = np.array([2.0, 1.6, 2.5, 3.0], np.float32)
    st, c, out = check_crafted(cs, img, records(xs, ys, ss))
    d = dr.descriptors(img, xs, ys, ss, out["orientation"][:4])
    d0 = dr.descriptors(img, xs, ys, ss, out["orientation"][:4], q22_carry=False)
    assert np.all(d["q22"] > 200) and not d["q21"].any() and np.isfinite(d["bound"]).all()
    assert all(len(j) == 0 for j in d["jumps"]), "no sample within reach of a discontinuity"
    got = out["data"][:4].astype(np.float64)
    assert np.all(np.abs(got - d["desc"]) <= d["bound"])
    # the variant's descriptor lies outside the band in which the kernel must agree with the carrying restatement
    assert np.all((np.abs(got - d0["desc"]) > 2.0 * d["bound"]).any(1)), "the kernel must carry Q22 votes"
    print("\nQ22:", st)


def test_borders_and_large_scales(cs):
    img = synth_image(200, 150, seed=5)
    w, h = 200, 150
    pos = [(0.0, 70.0), (0.5, 70.0), (w - 1.0, 70.0), (w - 0.5, 70.0), (100.0, 0.0), (100.0, h - 0.5),
           (0.0, 0.0), (w - 0.5, h - 0.5), (0.0, h - 1.0), (w - 1.0, 0.5)]
    scales = [1.6, 3.2, 12.0, 40.0]
    xs = np.array([p[0] for p in pos for _ in scales], np.float32)
    ys = np.array([p[1] for p in pos for _ in scales], np.float32)
    ss = np.array([s for _ in pos for s in scales], np.float32)
    tot = {}
    for sub in (1.0, 4.0):
        st, c, out = check_crafted(cs, img, records(xs, ys, ss, sub))
        add(tot, st)
        assert np.array_equal(out["xpos"][:len(xs)], xs * np.float32(sub))
    print("\nborders:", tot)


def test_two_equal_peaks(cs):
    """A roof symmetric about the keypoint: bins 0 and 16 hold equal peaks in float64.  The keypoint gets both
    orientations, 0 and 180 degrees, in either order."""
    w = 128
    x = np.arange(w, dtype=np.float64)
    img = np.tile((200 - 3 * np.abs(x - 63.5)).astype(np.float32), (w, 1))
    o = dr.orientations(img, [63.5], [64.0], [2.0])
    assert abs(o["sm"][0, 0] - o["sm"][0, 16]) <= 1e-13 * o["sm"][0, 0] and o["has2"][0] and o["near_tie"][0]
    assert set(np.nonzero(o["cand1"][0])[0]) == {0, 16}
    c, out = describe(cs, img, records([63.5], [64.0], [2.0], 2.0))
    assert c == 2
    got = np.sort(out["orientation"][:2].astype(np.float64))
    assert got[0] < 0.01 or got[1] > 359.99
    assert np.any(np.abs(got - 180.0) < 0.01)


def test_q1_and_slot_overflow(cs):
    img = synth_image(320, 240, seed=9)
    rng = np.random.default_rng(4)
    n = 200
    xs = rng.uniform(10, 310, n).astype(np.float32)
    ys = rng.uniform(10, 230, n).astype(np.float32)
    ss = rng.uniform(1.6, 4.0, n).astype(np.float32)
    # the finest subsampling: no secondaries, whatever the histogram says
    c1, out1 = describe(cs, img, records(xs, ys, ss, 1.0), maxPts=3 * n)
    assert c1 == n
    c8, out8 = describe(cs, img, records(xs, ys, ss, 8.0), maxPts=3 * n, finest=8.0)
    assert c8 == n
    # the same keypoints at another subsampling: secondaries where the restatement decides them
    o = dr.orientations(img, xs, ys, ss)
    full_n, full = describe(cs, img, records(xs, ys, ss, 2.0), maxPts=3 * n)
    nsec = full_n - n
    assert nsec >= 10 and (o["has2"] & o["has2_certain"]).sum() <= nsec <= (o["has2"] | ~o["has2_certain"]).sum()
    for f in ("orientation", "data"):
        assert raw(out1[f][:n]) == raw(full[f][:n]) == raw(out8[f][:n]), f
    key = {(r["xpos"], r["ypos"], r["scale"]): j for j, r in enumerate(full[n:full_n])}
    for extra in (0, 1, nsec // 2, nsec - 1):
        m = n + extra
        c, out = describe(cs, img, records(xs, ys, ss, 2.0), maxPts=m)
        assert c == max(min(n, m), min(n + nsec, m)) == m
        for f in WRITTEN:
            assert raw(out[f][:n]) == raw(full[f][:n]), f
        for r in out[n:m]:
            j = key[(r["xpos"], r["ypos"], r["scale"])]
            for f in WRITTEN:
                assert raw(r[f]) == raw(full[n + j][f]), f


def test_run_to_run(cs):
    img = synth_image(320, 240, seed=10)
    rng = np.random.default_rng(5)
    n = 300
    r = records(rng.uniform(0, 320, n), rng.uniform(0, 240, n), rng.uniform(1.6, 6, n), 2.0)
    c1, a = describe(cs, img, r, maxPts=2 * n)
    c2, b = describe(cs, img, r, maxPts=2 * n)
    assert c1 == c2 > n
    ka = np.lexsort((a[:c1]["orientation"], a[:c1]["ypos"], a[:c1]["xpos"]))
    kb = np.lexsort((b[:c2]["orientation"], b[:c2]["ypos"], b[:c2]["xpos"]))
    for f in WRITTEN:
        assert raw(a[:n][f]) == raw(b[:n][f]), f
        assert raw(a[:c1][ka][f]) == raw(b[:c2][kb][f]), f
