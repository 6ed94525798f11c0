"""The detector (detect3_kernel + cap32_fixup_kernel, and the round-1 kernels) against its restatement
(tests/detect_ref.py), record by record, at every strip and row-stream seam.

Per image: the levels equal the oracle's LowPass / ScaleUp / ScaleDown chain bit for bit; the primaries' tags decode
to (gx, gy, scale, level) with the level matching the subsampling; no two primaries share a tag; the decoded set is
the restatement's kept set up to marginal extrema; every field lies in its admissible set.  Secondaries are not read:
describe_kernel writes them without empty[0], so one may carry a stale tag of an earlier submit.

The batch size selects the rows per detector stream (hs = 12 / 32 / 96 for 1 / 2..7 / >= 8 images) and the pyramid
kernel's rows per warp; the cases use only the values the pipeline picks itself."""
import ctypes

import numpy as np
import pytest

import detect_ref as dr
import oracle
import refcases
from cudasift_b200.synth import synth_image
from test_describe_gpu import split_records

pytestmark = pytest.mark.gpu

HS_OF_BATCH, SEAM_SHAPES = dr.HS_OF_BATCH, dr.SEAM_SHAPES


def oracle_levels(img, octaves, up=False):
    lv = [oracle.lowpass(oracle.scaleup(img) if up else img, 1.0)]
    for _ in range(1, octaves):
        if lv[-1].shape[0] // 2 < 1 or lv[-1].shape[1] // 2 < 1:
            break
        lv.append(oracle.scaledown(lv[-1]))
    return lv


def extract(cs, imgs, octaves=5, thresh=2.0, lowest=0.0, up=False, maxPts=32768, u8=None):
    """Records and levels of every image, from one batched submit: [(records, [levels])]."""
    h, w = imgs[0].shape
    ex = cs.Extractor(w, h, octaves, maxPts, up, batch=len(imgs))
    try:
        if u8 is not None:
            buf = np.ascontiguousarray(u8, np.uint8)
            ex.submit_host_u8(buf.ctypes.data, 1.0, thresh, lowest)
            counts = [ex.wait()]
        else:
            ptrs = []
            for i, im in enumerate(imgs):
                hp = cs.lib().cs_extractor_host_image_at(ex.handle, i)
                ctypes.memmove(hp, np.ascontiguousarray(im, np.float32).ctypes.data, w * h * 4)
                ptrs.append(hp)
            ex.submit_host_batch(ptrs, 1.0, thresh, lowest)
            counts = ex.wait_batch(len(imgs))
        out = []
        for i in range(len(imgs)):
            levels = []
            for l in range(octaves):
                try:
                    levels.append(ex.read_level(i, l))
                except cs.CudaSiftError:
                    break
            out.append((ex.device_points_at(i, counts[i]), levels))
        return out
    finally:
        ex.close()


def check_image(img, pts, levels, octaves, thresh, lowest=0.0, up=False, limit=32, tagged=True, maxPts=None,
                refs=None):
    """Assert one image's records against the restatement; returns the statistics (and the Level objects)."""
    want = oracle_levels(img, octaves, up)
    assert len(levels) == len(want)
    for l, (a, b) in enumerate(zip(levels, want)):
        nan = np.isnan(a)                     # NaN payloads differ between the GPU and the CPU; positions may not
        assert np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32)), \
            ("level", l)
    pidx, sec = split_records(pts)
    clamp = maxPts is not None and len(pts) == maxPts
    if clamp:
        pidx = pidx[pidx < maxPts - 1]        # the clamped slot is overwritten by every later record
    else:
        # a secondary comes from another peak of the orientation histogram: a record equal to its primary in every
        # field is the same keypoint written twice (a pixel tested by two items), not a secondary
        o = pts["orientation"].view(np.uint32)
        twice = [i for i, j in sec.items() if o[i] == o[j]]
        assert not twice, ("keypoints written twice", pts[twice][["xpos", "ypos", "scale", "subsampling"]][:5])
    f = np.float32(0.5 if up else 1.0)
    low0 = np.float32(lowest) * np.float32(2.0 if up else 1.0)
    tags = pts["empty"][:, 0].copy().view(np.uint32)
    if tagged:
        t = tags[pidx]
        assert len(np.unique(t)) == len(t), "two primaries share a tag"
    tot = dict(records=0, marginal=0, widest_ulp=0.0)
    refs = [] if refs is None else refs
    seen = 0
    for l, lv in enumerate(levels):
        ref = dr.Level(lv, octaves, l, thresh, low0 / np.float32(1 << l), limit, want_flags=True)
        refs.append(ref)
        s = np.float32(1 << l)
        sel = pidx[pts["subsampling"][pidx] == s]
        p = pts[sel]
        rec = dict(x=p["xpos"] / f / s, y=p["ypos"] / f / s, scale=p["scale"] / f / s, sharpness=p["sharpness"],
                   edgeness=p["edgeness"])
        if tagged:
            t = tags[sel]
            assert np.all((t >> 29) == l), ("tag level != subsampling", l)
            gx, gy, sc = t & 0x1fff, (t >> 13) & 0x1fff, (t >> 26) & 7
        else:
            sc, gy, gx = ref.locate(rec)
        st = ref.check(sc, gy, gx, rec, exact_set=not clamp)
        seen += len(sel)
        tot["records"] += st["records"]
        tot["marginal"] += st["marginal"]
        tot["widest_ulp"] = max(tot["widest_ulp"], st["widest_ulp"])
    assert seen == len(pidx), "a primary at a subsampling no level has"
    return tot


def report(name, tots):
    t = dict(records=sum(x["records"] for x in tots), marginal=sum(x["marginal"] for x in tots),
             widest_ulp=max(x["widest_ulp"] for x in tots))
    print("\n%s: %s" % (name, t))
    assert t["marginal"] <= 0.001 * t["records"], ("marginal extrema above 0.1 % of the records", t)
    return t


def run_and_check(cs, name, imgs, octaves=5, thresh=2.0, lowest=0.0, up=False, limit=32, maxPts=32768, u8=None,
                  tagged=True):
    res = extract(cs, imgs, octaves, thresh, lowest, up, maxPts, u8)
    tots = [check_image(im, pts, lv, octaves, thresh, lowest, up, limit, tagged,
                        maxPts if maxPts < 32768 else None) for im, (pts, lv) in zip(imgs, res)]
    return report(name, tots), res


# --------------------------------------------------------------------------------------------------- seam shapes
@pytest.mark.parametrize("batch", sorted(HS_OF_BATCH))
def test_seam_shapes(cs, batch):
    for w, h, octaves in SEAM_SHAPES:
        imgs = [synth_image(w, h, seed=200 + 13 * i + w) for i in range(batch)]
        t, _ = run_and_check(cs, "seam %dx%d oct%d batch %d" % (w, h, octaves, batch), imgs, octaves, thresh=1.5)
        assert t["records"] > 50 * batch


def test_mixed_batch_of_16(cs):
    w, h = 491, 195
    rng = np.random.default_rng(8)
    imgs = [np.full((h, w), 100.0, np.float32), rng.uniform(0, 255, (h, w)).astype(np.float32)]
    imgs += [synth_image(w, h, seed=300 + i) for i in range(14)]
    run_and_check(cs, "mixed batch of 16", imgs, 5, thresh=1.5)


# ----------------------------------------------------------------------------------------------- planted extrema
def blobs(w, h, centres, sigma=1.3, amp=90.0, base=100.0):
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.full((h, w), base)
    for i, (cx, cy) in enumerate(centres):
        img += (amp if i % 2 == 0 else -amp) * np.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / (2 * sigma * sigma))
    return img.astype(np.float32)


def planted_centres(w, h):
    xs = [1, 244, 245, 488, 489, w - 2]
    ys = sorted({1, 12, 13, 24, 25, 32, 33, 64, 65, 96, 97, 192, 193, h - 2})
    out = []
    for y in ys:
        for x in xs:
            if all(max(abs(x - a), abs(y - b)) > 7 for a, b in out):
                out.append((x, y))
    return out


@pytest.mark.parametrize("batch", sorted(HS_OF_BATCH))
def test_planted_extrema_on_the_seams(cs, batch):
    w, h = 600, 260
    cen = planted_centres(w, h)
    img = blobs(w, h, cen)
    res = extract(cs, [img] * batch, 5, 2.0)
    tots = []
    for pts, lv in res:
        refs = []
        tots.append(check_image(img, pts, lv, 5, 2.0, refs=refs))
        r0 = refs[0]
        listed = set(zip(r0.gx[r0.must].tolist(), r0.gy[r0.must].tolist()))
        missing = [c for c in cen if c not in listed]
        assert not missing, ("planted extrema the restatement does not list", missing)
    report("planted batch %d" % batch, tots)


def test_equal_valued_pairs_across_a_strip_seam(cs):
    w, h = 600, 120
    cen = [(244.5, 30), (488.5, 60), (244.5, 90)]
    img = blobs(w, h, cen, sigma=1.6)
    for (x, y) in cen:
        xi = int(x)
        assert np.array_equal(img[:, xi - 7:xi + 1], img[:, xi + 8:xi:-1])     # mirror image about x
    refs = []
    (pts, lv), = extract(cs, [img], 5, 1.0)
    t = check_image(img, pts, lv, 5, 1.0, refs=refs)
    r0 = refs[0]
    dog = dr.dog_planes(lv[0], 5, 0)
    for (x, y) in cen:
        xi = int(x)
        assert np.array_equal(dog[:, :, xi], dog[:, :, xi + 1])
        # both pixels of the pair are extrema under a non-strict rule at some scale, so only the strict rule drops them
        assert any(weak_extremum(dog, s, y, xi, 1.0) and weak_extremum(dog, s, y, xi + 1, 1.0) for s in range(5))
        assert not ((np.abs(r0.gy - y) <= 1) & np.isin(r0.gx, (xi, xi + 1))).any()
    report("equal pairs", [t])


def weak_extremum(dog, s, y, x, thresh):
    """|c| > thresh and c >= (or <=) every one of its 26 neighbours."""
    c = dog[s + 1, y, x]
    nb = np.delete(dog[s:s + 3, y - 1:y + 2, x - 1:x + 2].ravel(), 13)
    return bool(abs(c) > thresh and ((c >= nb).all() or (c <= nb).all()))


# ------------------------------------------------------------------------------------------------------- dense input
def test_dense_input_overflows_the_lists(cs):
    cases = [(arr, th) for arr, th in refcases.dense_cases()] + [(synth_image(640, 480, seed=9), 0.05)]
    flag_max = kp_max = 0
    tots = []
    for arr, th in cases:
        arr = np.ascontiguousarray(arr, np.float32)
        refs = []
        (pts, lv), = extract(cs, [arr], 5, th)
        tots.append(check_image(arr, pts, lv, 5, th, refs=refs))
        for r in refs:
            a, b = r.step_stats(HS_OF_BATCH[1])
            flag_max, kp_max = max(flag_max, a), max(kp_max, b)
    assert flag_max > dr.D2_LCAP and kp_max > dr.D2_KQ, (flag_max, kp_max)
    report("dense (flags per step %d, keypoints per item %d)" % (flag_max, kp_max), tots)


def test_cap_exact_set(cs):
    img = synth_image(320, 240, seed=9)
    try:
        for limit in (4, 5):
            cs.set_tuning("cap32_limit", limit)
            refs = []
            (pts, lv), = extract(cs, [img], 5, 0.05)
            t = check_image(img, pts, lv, 5, 0.05, limit=limit, refs=refs)
            dropped = sum(r.dropped for r in refs)
            assert dropped > 20, dropped
            report("cap %d (dropped %d)" % (limit, dropped), [t])
    finally:
        cs.set_tuning("cap32_limit", 32)


# ---------------------------------------------------------------------------------------------------- option paths
def test_option_paths(cs):
    run_and_check(cs, "scaleUp", [synth_image(320, 240, seed=21)], 5, 2.0, up=True)
    run_and_check(cs, "lowestScale 2", [synth_image(400, 300, seed=22)], 5, 1.5, lowest=2.0)
    run_and_check(cs, "1 octave", [synth_image(491, 195, seed=23)], 1, 1.5)
    run_and_check(cs, "7 octaves", [synth_image(491, 195, seed=24)], 7, 1.5)
    u8 = np.clip(synth_image(491, 195, seed=25), 0, 255).astype(np.uint8)
    run_and_check(cs, "8-bit upload", [u8.astype(np.float32)], 5, 1.5, u8=u8)
    img = synth_image(491, 195, seed=26)
    (pts, lv), = extract(cs, [img], 5, 1.5, maxPts=40)
    assert len(pts) == 40, "quirk Q18: the count is clamped to maxPts"
    assert np.all((pts["xpos"] >= 0) & (pts["xpos"] <= 491) & (pts["ypos"] >= 0) & (pts["ypos"] <= 195))
    report("maxPts clamp", [check_image(img, pts, lv, 5, 1.5, maxPts=40)])


def test_non_finite_pixels(cs):
    img = synth_image(491, 195, seed=27)
    img[60, 100] = np.nan
    img[120, 300] = np.inf
    _, res = run_and_check(cs, "NaN and +Inf pixels", [img], 5, 1.5)
    # the claim under test: extrema with a NaN neighbour (which the reference's fminf / fmaxf skips and the kernel's
    # strict per-neighbour test rejects) exist here, and the reference's refinement rejects every one of them
    bordering = 0
    for l, lv in enumerate(res[0][1]):
        dog = dr.dog_planes(lv, 5, l)
        ref = dr.Level(lv, 5, l, 1.5)
        for i in range(len(ref.gx)):
            if np.isnan(dog[ref.s[i]:ref.s[i] + 3, ref.gy[i] - 1:ref.gy[i] + 2, ref.gx[i] - 1:ref.gx[i] + 2]).any():
                bordering += 1
                assert not ref.may[i], "an extremum with a NaN neighbour survives the refinement"
    assert bordering > 0


def test_round1_kernels(cs):
    try:
        cs.set_tuning("legacy", 1)
        for w, h, octaves in SEAM_SHAPES:
            run_and_check(cs, "round-1 %dx%d" % (w, h), [synth_image(w, h, seed=200 + w)], octaves, 1.5, tagged=False)
    finally:
        cs.set_tuning("legacy", 0)


# ------------------------------------------------------------------------------------------------- oversized levels
@pytest.mark.parametrize("w,h,up", [(8300, 64, False), (4150, 64, True), (64, 8300, False)])
def test_levels_past_the_tag_limit_are_refused(cs, w, h, up):
    """gx and gy have 13 bits in the tag: past 8193 px, (gx, gy) and (gx - 8192, gy + 1) share a tag and the cap's
    fix-up could delete a record that was never capped."""
    with pytest.raises(cs.CudaSiftError, match="size limit of 8193"):
        cs.Extractor(w, h, 5, 1024, up)
