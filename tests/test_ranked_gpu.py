"""GPU tests of ranked batch extraction (cs_extractor_create_ranked, cs_rank_records): each image's slot holds the
records a plain extractor finds, sorted by the rank key and cut to maxPts, byte for byte and in a fixed order."""
import ctypes

import numpy as np
import pytest

from cudasift_b200.synth import synth_image

pytestmark = pytest.mark.gpu

MAXC = 32768
PAIR = ("sharpness", "subsampling", "ypos", "xpos", "scale")     # a secondary orientation shares these with its primary


def rank_sort(p):
    return p[np.lexsort((p["orientation"], p["scale"], p["xpos"], p["ypos"], p["subsampling"], -np.abs(p["sharpness"])))]


def dev_image(cs, img):
    h, w = img.shape
    pitch = cs.iAlignUp(w, 128)
    ci = cs.CudaImage().Allocate(w, h, pitch, False, None, img)
    ci.Download()
    return ci, pitch


def extract(cs, img, octaves, thresh, up, maxPts, maxCandidates=None):
    """One submit on a fresh extractor: (records of slot 0, count, candidates)."""
    h, w = img.shape
    ex = cs.Extractor(w, h, octaves, maxPts, up, maxCandidates=maxCandidates)
    ci, pitch = dev_image(cs, img)
    ex.submit_device(ci.d_data, pitch, 1.0, thresh, 0.0)
    n = ex.wait()
    out = ex.device_points_at(0, n), n, ex.candidates(0)
    ex.close()
    return out


def pair_cut(p):
    """An N that keeps a primary orientation and drops its secondary (p sorted by the rank key)."""
    same = np.ones(len(p) - 1, bool)
    for f in PAIR:
        same &= p[f][1:] == p[f][:-1]
    ks = np.nonzero(same)[0]
    assert len(ks) > 0, "no orientation pair"
    return int(ks[len(ks) // 2]) + 1


def cases():
    import refcases
    dense, th = refcases.dense_cases()[0]
    return [("1920x1080", synth_image(1920, 1080, seed=7), 5, 3.0, False),
            ("1280x960", synth_image(1280, 960, seed=7), 5, 3.0, False),
            ("641x479", synth_image(641, 479, seed=7), 4, 2.0, False),
            ("640x480up", synth_image(640, 480, seed=7), 5, 3.0, True),
            ("dense", dense, 5, th, False)]


@pytest.mark.parametrize("case", range(5), ids=[c[0] for c in cases()])
def test_ranked_equals_sort_and_trim(cs, case):
    name, img, octaves, thresh, up = cases()[case]
    plain, found, pc = extract(cs, img, octaves, thresh, up, MAXC)
    assert pc == found > 100 and found < MAXC, (name, found)
    if name == "dense":
        assert found > 3000
    want = rank_sort(plain)
    cut = pair_cut(want)
    for n in sorted({1, 100, 1000, found - 1, found, found + 5, cut}):
        got, k, cand = extract(cs, img, octaves, thresh, up, n, MAXC)
        assert k == min(n, found) and cand == found, (name, n, k, cand)
        assert got.tobytes() == want[:k].tobytes(), (name, n)


def test_fixed_order_across_submits(cs):
    """Repeated submits of one batch, the third onward through the captured graph, give the same bytes in every slot
    without any canonical sort."""
    w, h = 960, 540
    imgs = [synth_image(w, h, seed=200 + i) for i in range(4)]
    cis = [dev_image(cs, im) for im in imgs]
    ex = cs.Extractor(w, h, 5, 500, False, batch=4, maxCandidates=16384)
    first = None
    for rep in range(5):
        ex.submit_device_batch([c[0].d_data for c in cis], cis[0][1], 1.0, 3.0, 0.0)
        counts = ex.wait_batch(4)
        slots = [ex.device_points_at(i, counts[i]) for i in range(4)]
        if first is None:
            first = slots
            for s in slots:
                assert len(s) == 500 and s.tobytes() == rank_sort(s).tobytes()
        for i in range(4):
            assert slots[i].tobytes() == first[i].tobytes(), (rep, i)
    ex.close()


def test_batch_equals_single_images(cs):
    """A batch of 12 images equals 12 single-image ranked extractors slot by slot, for device and host submits."""
    w, h, n, maxc = 640, 480, 300, 8192
    imgs = [synth_image(w, h, seed=300 + i) for i in range(12)]
    singles = [extract(cs, im, 5, 3.0, False, n, maxc) for im in imgs]
    ex = cs.Extractor(w, h, 5, n, False, batch=12, maxCandidates=maxc)
    cis = [dev_image(cs, im) for im in imgs]
    for rep in range(3):
        ex.submit_device_batch([c[0].d_data for c in cis], cis[0][1], 1.0, 3.0, 0.0)
        counts = ex.wait_batch(12)
        for i in range(12):
            assert counts[i] == singles[i][1] and ex.candidates(i) == singles[i][2], (rep, i)
            assert ex.device_points_at(i, counts[i]).tobytes() == singles[i][0].tobytes(), ("device", rep, i)
    ptrs = []
    for i in range(12):
        hp = cs.lib().cs_extractor_host_image_at(ex.handle, i)
        ctypes.memmove(hp, imgs[i].ctypes.data, w * h * 4)
        ptrs.append(hp)
    ex.submit_host_batch(ptrs, 1.0, 3.0, 0.0)
    counts = ex.wait_batch(12)
    for i in range(12):
        hostp = ex.host_points_at(i, counts[i])
        assert hostp.tobytes() == ex.device_points_at(i, counts[i]).tobytes() == singles[i][0].tobytes(), ("host", i)
    ex.close()


def test_overflow_is_reported(cs):
    import refcases
    img, th = refcases.dense_cases()[0]
    _, found, _ = extract(cs, img, 5, th, False, MAXC)
    maxc = found // 2
    for n in (100, maxc):
        got, k, cand = extract(cs, img, 5, th, False, n, maxc)
        assert cand == maxc and k == min(n, maxc), (n, k, cand)
        assert got.tobytes() == rank_sort(got).tobytes()


def crafted(dtype, rng, n):
    """Records with repeated |sharpness| (both signs), shared positions and orientation pairs."""
    p = np.zeros(n, dtype)
    p["sharpness"] = rng.choice(np.float32([1.5, 2.25, 3.0, 7.0, 0.0]), n) * rng.choice(np.float32([-1, 1]), n)
    p["sharpness"][: n // 2] = rng.standard_normal(n // 2).astype(np.float32) * 10
    p["subsampling"] = rng.choice(np.float32([0.5, 1, 2, 4]), n)
    p["ypos"] = rng.integers(0, 6, n).astype(np.float32) - 0.5
    p["xpos"] = rng.integers(0, 6, n).astype(np.float32) * 1.25
    p["scale"] = rng.choice(np.float32([1.0, 1.6, -0.0, 0.5]), n)
    p["orientation"] = np.arange(n, dtype=np.float32) * 0.25      # unique: no two records equal on all six fields
    p["data"] = rng.random((n, 128)).astype(np.float32)
    p["edgeness"] = rng.random(n).astype(np.float32)
    pair = rng.random(n) < 0.3                                     # orientation pairs: copy fields 1-5 of the previous record
    pair[0] = False
    for f in PAIR:
        p[f][1:][pair[1:]] = p[f][:-1][pair[1:]]
    return p


@pytest.mark.parametrize("n", [1, 2, 37, 1000, 4099, 65536])
def test_rank_records_crafted(cs, n):
    rng = np.random.default_rng(n)
    recs = crafted(cs.SIFT_DTYPE, rng, n)
    want = rank_sort(recs)
    for maxOut in sorted({1, max(1, n // 3), n, n + 7}):
        outs = []
        for perm in range(3):
            shuf = recs[rng.permutation(n)] if perm else recs
            outs.append(cs.rank_records(shuf, maxOut))
        k = min(n, maxOut)
        for o in outs:
            assert len(o) == k and o.tobytes() == want[:k].tobytes(), (n, maxOut)


def test_legacy_rejected(cs):
    cs.set_tuning("legacy", 1)
    try:
        assert cs.lib().cs_extractor_create_ranked(640, 480, 5, 100, 0, 1, 1000) is None
        assert b"CS_E_ARG" in cs.lib().cs_last_error()
        with pytest.raises(cs.CudaSiftError):
            cs.Extractor(640, 480, 5, 100, False, maxCandidates=1000)
    finally:
        cs.set_tuning("legacy", 0)
