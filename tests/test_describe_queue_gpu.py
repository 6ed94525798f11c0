"""GPU tests of the describe stage's batch-wide keypoint queue: one resident wave of CTAs takes the keypoints of all
images of a batch from one counter, so images with very different keypoint counts (none at all included) share the
CTAs.  Every image must still get exactly the records and counts it gets alone, batch after batch."""
import numpy as np
import pytest

from cudasift_b200.synth import synth_image

pytestmark = pytest.mark.gpu

W, H = 1920, 1080
FIELDS = ("xpos", "ypos", "scale", "sharpness", "edgeness", "orientation", "subsampling", "data")


def canon(p):
    return p[np.lexsort((p["orientation"], p["scale"], p["xpos"], p["ypos"], p["subsampling"]))]


def dev_image(cs, img):
    pitch = cs.iAlignUp(W, 128)
    ci = cs.CudaImage().Allocate(W, H, pitch, False, None, img)
    ci.Download()
    return ci, pitch


def images():
    """dense (many small shapes), blank (no keypoints at all), and the benchmark's synthetic 1920x1080 image"""
    dense = synth_image(W, H, seed=77, shapes=8000, small=7900)
    blank = np.full((H, W), 128.0, np.float32)
    return {"dense": dense, "blank": blank, "synth": synth_image(W, H, seed=1000)}


def single(cs, ci, pitch, maxPts):
    ex = cs.Extractor(W, H, 5, maxPts, False)
    ex.submit_device(ci.d_data, pitch, 1.0, 3.0, 0.0)
    n = ex.wait()
    pts = ex.device_points_at(0, n)
    ex.close()
    return n, pts


def assert_identical(a, b, what):
    a, b = canon(a), canon(b)
    assert len(a) == len(b), (what, len(a), len(b))
    for f in FIELDS:
        assert np.array_equal(a[f], b[f]), (what, f)


def test_uneven_batches_equal_single_images(cs):
    """A batch mixing a dense image, blank images and the synthetic image, submitted four times through one extractor
    in two orders (the later submits replay the captured graph): the queue word and the orientation histograms come
    back clean, and every image gets its single-image records byte for byte."""
    maxPts = 65536
    imgs = images()
    cis = {k: dev_image(cs, v) for k, v in imgs.items()}
    pitch = cis["synth"][1]
    ref = {k: single(cs, ci, pitch, maxPts) for k, (ci, pitch) in cis.items()}
    assert ref["blank"][0] == 0
    assert 0 < ref["synth"][0] < ref["dense"][0] < maxPts, {k: v[0] for k, v in ref.items()}
    orders = (["blank", "dense", "blank", "synth", "blank"], ["synth", "blank", "blank", "blank", "dense"])
    ex = cs.Extractor(W, H, 5, maxPts, False, batch=5)
    for rep in range(4):
        order = orders[rep % 2]
        ex.submit_device_batch([cis[k][0].d_data for k in order], pitch, 1.0, 3.0, 0.0)
        counts = ex.wait_batch(len(order))
        assert counts == [ref[k][0] for k in order], (rep, counts)
        for slot, k in enumerate(order):
            assert_identical(ex.device_points_at(slot, counts[slot]), ref[k][1], (rep, slot, k))
    # a batch of one through the same extractor after the batches of five
    ex.submit_device_batch([cis["synth"][0].d_data], pitch, 1.0, 3.0, 0.0)
    counts = ex.wait_batch(1)
    assert counts == [ref["synth"][0]]
    assert_identical(ex.device_points_at(0, counts[0]), ref["synth"][1], "batch of one")
    ex.close()


def test_secondary_overflow_counts_equal_single_images(cs):
    """maxPts between the synthetic image's primaries and its primaries plus secondaries: the secondary orientations
    overflow their slots, and the counts of the batched images equal those of the single calls."""
    imgs = images()
    cis = {k: dev_image(cs, v) for k, v in imgs.items()}
    pitch = cis["synth"][1]
    n, pts = single(cs, *cis["synth"], 65536)
    # a secondary repeats its primary's position and scale with another orientation
    prim = len(np.unique(np.stack([pts["xpos"], pts["ypos"], pts["scale"], pts["subsampling"]]).T, axis=0))
    assert prim + 8 < n, (prim, n)
    maxPts = (prim + n) // 2
    ref = {k: single(cs, ci, pitch, maxPts)[0] for k, (ci, pitch) in cis.items()}
    assert ref["synth"] == maxPts and ref["dense"] == maxPts and ref["blank"] == 0, ref
    order = ["dense", "blank", "synth", "blank", "synth", "dense"]
    ex = cs.Extractor(W, H, 5, maxPts, False, batch=len(order))
    for rep in range(3):
        ex.submit_device_batch([cis[k][0].d_data for k in order], pitch, 1.0, 3.0, 0.0)
        assert ex.wait_batch(len(order)) == [ref[k] for k in order], rep
    ex.close()
