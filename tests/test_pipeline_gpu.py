"""GPU tests of the extraction pipeline object: one Pipeline per (size, octaves, scaleUp, arena) serves the batched
kernels and the round-1 kernels.  The drop-in call switches between the two on one arena, a freed arena's pipeline is
dropped, a legacy extractor gives the same records on every submit, and a misaligned arena is refused."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

W, H = 640, 480
FIELDS = ("xpos", "ypos", "scale", "sharpness", "edgeness", "orientation", "subsampling", "data")


def canon(p):
    return p[np.lexsort((p["orientation"], p["scale"], p["xpos"], p["ypos"], p["subsampling"]))]


def assert_identical(a, b, what):
    a, b = canon(a), canon(b)
    assert len(a) == len(b) > 100, (what, len(a), len(b))
    for f in FIELDS:
        assert a[f].tobytes() == b[f].tobytes(), (what, f)


@pytest.fixture
def image():
    from cudasift_b200.synth import synth_image
    return synth_image(W, H, seed=41)


@pytest.fixture
def legacy(cs):
    """Switches the round-1 kernels on for the test's calls that ask for it; always off afterwards."""
    yield lambda on: cs.set_tuning("legacy", 1 if on else 0)
    cs.set_tuning("legacy", 0)


def extract_sift(cs, img, tmp, pitch=None):
    """The drop-in ExtractSift of a device copy of img (row pitch `pitch` floats) with temp memory tmp."""
    ci = cs.CudaImage().Allocate(W, H, pitch or cs.iAlignUp(W, 128), False, None, img)
    ci.Download()
    sd = cs.InitSiftData(cs.SiftData(), 8192, False, True)
    n = cs.ExtractSift(sd, ci, 5, 1.0, 3.0, 0.0, False, tmp)
    return sd._buf.download(cs.SIFT_DTYPE, n)


def test_one_arena_both_kernel_sets(cs, image, legacy):
    """Batched, legacy, round-1 by pitch, batched again: one arena and one cached pipeline, the same records."""
    tmp = cs.AllocSiftTempMemory(W, H, 5, False)
    try:
        first = extract_sift(cs, image, tmp)
        legacy(True)
        assert_identical(extract_sift(cs, image, tmp), first, "legacy")
        legacy(False)
        assert_identical(extract_sift(cs, image, tmp, pitch=W + 1), first, "odd pitch")
        assert_identical(extract_sift(cs, image, tmp), first, "batched again")
    finally:
        cs.FreeSiftTempMemory(tmp)


def test_freed_arena_pipeline_is_dropped(cs, image, legacy):
    """A new arena of the same size may take a freed arena's address: the pipeline built on the old one must be gone."""
    tmp = cs.AllocSiftTempMemory(W, H, 5, False)
    try:
        first = extract_sift(cs, image, tmp)
    finally:
        cs.FreeSiftTempMemory(tmp)
    tmp = cs.AllocSiftTempMemory(W, H, 5, False)
    try:
        assert_identical(extract_sift(cs, image, tmp), first, "new arena")
        legacy(True)
        assert_identical(extract_sift(cs, image, tmp), first, "new arena, legacy")
    finally:
        cs.FreeSiftTempMemory(tmp)


def test_repeated_legacy_submits(cs, image, legacy):
    """A legacy extractor gives every submit, the second and later included, the records of a single call."""
    from cudasift_b200.synth import synth_image
    imgs = [image, synth_image(W, H, seed=42)]
    legacy(True)
    want = [cs.extract_host(im) for im in imgs]
    ex = cs.Extractor(W, H, 5, 32768, False)
    try:
        devs = []
        for im in imgs:
            ci = cs.CudaImage().Allocate(W, H, cs.iAlignUp(W, 128), False, None, im)
            ci.Download()
            devs.append(ci)
        for k in range(6):
            i = k % 2
            ex.submit_device(devs[i].d_data, devs[i].pitch, 1.0, 3.0, 0.0)
            n = ex.wait()
            assert_identical(ex.device_points_at(0, n), want[i], ("device", k))
        for k in range(6):
            i = k % 2
            ex.submit_host(imgs[i].ctypes.data, 1.0, 3.0, 0.0)
            n = ex.wait()
            assert_identical(ex.host_points(n).copy(), want[i], ("host", k))
    finally:
        ex.close()


def test_offset_arena_is_refused(cs, image):
    """Temp memory 4 bytes past an allocation is refused before any launch (CS_E_ARG, naming the alignment), and the
    next call with aligned temp memory is unaffected."""
    tmp = cs.AllocSiftTempMemory(W, H, 5, False)
    try:
        want = extract_sift(cs, image, tmp)
        with pytest.raises(cs.CudaSiftError, match="16-byte aligned"):
            extract_sift(cs, image, tmp + 4)
        assert_identical(extract_sift(cs, image, tmp), want, "after the refusal")
    finally:
        cs.FreeSiftTempMemory(tmp)
