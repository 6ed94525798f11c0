"""Images with a row pitch above their width in every dense call that takes cs_image: UndistortImages, PatchMatchStereo,
PatchMatchStereoGeometric, FuseDepthMaps and TextureMesh must give the same bytes on pitched images as on dense ones.
The pitched images have a different pad per image (1, 7 and 64 floats; the odd pads leave rows that are not 16-byte
aligned), and the pad is NaN, so a read past a row's last pixel shows in the output."""
import numpy as np
import pytest

import cudasift_b200 as cs
import stereo_cases as sc
import texture_cases as tc

pytestmark = pytest.mark.gpu

PADS = (1, 7, 64)


def _pitched_upload(images):
    """_upload_images with image k in a buffer of rows pitch = width + PADS[k % 3] floats, the pad filled with NaN."""
    arrs = [np.ascontiguousarray(im, np.float32) for im in images]
    bufs, rows = [], []
    try:
        for k, im in enumerate(arrs):
            h, w = im.shape
            pitch = w + PADS[k % len(PADS)]
            host = np.full((h, pitch), np.nan, np.float32)
            host[:, :w] = im
            b = cs.DeviceBuffer(host.nbytes)
            bufs.append(b)
            b.upload(host)
            rows.append(cs.StereoImage(b.ptr, w, h, pitch))
    except BaseException:
        for b in bufs:
            b.free()
        raise
    table = (cs.StereoImage * max(len(arrs), 1))(*rows)
    return arrs, bufs, table


def _same(a, b):
    """Equal bytes, item by item, through nested tuples and lists of arrays and numbers."""
    if isinstance(a, (tuple, list)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
    elif isinstance(a, float) and not isinstance(b, np.ndarray):
        return                              # the call's elapsed ms
    else:
        x, y = np.ascontiguousarray(a), np.ascontiguousarray(b)
        assert x.dtype == y.dtype and x.shape == y.shape
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


def _both(monkeypatch, call):
    dense = call()
    with monkeypatch.context() as m:
        m.setattr(cs, "_upload_images", _pitched_upload)
        pitched = call()
    return dense, pitched


@pytest.fixture(scope="module")
def scene():
    Ks, Rs, ts, views = sc.render(6, 160, 120, seed=1)
    images = [v[0] for v in views]
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(6)]) if b != a][:4], 3.0, 12.0) for a in range(6)]
    return Ks, Rs, ts, images, jobs


def test_undistort(monkeypatch, scene):
    Ks, _, _, images, _ = scene
    dists = np.array([[-0.12, 0.03], [0.08, -0.02], [0.05, 0.0], [-0.04, 0.01], [0.1, -0.05], [-0.2, 0.06]])
    dense, pitched = _both(monkeypatch, lambda: cs.UndistortImages(images, Ks, dists))
    _same(dense, pitched)
    assert dense[1].sum() > 0 and all(np.isfinite(x).all() for x in pitched[0])


def test_patch_match_geometric_and_fusion(monkeypatch, scene):
    Ks, Rs, ts, images, jobs = scene
    kw = dict(windowRadius=3, windowStep=1, numIterations=3, topK=2, seed=3)
    pm = _both(monkeypatch, lambda: cs.PatchMatchStereo(images, Ks, Rs, ts, jobs, **kw))
    _same(pm[0], pm[1])
    d, n, c = pm[0][:3]
    assert all(np.isfinite(x).all() for x in d + c)
    geo = _both(monkeypatch, lambda: cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, d, n, **kw))
    _same(geo[0], geo[1])
    dg, ng, cg = geo[0][:3]
    fused = _both(monkeypatch, lambda: cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, dg, ng, cg))
    _same(fused[0], fused[1])
    assert fused[0][4] > 0 and np.isfinite(fused[1][2]).all()
    print("pitched: %d fused points" % fused[0][4])


def test_texture_mesh(monkeypatch, scene):
    Ks, Rs, ts, images, _ = scene
    v, t = tc.scene_mesh(jitter=0.3, Rs=Rs, ts=ts)
    for pad in (0, 5):
        dense, pitched = _both(monkeypatch, lambda: cs.TextureMesh(images, Ks, Rs, ts, v, t, padding=pad))
        _same(dense, pitched)
        atlas, stats = dense[0], dense[5]
        assert stats[7] > 0 and np.isfinite(pitched[0]).all()
        # some chart touches its image's right border, where a read past the row would meet the NaN pad
        W = [im.shape[1] for im in images]
        print("pitched texturing, padding %d: stats %s" % (pad, list(stats)))
        if pad:
            assert any(x0 + w == W[a] for a, x0, _, w, _, _, _, _ in dense[3])
