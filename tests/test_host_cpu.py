"""Host-side logic of the batched pipeline that needs no GPU: the detector's work list, the standalone synthetic-input
module of the reference bench arm, the bench helpers."""
import importlib
import os
import sys

import numpy as np
import pytest

import cudasift_b200 as cs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def items(w, h, octaves, up, n, hs):
    L = cs.lib()
    cap = 200000
    out = np.zeros(4 * cap, np.uint32)
    cnt = L.cs_detector_items(w, h, octaves, int(up), n, hs, out.ctypes.data, cap)
    assert 0 <= cnt <= cap
    return out[:4 * cnt].reshape(cnt, 4).astype(np.int64)


@pytest.mark.parametrize("w,h,octaves,up,n,hs", [(1920, 1080, 5, False, 1, 16), (1920, 1080, 5, False, 3, 64), (641, 479, 4, False, 2, 32),
                                                 (150, 100, 3, True, 1, 16), (1000, 700, 7, False, 1, 16), (20, 12, 5, False, 1, 16),
                                                 (247, 131, 2, False, 1, 7), (3, 3, 1, False, 1, 16)])
def test_detector_items_cover_every_interior_pixel_once(w, h, octaves, up, n, hs):
    """Every interior pixel (1..w-2, 1..h-2) of every level of every image is tested by exactly one item and stream."""
    it = items(w, h, octaves, up, n, hs)
    lw, lh = [w * (2 if up else 1)], [h * (2 if up else 1)]
    for i in range(1, octaves):
        if lw[-1] // 2 < 1 or lh[-1] // 2 < 1:
            break
        lw.append(lw[-1] // 2); lh.append(lh[-1] // 2)
    cover = {(b, l): np.zeros((lh[l], lw[l]), np.int32) for b in range(n) for l in range(len(lw))}
    for key, x0, ry0, hsi in it:
        l, b = int(key) & 0xff, int(key) >> 8
        assert x0 % 4 == 0                                    # TMA box alignment: x0 - 4 is a multiple of 4 floats
        assert 1 <= hsi <= hs
        cols = [x0 + d for d in range(1, 245) if x0 + d <= lw[l] - 2]
        rows = [r for r in range(ry0, ry0 + 2 * hsi) if r <= lh[l] - 2]
        for r in rows:
            cover[(b, l)][r, cols] += 1
    for (b, l), c in cover.items():
        if lw[l] < 3 or lh[l] < 3:
            assert c.sum() == 0
            continue
        assert (c[1:-1, 1:-1] == 1).all(), (b, l)
        assert c[0].sum() == 0 and c[-1].sum() == 0 and c[:, 0].sum() == 0 and c[:, -1].sum() == 0
    # coarsest level first
    levels = [int(k) & 0xff for k in it[:, 0]]
    assert levels == sorted(levels, reverse=True)


def test_synth_loads_without_the_package():
    """bench.py --impl reference generates its inputs without importing cudasift_b200 (whose library it must not load)."""
    code = ("import sys; sys.path.append(%r); import synth; a = synth.synth_image(64, 48, seed=1); d = synth.synth_descriptors(8, 1); "
            "assert 'cudasift_b200' not in sys.modules; print(a.shape, d.dtype.itemsize)") % os.path.join(ROOT, "cudasift_b200")
    import subprocess
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "(48, 64) 576" in out.stdout
    from cudasift_b200.synth import synth_image
    import hashlib
    assert synth_image(64, 48, seed=1).shape == (48, 64)


def test_bench_helpers():
    sys.path.insert(0, ROOT)
    bench = importlib.import_module("bench")
    a = bench.workload_config(32, 8, 1920, 1710.62)
    b = bench.workload_config(32, 8, 1920, 1710.58)
    assert a == b and a["features_per_image"] == 1710.6
    info = bench.bind_numa(0)                  # no GPU here: must not raise, must say it did not bind
    assert isinstance(info, dict) and "bound" in info
    s = bench.ClockSampler(0)
    s.start()
    r = s.stop()
    assert "sm_mhz" in r and "reasons" in r
    assert len(bench.level_sizes()) == 5 and bench.level_sizes()[4] == (120, 67)


def test_new_abi_symbols_present():
    L = cs.lib()
    for name in ("cs_extractor_create_batch", "cs_extractor_submit_device_batch", "cs_extractor_submit_host_batch",
                 "cs_extractor_wait_batch", "cs_extractor_profile_batch", "cs_extractor_read_level", "cs_max_batch",
                 "cs_detector_items", "cs_extractor_device_points_at", "cs_extractor_host_points_at"):
        assert hasattr(L, name), name
    assert L.cs_max_batch() == 32
    assert L.cs_set_tuning(b"cap32_limit", 32) == 0 and L.cs_set_tuning(b"legacy", 0) == 0
    for key in (b"no_such_key", b"detect_variant", b"detect_skip", b"d2_variant"):   # no longer tuning keys
        assert L.cs_set_tuning(key, 1) < 0, key


def test_demo_png_decoder_matches_opencv(tmp_path):
    """examples/sift_demo.cpp decodes PNG itself (zlib inflate + the five PNG filters) and converts colour to grey with
    cv::cvtColor's fixed-point weights: checked here without a GPU (--decode-only) on grey, RGB and RGBA files written by
    OpenCV, whose encoder chooses among the filter types per row."""
    import subprocess
    cv2 = pytest.importorskip("cv2")
    from cudasift_b200 import build
    from cudasift_b200.synth import synth_image
    demo = build.build_demo()
    assert demo and os.path.exists(demo)
    rng = np.random.default_rng(5)
    base = np.clip(synth_image(333, 217, seed=3), 0, 255).astype(np.uint8)
    rgb = np.stack([base, np.roll(base, 5, 1), (rng.random(base.shape) * 255).astype(np.uint8)], axis=2)
    rgba = np.concatenate([rgb, np.full(base.shape + (1,), 200, np.uint8)], axis=2)
    for name, img, want in (("grey", base, base), ("rgb", rgb, cv2.cvtColor(rgb, cv2.COLOR_BGR2GRAY)),
                            ("rgba", rgba, cv2.cvtColor(rgb, cv2.COLOR_BGR2GRAY))):
        src, dst = str(tmp_path / (name + ".png")), str(tmp_path / (name + ".pgm"))
        assert cv2.imwrite(src, img)
        r = subprocess.run([demo, "--decode-only", src, dst], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=60)
        assert r.returncode == 0, r.stdout
        with open(dst, "rb") as f:
            assert f.readline() == b"P5\n"
            w, h = [int(v) for v in f.readline().split()]
            assert f.readline() == b"255\n"
            got = np.frombuffer(f.read(), np.uint8).reshape(h, w)
        assert np.array_equal(got, want), name


def test_bench_step_definition_is_shared_by_both_arms():
    """bench.py: both arms derive the passes per step from (steps, batch) by one rule, so the `config` objects the driver
    compares are identical, and the driver's --steps 20 gives a timed region of >= 7680 images per GPU."""
    import types
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(ROOT, "bench.py")).read()
    head = src.split("# ------------------------------------------------------------------------------------------ host placement")[0]
    ns = {"__file__": os.path.join(ROOT, "bench.py"), "__name__": "bench_head"}
    exec(compile(head, "bench_head", "exec"), ns)
    for steps in (1, 5, 20, 100, 300):
        a = types.SimpleNamespace(steps=steps, batch=32, rounds=0)
        r = ns["rounds_per_step"](a)
        assert steps * 32 * r >= ns["MIN_TIMED_IMAGES"] and (r == 1 or steps * 32 * (r - 1) < ns["MIN_TIMED_IMAGES"])
        assert ns["workload_config"](32, 8, 1920, 1710.6, r) == ns["workload_config"](32, 8, 1920, 1710.6, r)
        assert ns["workload_config"](32, 8, 1920, 1710.6, r)["images_per_step_per_gpu"] == 32 * r
    assert ns["rounds_per_step"](types.SimpleNamespace(steps=20, batch=32, rounds=3)) == 3
