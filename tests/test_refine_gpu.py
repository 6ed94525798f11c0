"""GPU checks of cs_mesh_refine (RefineMesh) against tests/refine_oracle.py: the output vertices, info [4] and stats [8]
bit-equal to the oracle on every case of refine_cases and on the small jittered scene, at 4 to 8 candidate
evaluations; two calls give the same bytes; maxIterations 0 returns the input bytes and E_0; pitched images; statuses
1, 2 and 3; the launch count against the header's formula; and on the jittered scene at 640 x 480 with 8 views, a lower
E and an RMS distance to the true planes that falls by at least the factor the oracle's run in test_refine_cpu.py
showed."""
import ctypes

import numpy as np
import pytest

import cudasift_b200 as cs
import refine_cases as rc
import refine_oracle as ro
from test_dense_pitch_gpu import _pitched_upload
from test_refine_cpu import DEFAULTS, RMS_FACTOR

pytestmark = pytest.mark.gpu


def run(c, upload=None, **over):
    """cs_mesh_refine on a case with every output; returns (vertices, info, stats, return value, launches)."""
    kw = DEFAULTS | c["kw"] | over
    v, t, imgs = c["v"], c["t"], c["imgs"]
    V, T = len(v), len(t)
    pairs = np.ascontiguousarray(np.asarray(c["pairs"], np.int32).reshape(-1, 2))
    arrs, bufs, table = (upload or cs._upload_images)(imgs)
    K, R, tt = (np.ascontiguousarray(np.asarray(a, np.float64)) for a in (c["Ks"], c["Rs"], c["ts"]))
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    try:
        ins = [cs.DeviceBuffer(max(v.nbytes, 4)), cs.DeviceBuffer(max(t.nbytes, 4)), cs.DeviceBuffer(max(v.nbytes, 4))]
        bufs += ins
        if V:
            ins[0].upload(np.ascontiguousarray(v, np.float32))
            ins[2].upload(np.full((V, 3), -7.0, np.float32))
        if T:
            ins[1].upload(np.ascontiguousarray(t, np.int32))
        info, stats = np.full(4, -1.0), np.full(8, -1, np.int64)
        before = cs.lib().cs_launch_count()
        r = cs.lib().cs_mesh_refine(table, len(imgs), p(K), p(R), p(tt), ins[0].ptr, V, ins[1].ptr, T,
                                    p(pairs) if len(pairs) else None, len(pairs), kw["windowRadius"],
                                    kw["smoothness"], kw["step"], kw["maxIterations"], kw["depthTol"], ins[2].ptr,
                                    p(info), p(stats), None)
        launches = cs.lib().cs_launch_count() - before
        assert r >= 0, cs.lib().cs_last_error()
        out = ins[2].download(np.float32, 3 * V).reshape(V, 3)
        return out, info, [int(x) for x in stats], r, launches
    finally:
        for b in bufs:
            b.free()


def oracle(c, **over):
    kw = DEFAULTS | c["kw"] | over
    return ro.refine(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], c["pairs"], **kw)


def launch_count(st):
    if st[7] == 2:
        return 1
    if st[4] == 0:
        return 0
    return 5 + st[4] * (5 * st[0] + 5) + st[4] - 1


def compare(got, ref):
    out, info, stats, r, launches = got
    assert stats == ref["stats"], (stats, ref["stats"])
    assert r == ref["stats"][7]
    assert np.asarray(info).tobytes() == np.asarray(ref["info"], np.float64).tobytes(), (info, ref["info"])
    assert out.tobytes() == np.asarray(ref["vertices"], np.float32).tobytes()
    assert launches == launch_count(stats), (launches, stats)


@pytest.mark.parametrize("iters", [4, 8])
@pytest.mark.parametrize("name", sorted(rc.CASES))
def test_cases(name, iters):
    c = rc.CASES[name]()
    ref = oracle(c, maxIterations=iters)
    got = run(c, maxIterations=iters)
    print("%s %d: info %s stats %s" % (name, iters, got[1], got[2]))
    compare(got, ref)


def test_scene_small():
    c = rc.scene()
    ref = oracle(c, maxIterations=6)
    compare(run(c, maxIterations=6), ref)


def test_repeats_and_zero_iterations():
    c = rc.repeated()
    a, b = run(c), run(c)
    for x, y in zip(a[:3], b[:3]):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
    z = run(c, maxIterations=0)
    ref = oracle(c, maxIterations=0)
    assert z[0].tobytes() == c["v"].tobytes() and z[2][7] == 3 and z[2][4] == 1
    assert np.asarray(z[1][:2]).tobytes() == np.asarray(ref["info"][:2]).tobytes() == np.asarray(a[1][:2]).tobytes()
    assert np.asarray(z[1][2:]).tobytes() == np.asarray(z[1][:2]).tobytes()


def test_pitched_images(monkeypatch):
    c = rc.windows_cut()
    dense = run(c, maxIterations=6)
    pitched = run(c, upload=_pitched_upload, maxIterations=6)
    for x, y in zip(dense[:3], pitched[:3]):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
    assert dense[2][5] > 0
    with monkeypatch.context() as m:
        m.setattr(cs, "_upload_images", _pitched_upload)
        out, info, stats, _ = cs.RefineMesh(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], c["pairs"],
                                            **(DEFAULTS | c["kw"] | dict(maxIterations=6)))
    assert out.tobytes() == dense[0].tobytes() and list(stats) == dense[2]


def test_statuses():
    c = rc.repeated()
    s3 = run(c, maxIterations=2)
    assert s3[2][7] == 3 and s3[2][4] == 3
    none = dict(c, pairs=np.zeros((0, 2), np.int32))
    s1 = run(none)
    ref1 = oracle(none)
    compare(s1, ref1)
    assert s1[2][7] == 1 and s1[0].tobytes() == c["v"].tobytes() and s1[2][3] == 0
    bad = dict(c, t=c["t"].copy())
    bad["t"][3, 2] = bad["t"][3, 0]
    s2 = run(bad)
    assert s2[2][7] == 2 and s2[4] == 1 and (s2[1] == 0).all()
    empty = dict(c, t=np.zeros((0, 3), np.int32))
    s0 = run(empty)
    assert s0[2] == [len(c["pairs"]), 0, len(c["v"]), 0, 0, 0, 0, 1] and s0[4] == 0
    assert s0[0].tobytes() == c["v"].tobytes()
    s00 = run(rc.rejects())
    assert s00[2][7] in (0, 3) and s00[2][4] > s00[2][5] + 1


def test_jittered_scene_640():
    c = rc.scene(n=8, width=640, height=480)
    out, info, stats, _ = cs.RefineMesh(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], c["pairs"])
    free = np.zeros(len(c["v"]), bool)
    free[:] = ro.topology(len(c["v"]), c["t"], c["v"].astype(np.float64))["free"]
    before = rc.plane_rms(c["v"], c["rect"], c["rects"], free)
    after = rc.plane_rms(out, c["rect"], c["rects"], free)
    E = lambda a, b: a + DEFAULTS["smoothness"] * b
    print("640x480 x 8: info %s stats %s rms %.5f -> %.5f" % (info, stats, before, after))
    assert E(info[2], info[3]) < E(info[0], info[1])
    assert after <= RMS_FACTOR * before
