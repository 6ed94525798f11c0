"""GPU checks of cs_texture_mesh (TextureMesh) against tests/texture_oracle.py: labels, charts, texture coordinates,
atlas bytes, info and stats bit-equal to the oracle on the scene mesh (lambda 0, 0.5 and 5, with and without jitter)
and on a PoissonMesh -> SimplifyMesh sphere; determinism; image groups; the truncation prefixes; statuses and launch
counts; and the chain PatchMatch -> geometric pass -> fusion -> PoissonMeshScreened -> SimplifyMesh -> TextureMesh,
whose textured render must be clearly closer to the views than the per-vertex-intensity render."""
import ctypes

import numpy as np
import pytest

import cudasift_b200 as cs
import mesh_cases as mc
import stereo_cases as sc
import texture_cases as tc
import texture_oracle as to
from cudasift_b200 import synth

pytestmark = pytest.mark.gpu

ATLAS_WIDTH = 1024
# Median absolute grey-level difference of the textured render against the per-vertex-intensity render's, over the
# pixels of every view where the mesh agrees with the scene: the textured one must be at most this share of the other.
# Measured on an H100 80GB HBM3: 0.25 against 2.46 grey levels (ratio 0.103); the bound leaves 3x room.
CHAIN_RATIO = 0.3


@pytest.fixture(scope="module")
def scene():
    imgs, Ks, Rs, ts, _ = tc.scene_views()
    return imgs, Ks, Rs, ts


def _compare(got, ref):
    atlas, uv, labels, charts, info, stats, _ = got
    assert list(stats) == ref["stats"]
    assert np.array_equal(labels, ref["labels"])
    assert np.array_equal(charts, ref["charts"])
    assert np.array_equal(uv.view(np.uint32), ref["uv"].view(np.uint32))
    assert np.array_equal(atlas.view(np.uint32), ref["atlas"].view(np.uint32))
    assert list(info) == ref["info"]


@pytest.mark.parametrize("jitter", [0.0, 0.3])
@pytest.mark.parametrize("lam", [0.0, 0.5, 5.0])
def test_oracle_equality_scene(scene, lam, jitter):
    imgs, Ks, Rs, ts = scene
    v, t = tc.scene_mesh(jitter=jitter)
    got = cs.TextureMesh(imgs, Ks, Rs, ts, v, t, smoothness=lam, atlasWidth=ATLAS_WIDTH)
    ref = to.texture(imgs, Ks, Rs, ts, v, t, lam=lam, atlasWidth=ATLAS_WIDTH)
    print("scene lambda %g jitter %g: stats %s info %s" % (lam, jitter, list(got[5]), list(got[4])))
    _compare(got, ref)
    if lam == 0.0:
        assert np.array_equal(got[2], ref["start"]) and got[5][6] == 0


@pytest.fixture(scope="module")
def sphere():
    x, n = mc.sphere(20000)
    v, t, _, _, _, _, _ = cs.PoissonMesh(x, n, depth=5)
    gv, gt, _, _, _, _ = cs.SimplifyMesh(v, t, targetTriangles=len(t) // 4)
    Ks, Rs, ts = tc.ring_cameras(8, 160, 120, mc.CENTRE, 3.0)
    imgs = [synth.synth_image(160, 120, seed=50 + a).astype(np.float32) for a in range(8)]
    return imgs, Ks, Rs, ts, gv, gt


def test_oracle_equality_sphere(sphere):
    imgs, Ks, Rs, ts, v, t = sphere
    got = cs.TextureMesh(imgs, Ks, Rs, ts, v, t, smoothness=0.5, atlasWidth=ATLAS_WIDTH)
    ref = to.texture(imgs, Ks, Rs, ts, v, t, lam=0.5, atlasWidth=ATLAS_WIDTH)
    print("sphere: %d faces, stats %s" % (len(t), list(got[5])))
    _compare(got, ref)
    assert got[5][1] < len(t) // 4


def test_determinism_and_groups(sphere):
    imgs, Ks, Rs, ts, v, t = sphere
    a = cs.TextureMesh(imgs, Ks, Rs, ts, v, t, atlasWidth=ATLAS_WIDTH)
    b = cs.TextureMesh(imgs, Ks, Rs, ts, v, t, atlasWidth=ATLAS_WIDTH)
    for x, y in zip(a[:6], b[:6]):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    # groups of 3, 2 and 1 images: the same bytes, and the launch count grows by 2 per group
    counts = []
    try:
        for per in (3, 2, 1):
            assert cs.lib().cs_set_tuning(b"texture_group_bytes", per * 160 * 120 * 8) == 0
            before = cs.lib().cs_launch_count()
            c = cs.TextureMesh(imgs, Ks, Rs, ts, v, t, atlasWidth=ATLAS_WIDTH)
            counts.append((cs.lib().cs_launch_count() - before, c[5]))
            for x, y in zip(a[:6], c[:6]):
                assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
    finally:
        cs.lib().cs_set_tuning(b"texture_group_bytes", 0)
    for (n, st), groups in zip(counts, (3, 4, 8)):
        assert n == 14 + 2 * groups + st[4] + st[3] * st[5], (n, groups, list(st))


def _raw_call(imgs, Ks, Rs, ts, v, t, maxRows, maxCharts, lam=0.5, maxSweeps=100, faceChart=True):
    arrs, bufs, table = cs._upload_images(imgs)
    T = len(t)
    S = len(imgs)
    K, R, tt = (np.ascontiguousarray(np.asarray(a, np.float64)) for a in (Ks, Rs, ts))
    try:
        ins = [cs.DeviceBuffer(max(v.nbytes, 4)), cs.DeviceBuffer(max(t.nbytes, 4))]
        outs = [cs.DeviceBuffer(4 * max(maxRows, 1) * ATLAS_WIDTH), cs.DeviceBuffer(24 * T), cs.DeviceBuffer(4 * T),
                cs.DeviceBuffer(4 * T)]
        bufs += ins + outs
        ins[0].upload(np.ascontiguousarray(v, np.float32))
        ins[1].upload(np.ascontiguousarray(t, np.int32))
        charts = np.full((max(maxCharts, 1), 8), -7, np.int32)
        info, stats = np.zeros(2), np.zeros(11, np.int64)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        C = cs.lib().cs_texture_mesh(table, S, p(K), p(R), p(tt), ins[0].ptr, len(v), ins[1].ptr, T, lam, 75.0, 0.01,
                                     2, ATLAS_WIDTH, maxSweeps, outs[0].ptr if maxRows else None, maxRows,
                                     outs[1].ptr, outs[2].ptr, outs[3].ptr if faceChart else None,
                                     p(charts) if maxCharts else None, maxCharts, p(info), p(stats), None)
        rows = int(min(stats[8], maxRows))
        return dict(ret=C, stats=stats, info=info, charts=charts, atlas=outs[0].download(np.float32, rows * ATLAS_WIDTH)
                    .reshape(rows, ATLAS_WIDTH), uv=outs[1].download(np.float32, 6 * T).reshape(T, 3, 2),
                    labels=outs[2].download(np.int32, T), faceChart=outs[3].download(np.int32, T))
    finally:
        for b in bufs:
            b.free()


def test_truncation_prefixes(scene):
    imgs, Ks, Rs, ts = scene
    v, t = tc.scene_mesh(jitter=0.3)
    ref = to.texture(imgs, Ks, Rs, ts, v, t, lam=0.5, atlasWidth=ATLAS_WIDTH)
    C, full = ref["ret"], ref["stats"][8]
    for rows, nc in ((full // 3, C // 2), (0, 0), (full + 5, C + 3), (1, 1)):
        g = _raw_call(imgs, Ks, Rs, ts, v, t, rows, nc)
        assert g["ret"] == C and g["stats"][9] == min(rows, full) and list(g["stats"][:9]) == ref["stats"][:9]
        assert np.array_equal(g["atlas"], ref["atlas"][:rows])
        assert np.array_equal(g["charts"][:min(nc, C)], ref["charts"][:nc])
        assert (g["charts"][min(nc, C):] == -7).all()
        assert np.array_equal(g["uv"].view(np.uint32), ref["uv"].view(np.uint32))
        assert np.array_equal(g["faceChart"], ref["faceChart"])


def test_statuses_and_launches(scene):
    imgs, Ks, Rs, ts = scene
    v, t = tc.scene_mesh()
    before = cs.lib().cs_launch_count()
    g = _raw_call(imgs, Ks, Rs, ts, v, t, 200, 10)
    st = g["stats"]
    assert st[10] == 0 and cs.lib().cs_launch_count() - before == 14 + 2 + st[4] + st[3] * st[5]
    g3 = _raw_call(imgs, Ks, Rs, ts, v, t, 200, 10, lam=5.0, maxSweeps=1)
    ref = to.texture(imgs, Ks, Rs, ts, v, t, lam=5.0, maxSweeps=1, atlasWidth=ATLAS_WIDTH)
    assert g3["stats"][10] == 3 == ref["stats"][10] and g3["stats"][5] == 1
    assert np.array_equal(g3["labels"], ref["labels"])
    g0 = _raw_call(imgs, Ks, Rs, ts, v, t, 200, 10, maxSweeps=0)
    assert g0["stats"][10] == 3 and g0["stats"][5] == 0 and np.array_equal(g0["labels"], to.texture(
        imgs, Ks, Rs, ts, v, t, maxSweeps=0, atlasWidth=ATLAS_WIDTH)["start"].astype(np.int32))
    bad = t.copy()
    bad[3, 2] = bad[3, 0]
    before = cs.lib().cs_launch_count()
    g2 = _raw_call(imgs, Ks, Rs, ts, v, bad, 200, 10)
    assert g2["ret"] == 0 and g2["stats"][10] == 2 and cs.lib().cs_launch_count() - before == 1
    assert (g2["charts"] == -7).all()
    nan = v.copy()
    nan[t[7, 1], 0] = np.nan
    assert _raw_call(imgs, Ks, Rs, ts, nan, t, 200, 10)["stats"][10] == 2


def _render(K, R, t, W, H, verts, tris, shade):
    """The oracle's rasteriser: per covered pixel the face and its perspective-correct barycentrics; shade(f, lam)
    gives the value.  Returns (image, depth, covered)."""
    buf = to.depth_buffer(K, R, t, W, H, verts, tris)
    cov = buf != to.EMPTY
    ys, xs = np.nonzero(cov)
    f = (buf[cov] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    X = np.asarray(verts, np.float64)[np.asarray(tris, np.int64)[f]]
    u, v, z = to.project(K, R, t, X)
    w = []
    for k in range(3):
        a, b = k, (k + 1) % 3
        w.append((u[:, b] - u[:, a]) * (ys - v[:, a]) - (v[:, b] - v[:, a]) * (xs - u[:, a]))
    lam = np.stack([w[1] / z[:, 0], w[2] / z[:, 1], w[0] / z[:, 2]], 1)
    lam = lam / lam.sum(1, keepdims=True)
    out = np.zeros((H, W))
    depth = np.full((H, W), np.inf)
    out[cov] = shade(f, lam)
    depth[cov] = (buf[cov] >> np.uint64(32)).astype(np.uint32).view(np.float32)
    return out, depth, cov


def _bilinear(img, x, y):
    H, W = img.shape
    x, y = np.clip(x, 0, W - 1.001), np.clip(y, 0, H - 1.001)
    x0, y0 = np.floor(x).astype(int), np.floor(y).astype(int)
    fx, fy = x - x0, y - y0
    return ((1 - fy) * ((1 - fx) * img[y0, x0] + fx * img[y0, x0 + 1]) +
            fy * ((1 - fx) * img[y0 + 1, x0] + fx * img[y0 + 1, x0 + 1]))


def test_chain_textured_render_beats_vertex_intensity():
    Ks, Rs, ts, views = sc.render(8, 320, 240, seed=2, texels=96)
    images = [v[0] for v in views]
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(8)]) if b != a][:4], 3.0, 12.0) for a in range(8)]
    d, nr, c, _, _ = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs)
    dg, ng, cg, _, _ = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, d, nr)
    xyz, nrm, inten, _, _, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, dg, ng, cg)
    verts, tris, vint, _, _, _, _ = cs.PoissonMeshScreened(xyz, nrm, inten, depth=7, trim=0.5)
    gv, gt, gi, _, sst, _ = cs.SimplifyMesh(verts, tris, vint, targetTriangles=len(tris) // 10)
    atlas, uv, labels, charts, info, stats, ms = cs.TextureMesh(images, Ks, Rs, ts, gv, gt)
    assert stats[10] in (0, 3) and info[1] <= info[0]
    tex_err, int_err = [], []
    for a in range(8):
        H, W = images[a].shape
        def by_texture(f, lam):
            U = uv[f].astype(np.float64)
            x, y = (lam[:, :, None] * U).sum(1).T
            val = _bilinear(atlas.astype(np.float64), np.nan_to_num(x), np.nan_to_num(y))
            return np.where(np.isfinite(U).all(axis=(1, 2)), val, np.nan)
        def by_vertex(f, lam):
            return (lam * gi[gt[f]].astype(np.float64)).sum(1)
        img_t, dep, cov = _render(Ks[a], Rs[a], ts[a], W, H, gv, gt, by_texture)
        img_v, _, _ = _render(Ks[a], Rs[a], ts[a], W, H, gv, gt, by_vertex)
        with np.errstate(invalid="ignore"):
            ok = cov & (np.abs(dep - views[a][1]) <= 0.01 * views[a][1]) & np.isfinite(img_t)
        tex_err.append(np.abs(img_t[ok] - images[a][ok]))
        int_err.append(np.abs(img_v[ok] - images[a][ok]))
    mt, mv = float(np.median(np.concatenate(tex_err))), float(np.median(np.concatenate(int_err)))
    print("chain: %d -> %d faces, %d charts, %d atlas rows, unseen %d, sweeps %d, %.1f ms; median |error| textured "
          "%.2f, per-vertex intensity %.2f (ratio %.3f)" % (len(tris), len(gt), stats[7], stats[8], stats[1], stats[5],
                                                            ms, mt, mv, mt / mv))
    assert mt <= CHAIN_RATIO * mv
