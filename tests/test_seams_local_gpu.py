"""cs_level_texture_seams_local on the GPU against tests/seam_local_oracle.py, after cs_level_texture_seams, on the
flat and jittered scenes with a gain, an offset and a radial falloff per view: every integer statistic, the seam
energy, every seam texel and every texel outside the free set bit for bit; the free texels within the CG bound of
the exact solution; the CG count against the oracle's PCG; statuses 1, 2 and 3; the launch count; determinism past
2048 x 256 free texels; the domain against the global call's texel count; and the dense chain's seam step."""
import numpy as np
import pytest

import cudasift_b200 as cs
import seam_local_oracle as lo
import seam_oracle as so
import texture_cases as tc
from test_seams_local_cpu import ramp, seam_step, vignetted

pytestmark = pytest.mark.gpu

TOL, STRIP = 1e-4, 20
# The chain's mean seam step after local levelling / after the global call alone.  The chain is simplified to 1 % so
# that faces are large enough for the vignetting to survive the global call's per-vertex offsets (4.00 -> 0.52 on the
# H100).  At 10 % the global call already reaches the floor the views' misregistration sets (1.18, against 0.55 for
# unperturbed views) and the local call does not lower it (1.34); DESIGN.md section 8.
CHAIN_RATIO = 0.5


@pytest.fixture(scope="module", params=[0.0, 0.3], ids=["flat", "jittered"])
def scene(request):
    imgs, Ks, Rs, ts, _ = tc.scene_views()
    v, t = tc.scene_mesh(jitter=request.param)
    atlas, uv, labels, charts = cs.TextureMesh(vignetted(imgs), Ks, Rs, ts, v, t)[:4]
    glob, _, _, gstats, _ = cs.LevelTextureSeams(v, t, atlas, uv, labels, charts)
    return v, t, glob, uv, labels, charts, gstats


def test_against_the_oracle(scene):
    v, t, atlas, uv, labels, charts, gstats = scene
    out, info, stats, ms = cs.LevelTextureSeamsLocal(v, t, atlas, uv, labels, charts, stripWidth=STRIP, tol=TOL)
    r = lo.level(v, t, labels, uv, charts, atlas, stripWidth=STRIP, tol=TOL)
    print("stats %s, oracle %s, info %s, %.2f ms" % (list(stats), r["stats"], list(info), ms))
    assert list(stats[:6]) == r["stats"][:6] and stats[7] == r["stats"][7] == 0
    assert abs(int(stats[6]) - r["stats"][6]) <= 1
    assert info[0] == r["info"][0]
    assert info[1] <= TOL
    assert stats[5] == gstats[6]                    # the domain is the global call's texel set
    # every seam texel and every texel outside the free set, bit for bit
    flat, want = out.reshape(-1), r["atlas"].reshape(-1)
    fixed = np.ones(flat.size, bool)
    fixed[r["free"]] = False
    assert np.array_equal(flat[fixed].view(np.uint32), want[fixed].view(np.uint32))
    # free texels: |delta - delta*| <= |A^-1| |r| <= tol |b| / lambda_min, plus the rounding to float
    lmin = lo.spl.eigsh(r["A"], k=1, sigma=0, which="LM", return_eigenvectors=False)[0]
    bound = TOL * np.linalg.norm(r["b"]) / lmin
    g = atlas.reshape(-1)[r["free"]].astype(np.float64)
    exact = g + r["delta"]
    err = np.abs(flat[r["free"]].astype(np.float64) - exact)
    assert err.max() <= bound + 2.0 ** -23 * np.abs(exact).max(), (err.max(), bound)
    assert abs(info[2] - r["info"][2]) <= bound


def test_statuses_and_launches(scene):
    v, t, atlas, uv, labels, charts, _ = scene
    out, info, stats, _ = cs.LevelTextureSeamsLocal(v, t, atlas, uv, labels, charts, maxIterations=1)
    assert stats[7] == 3 and stats[6] == 1
    one = np.where(labels == np.bincount(labels[labels >= 0]).argmax(), labels, -1).astype(np.int32)
    out, info, stats, _ = cs.LevelTextureSeamsLocal(v, t, atlas, uv, one, charts)
    assert stats[7] == 1 and stats[1] == stats[3] == stats[4] == stats[6] == 0
    assert np.array_equal(out.view(np.uint32), atlas.view(np.uint32)) and list(info) == [0.0] * 3
    bad = t.copy()
    bad[0, 0] = len(v)
    _, info, stats, _ = cs.LevelTextureSeamsLocal(v, bad, atlas, uv, labels, charts)
    assert list(stats) == [0] * 7 + [2] and list(info) == [0.0] * 3
    for w in (1, 7, STRIP):
        before = cs.lib().cs_launch_count()
        cs.LevelTextureSeamsLocal(v, t, atlas, uv, labels, charts, stripWidth=w)
        assert cs.lib().cs_launch_count() - before == 15 + w
    before = cs.lib().cs_launch_count()
    cs.LevelTextureSeamsLocal(v, bad, atlas, uv, labels, charts)
    assert cs.lib().cs_launch_count() - before == 2


def test_constant_atlas_is_unchanged(scene):
    v, t, atlas, uv, labels, charts, _ = scene
    const = np.full(atlas.shape, 128.0, np.float32)
    out, info, stats, _ = cs.LevelTextureSeamsLocal(v, t, const, uv, labels, charts)
    assert stats[7] == 0 and stats[6] == 0 and stats[4] > 0
    assert np.array_equal(out.view(np.uint32), const.view(np.uint32))


def test_two_calls_give_the_same_bytes(scene):
    v, t, atlas, uv, labels, charts, _ = scene
    a, b = (cs.LevelTextureSeamsLocal(v, t, atlas, uv, labels, charts) for _ in range(2))
    for x, y in zip(a[:3], b[:3]):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))


def test_determinism_past_two_levels_of_totals():
    """The analytic ramp stretched to 13 441 rows of 32-texel charts with noise on the atlas: more than 2048 x 256 free
    texels, so all three total levels run."""
    v, t, lab, uv, charts, atlas = ramp(c=32, L=420)
    atlas = atlas + np.random.default_rng(5).uniform(-10, 10, atlas.shape).astype(np.float32)
    r1 = cs.LevelTextureSeamsLocal(v, t, atlas, uv, lab, charts, padding=0, maxIterations=50)
    r2 = cs.LevelTextureSeamsLocal(v, t, atlas, uv, lab, charts, padding=0, maxIterations=50)
    print("ramp: stats %s, %.1f ms" % (list(r1[2]), r1[3]))
    assert r1[2][4] > 2048 * 256
    for x, y in zip(r1[:3], r2[:3]):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))


def test_chain_seam_step_falls():
    """The dense chain of test_seams_gpu's chain test, simplified to 1 %, with every view given its own gain, offset
    and radial falloff: the mean seam step after the global call, and after the global and the local call."""
    import stereo_cases as sc
    Ks, Rs, ts, views = sc.render(8, 320, 240, seed=2, texels=96)
    images = vignetted([v[0] for v in views], seed=5)
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(8)]) if b != a][:4], 3.0, 12.0) for a in range(8)]
    d, nr, c, _, _ = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs)
    dg, ng, cg, _, _ = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, d, nr)
    xyz, nrm, inten, _, _, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, dg, ng, cg)
    verts, tris, vint, _, _, _, _ = cs.PoissonMeshScreened(xyz, nrm, inten, depth=7, trim=0.5)
    gv, gt, gi, _, _, _ = cs.SimplifyMesh(verts, tris, vint, targetTriangles=len(tris) // 100)
    atlas, uv, labels, charts, _, _, _ = cs.TextureMesh(images, Ks, Rs, ts, gv, gt)
    glob, _, _, gstats, gms = cs.LevelTextureSeams(gv, gt, atlas, uv, labels, charts)
    out, info, stats, ms = cs.LevelTextureSeamsLocal(gv, gt, glob, uv, labels, charts)
    fc = so.build(gv, gt, labels, uv, charts, atlas)["faceChart"]
    before = seam_step(gt, labels, uv, charts, fc, atlas)
    after_g = seam_step(gt, labels, uv, charts, fc, glob)
    after_l = seam_step(gt, labels, uv, charts, fc, out)
    print("chain: %d faces, stats %s, %.1f + %.1f ms; mean seam step %.2f -> global %.2f -> local %.2f (ratio %.3f)"
          % (len(gt), list(stats), gms, ms, before, after_g, after_l, after_l / after_g))
    assert gstats[7] == 0 and stats[7] == 0 and after_l <= CHAIN_RATIO * after_g
