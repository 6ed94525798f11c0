"""cs_rotation_averaging on the device against its float64 statement (rotavg_oracle.py): the trace, costs, rotations
and residuals under both losses, determinism and the launch count, robustness to wrong edges, and the edge cases."""
import numpy as np
import pytest

import global_cases as gc
import rotavg_oracle as ro

pytestmark = pytest.mark.gpu

# The median rotation error (degrees, after alignment) of the images with no replaced edge, under Geman-McClure at 5
# degrees, on view_graph(seed, 100, 8, noiseDeg=0.05, outliers=0.2) for seeds 21-25: the float64 statement reaches
# 0.027-0.046 on the CPU, and the device must stay below the same bound.  The start is only as good as the spanning
# tree (DESIGN.md section 9): the weights make a replaced edge unlikely in the tree, not impossible, so these seeds show
# recovery when the tree holds few of them, not for every graph.
ROBUST_BOUND_DEG = 0.05
ROBUST_SEEDS = range(21, 26)


def _run(cs, g, N, **kw):
    R, res, inl, cost, trace, stats, ms = cs.RotationAveraging(N, g["edges"], g["Rrel"], g["weights"], **kw)
    return dict(R=R, residuals=res, inlier=inl, cost=cost, trace=trace, stats=stats)


def _oracle(g, N, refImage=0, maxIterations=50, maxLinearIterations=200, linearTol=1e-8, sigmaDeg=5.0,
            maxAngleDeg=5.0):
    return ro.average(N, g["edges"], g["Rrel"], g["weights"], refImage, maxIterations, maxLinearIterations, linearTol,
                      sigmaDeg, maxAngleDeg)


def _compare(got, want, rtol, cgSlack=0):
    """Statistics, inlier bytes, trace, costs, rotations and residuals against the oracle.  The CG counts must be equal
    (cgSlack 0), except on the large graph, where the device's fixed-order dot products and numpy's pairwise sums can put
    r.r on either side of the stop threshold (cgSlack 1 per iteration); one CG iteration more or less there moves x by
    less than linearTol |b| / diag, below the 1e-6 checked."""
    keep = [0, 1, 2, 3, 5]
    assert got["stats"][keep].tolist() == want["stats"][keep].tolist()
    assert abs(got["stats"][4] - want["stats"][4]) <= cgSlack * got["stats"][3]
    assert np.array_equal(got["inlier"], want["inlier"])
    np.testing.assert_allclose(got["trace"][:, 1], want["trace"][:, 1], rtol=0, atol=cgSlack)
    np.testing.assert_allclose(got["trace"][:, 0], want["trace"][:, 0], rtol=rtol, atol=1e-12)
    np.testing.assert_allclose(got["cost"], want["cost"], rtol=rtol, atol=1e-12)
    np.testing.assert_allclose(got["R"], want["R"], rtol=0, atol=rtol)
    np.testing.assert_allclose(got["residuals"], want["residuals"], rtol=rtol, atol=1e-9)


@pytest.mark.parametrize("sigmaDeg", [0.0, 5.0])
def test_small_graph_against_the_oracle(cs, sigmaDeg):
    g = gc.view_graph(11, 40, noiseDeg=0.5, outliers=0.1)
    _compare(_run(cs, g, 40, sigmaDeg=sigmaDeg, maxIterations=10), _oracle(g, 40, sigmaDeg=sigmaDeg, maxIterations=10),
             1e-9)


@pytest.mark.parametrize("sigmaDeg", [0.0, 5.0])
def test_hundreds_of_images_against_the_oracle(cs, sigmaDeg):
    g = gc.view_graph(12, 300, neighbours=8, noiseDeg=0.3, outliers=0.1)
    _compare(_run(cs, g, 300, sigmaDeg=sigmaDeg, maxIterations=8),
             _oracle(g, 300, sigmaDeg=sigmaDeg, maxIterations=8), 1e-6, cgSlack=1)


def test_determinism_and_launches(cs):
    L = cs.lib()
    for N, nb in ((30, 4), (3000, 10)):
        g = gc.view_graph(13, N, neighbours=nb, noiseDeg=0.3, outliers=0.1)
        n0 = L.cs_launch_count()
        a = _run(cs, g, N, maxIterations=5)
        assert L.cs_launch_count() - n0 == 1
        b = _run(cs, g, N, maxIterations=5)
        for k in ("R", "residuals", "inlier", "trace", "stats"):
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), (N, k)
        assert a["cost"] == b["cost"]


@pytest.mark.parametrize("seed", ROBUST_SEEDS)
def test_wrong_edges_are_flagged(cs, seed):
    g = gc.view_graph(seed, 100, neighbours=8, noiseDeg=0.05, outliers=0.2)
    clean = np.ones(100, bool)                                  # the inlier images: none of their edges replaced
    clean[g["edges"][g["outlier"]].ravel()] = False
    want = _oracle(g, 100, maxIterations=100)
    _, werr = ro.align(want["R"], g["Rs"])
    assert np.median(werr[clean]) < ROBUST_BOUND_DEG and (~want["inlier"][g["outlier"]]).all()
    got = _run(cs, g, 100, maxIterations=100)
    _, err = ro.align(got["R"], g["Rs"])
    assert np.median(err[clean]) < ROBUST_BOUND_DEG
    assert (~got["inlier"][g["outlier"]]).all() and got["inlier"][~g["outlier"]].all()


def test_disconnected_component_and_no_edges(cs):
    g = gc.view_graph(14, 40, noiseDeg=0.2, components=2)
    got = _run(cs, g, 40, refImage=25, maxIterations=10)
    half = np.arange(40) >= 20                                  # refImage 25's group
    assert np.isnan(got["R"][~half]).all() and np.isfinite(got["R"][half]).all()
    outside = ~half[g["edges"][:, 0]]
    assert np.isnan(got["residuals"][outside]).all() and not got["inlier"][outside].any()
    assert got["stats"][2] == 20 and got["stats"][1] == 19 and got["stats"][0] == (~outside).sum()
    _compare(got, _oracle(g, 40, refImage=25, maxIterations=10), 1e-9)
    # no edges: no CUDA call
    L = cs.lib()
    n0 = L.cs_launch_count()
    R, res, inl, cost, trace, stats, ms = cs.RotationAveraging(5, np.zeros((0, 2)), np.zeros((0, 3, 3)), [],
                                                               refImage=3)
    assert L.cs_launch_count() == n0 and ms == (0.0, 0.0)
    assert (R[3] == np.eye(3)).all() and np.isnan(R[[0, 1, 2, 4]]).all() and stats.tolist() == [0, 0, 1, 0, 0, 0]


def test_start_only(cs):
    """maxIterations = 0 evaluates the spanning tree's rotations."""
    g = gc.view_graph(15, 30, noiseDeg=1.0)
    got = _run(cs, g, 30, maxIterations=0)
    R0, _ = ro.spanning_tree(30, g["edges"], g["Rrel"], g["weights"], 0)
    np.testing.assert_allclose(got["R"], R0, rtol=0, atol=1e-12)
    assert got["cost"][0] == got["cost"][1] and got["stats"][3] == 0 and len(got["trace"]) == 0


# ---- global positioning ----

import globalpos_oracle as go                                    # noqa: E402
import triangulate_cases as tc                                   # noqa: E402
from cudasift_b200.records import SIFT_DTYPE                     # noqa: E402


class _Records:
    """One image's records (positions only) in device memory, as the wrappers take them (d_data, numPts)."""

    def __init__(self, cs, p):
        rec = np.zeros(len(p), SIFT_DTYPE)
        rec["xpos"], rec["ypos"] = p[:, 0], p[:, 1]
        self.buf = cs.DeviceBuffer(max(rec.nbytes, 8))
        if len(p):
            self.buf.upload(rec)
        self.d_data, self.numPts = self.buf.ptr, len(p)


def _scene(seed, N=20, T=150, noise=0.5):
    return tc.scene(seed, numImages=N, numTracks=T, lengths=(3, 8), noise=noise, outliers=(0.0, 0.0), away=0)


def _gp_compare(got, want, rtol):
    t, points, cost, trace, stats, ms = got
    assert stats[3] == want["stats"]["used"] and stats[4] == want["stats"]["tracks"]
    assert stats[5] == want["stats"]["images"] and stats[6] == want["stats"]["iterations"]
    np.testing.assert_array_equal(trace[:, [2, 3]], want["trace"][:, [2, 3]])
    np.testing.assert_allclose(trace[:, :2], want["trace"][:, :2], rtol=rtol, atol=1e-14)
    np.testing.assert_allclose(cost, want["cost"], rtol=rtol, atol=1e-14)
    np.testing.assert_allclose(t, want["t"], rtol=0, atol=rtol)
    np.testing.assert_allclose(points, want["points"], rtol=0, atol=rtol)


@pytest.mark.parametrize("loss", ["trivial", "cauchy"])
def test_positioning_small_scene_against_the_oracle(cs, loss):
    xy, Ks, Rs, ts, off, mem, pts = _scene(31)
    datas = [_Records(cs, p) for p in xy]
    got = cs.GlobalPositioning(datas, Ks, Rs, off, mem, seed=5, loss=loss, lossScale=0.01, maxIterations=15)
    want = go.position(xy, Ks, Rs, off, mem, seed=5, kind=cs.LOSSES[loss], lossScale=0.01, maxIterations=15)
    _gp_compare(got, want, 1e-9)


@pytest.mark.parametrize("loss", ["trivial", "soft_l1"])
def test_positioning_hundreds_of_images_against_the_oracle(cs, loss):
    xy, Ks, Rs, ts, off, mem, pts = _scene(32, N=200, T=1500)
    datas = [_Records(cs, p) for p in xy]
    got = cs.GlobalPositioning(datas, Ks, Rs, off, mem, seed=6, loss=loss, lossScale=0.01, maxIterations=8)
    want = go.position(xy, Ks, Rs, off, mem, seed=6, kind=cs.LOSSES[loss], lossScale=0.01, maxIterations=8)
    _gp_compare(got, want, 1e-6)


def test_positioning_determinism_launches_and_edge_cases(cs):
    L = cs.lib()
    for N, T in ((10, 40), (400, 6000)):
        xy, Ks, Rs, ts, off, mem, pts = _scene(33, N=N, T=T)
        datas = [_Records(cs, p) for p in xy]
        n0 = L.cs_launch_count()
        a = cs.GlobalPositioning(datas, Ks, Rs, off, mem, seed=9, maxIterations=10)
        assert L.cs_launch_count() - n0 == 3
        b = cs.GlobalPositioning(datas, Ks, Rs, off, mem, seed=9, maxIterations=10)
        for x, y in zip(a[:5], b[:5]):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), N
    # an image with NaN R and an image with a rotation but no observation get NaN t; T == 0 makes no CUDA call
    xy, Ks, Rs, ts, off, mem, pts = _scene(34, N=12, T=80)
    xy = xy + [np.zeros((0, 2), np.float32)]
    Ks, Rs = np.concatenate([Ks, Ks[:1]]), np.concatenate([Rs, Rs[:1]]).copy()
    Rs[3] = np.nan
    datas = [_Records(cs, p) for p in xy]
    t, points, cost, trace, stats, ms = cs.GlobalPositioning(datas, Ks, Rs, off, mem, maxIterations=10)
    assert np.isnan(t[[3, 12]]).all() and np.isfinite(np.delete(t, [3, 12], 0)).all() and stats[5] == 11
    want = go.position(xy, Ks, Rs, off, mem, maxIterations=10)
    np.testing.assert_allclose(t, want["t"], rtol=0, atol=1e-9)
    n0 = L.cs_launch_count()
    t, points, cost, trace, stats, ms = cs.GlobalPositioning(datas, Ks, Rs, [0], np.zeros((0, 2)))
    assert L.cs_launch_count() == n0 and np.isnan(t).all() and cost == (0.0, 0.0) and not stats.any()


def test_global_chain_end_to_end(cs):
    """VerifyEssentialBatch -> RotationAveraging -> GlobalPositioning -> TriangulateTracks -> BundleAdjust on 40 shell
    cameras: the centres within 1e-3 of the scene scale after a similarity, the final cost within 1 % of adjustment
    started from the true poses."""
    N = 40
    xy, Ks, Rs, ts, off, mem, pts = tc.scene(35, numImages=N, numTracks=1500, lengths=(4, 16), noise=0.5,
                                             outliers=(0.0, 0.0), away=0)
    datas = [_Records(cs, p) for p in xy]
    shared = {}
    for k in range(len(off) - 1):
        ms_ = mem[off[k]:off[k + 1]]
        for u in range(len(ms_)):
            for w in range(u + 1, len(ms_)):
                (a, f), (b, g) = sorted([tuple(ms_[u]), tuple(ms_[w])])
                if a != b:
                    shared.setdefault((a, b), []).append((f, g))
    pairs = [(a, b) for (a, b), fg in sorted(shared.items()) if len(fg) >= 15]
    jobs = [(datas[a], datas[b], np.array(shared[(a, b)], np.int32)) for a, b in pairs]
    K1 = np.stack([Ks[a] for a, b in pairs])
    K2 = np.stack([Ks[b] for a, b in pairs])
    E, R, t, inliers, vstats, _ = cs.VerifyEssentialBatch(jobs, K1, K2, numLoops=1024, thresh=2.0)
    counts = np.array([len(x) for x in inliers], np.float64)
    keep = counts >= 15
    edges = np.array(pairs, np.int32)[keep]
    Rabs, deg, good, *_ = cs.RotationAveraging(N, edges, R[keep], counts[keep])
    assert np.isfinite(Rabs).all()
    tg, _, _, _, gstats, _ = cs.GlobalPositioning(datas, Ks, Rabs, off, mem, maxIterations=100)
    assert np.isfinite(tg).all()
    P, _, _, inl, _, _ = cs.TriangulateTracks(datas, Ks, Rabs, tg, off, mem)
    Rb, tb, _, _, _, cost, *_ = cs.BundleAdjust(datas, Ks, Rabs, tg, off, mem, P, use=inl, maxIterations=100)
    P0, _, _, inl0, _, _ = cs.TriangulateTracks(datas, Ks, Rs, ts, off, mem)
    _, _, _, _, _, cost0, *_ = cs.BundleAdjust(datas, Ks, Rs, ts, off, mem, P0, use=inl0, maxIterations=100)
    C = -np.einsum("aji,aj->ai", Rs, ts)
    Cb = -np.einsum("aji,aj->ai", Rb, tb)
    sc, Ra, ta = go.umeyama(Cb, C)
    err = np.linalg.norm(sc * Cb @ Ra.T + ta - C, axis=1)
    assert np.max(err) < 1e-3 * tc.scale(Ks, Rs, ts), np.max(err)
    assert abs(cost[1] - cost0[1]) <= 0.01 * cost0[1], (cost, cost0)
