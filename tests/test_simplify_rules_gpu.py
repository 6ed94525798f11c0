"""GPU checks of cs_simplify_mesh (SimplifyMesh) rule by rule against tests/simplify_oracle.py: every case runs on the
GPU and in the float64 oracle with the same arguments, and the stats must be equal, the triangles integer-equal and
the vertices, intensities and info bit-equal.  The cases reach the frozen test on non-manifold vertices, the link,
boundary and flip refusals, the minimiser's fallback and its tie order, zero-area faces, A = 0, float32 keys that
underflow or overflow, boundaryWeight, maxError, every target, permuted and unused vertex ids, several components,
block-edge sizes, truncated outputs, and fans, where every closed ring holds the centre.  Flat grids must reach their
budget: with every error 0 the tie order alone decides how many edges a pass selects."""
import ctypes
import math

import numpy as np
import pytest

import cudasift_b200 as cs
import simplify_cases as scs
import simplify_oracle as so

pytestmark = pytest.mark.gpu

FLT_MAX = float(np.finfo(np.float32).max)
FLT_MIN = float(np.finfo(np.float32).tiny)
# Passes the oracle needs to take a flat grid to 10 % with the tie order s(id) (133 at 40 x 40, 177 at 64 x 64), with
# a 10 % margin.  With the raster tie order a pass selects one edge and both grids end at the 1000-pass cap.
FLAT_PASS_BOUND = {40: 150, 64: 200}
FAN_CAP_TRIANGLES = 2100   # more faces than 1000 passes of one collapse can drop: the call ends at the pass cap


def _bits(a, dtype):
    return np.ascontiguousarray(a, dtype).view(np.uint32 if dtype == np.float32 else np.uint64)


def _inten(v, seed=5):
    return np.random.default_rng(seed).uniform(0, 1, len(v)).astype(np.float32)


def compare(v, t, inten=None, target=0, maxError=math.inf, boundaryWeight=1.0):
    """Run the GPU and the oracle on the same arguments and assert that every output is equal; returns both."""
    gv, gt, gi, info, stats, _ = cs.SimplifyMesh(v, t, inten, targetTriangles=target, maxError=maxError,
                                                 boundaryWeight=boundaryWeight)
    ref = so.simplify(v, t, inten, target=target, maxError=maxError, boundaryWeight=boundaryWeight)
    assert list(stats) == ref["stats"]
    assert np.array_equal(gt, ref["triangles"])
    assert np.array_equal(_bits(gv, np.float32), _bits(ref["vertices"], np.float32))
    assert np.array_equal(_bits(info[:1], np.float64), _bits([ref["info"]], np.float64))
    if inten is not None:
        assert np.array_equal(_bits(gi, np.float32), _bits(ref["intensity"], np.float32))
    else:
        assert gi is None
    return (gv, gt, gi, info, stats), ref


# ---- topology: rules 1 and 4 ------------------------------------------------------------------------------------------
TOPOLOGY = {
    "bowtie": scs.bowtie,
    "tetrahedron": scs.tetrahedron,
    "three_faces": lambda: scs.three_faces()[:2],
    "flipped": lambda: scs.flipped()[:2],
    "grid": lambda: scs.grid(6),
    "two_chains": scs.two_chains,
    "cycle_and_chain": scs.cycle_and_chain,
    "four_faces": scs.four_faces,
    "mobius": scs.mobius,
    "repeated_face": scs.repeated_face,
    "pillow": scs.pillow,
}
# frozen vertices the oracle's rule 1 gives each mesh (the GPU must agree through stats[1])
FROZEN = {"bowtie": 1, "two_chains": 1, "cycle_and_chain": 1, "three_faces": 2, "four_faces": 2, "flipped": 3,
          "repeated_face": 3, "mobius": 2}


@pytest.mark.parametrize("with_inten", [False, True])
@pytest.mark.parametrize("case", sorted(TOPOLOGY))
def test_topology(case, with_inten):
    v, t = TOPOLOGY[case]()
    for target in (0, len(t) // 2):
        (gv, _, _, _, stats), ref = compare(v, t, _inten(v) if with_inten else None, target=target)
        assert stats[1] == FROZEN.get(case, 0)
        # a frozen vertex never moves
        for x in np.flatnonzero(ref["frozen"]):
            assert any(np.array_equal(p, v[x]) for p in gv), (case, x)
    if case in ("tetrahedron", "pillow"):
        assert stats[8] == 1 and stats[3] == 0 and stats[5] == len(t)


# ---- geometry: rules 2, 3 and 6 ---------------------------------------------------------------------------------------
GEOMETRY = {
    "collinear": scs.collapsed_rows,
    "coincident": lambda: scs.collapsed_rows(coincident=True),
    "flat": lambda: scs.grid(8),
    "flat_jittered": lambda: scs.grid(8, jitter=0.2),
    "folded": scs.folded_grid,
    "box": scs.box,
    "tilted": scs.tilted_grid,
    "tilted_jittered": lambda: scs.tilted_grid(8, jitter=0.2, seed=2),
    "bumpy": scs.bumpy_grid,
}


@pytest.mark.parametrize("with_inten", [False, True])
@pytest.mark.parametrize("case", sorted(GEOMETRY))
def test_geometry(case, with_inten):
    v, t = GEOMETRY[case]()
    for target in (0, len(t) // 4):
        compare(v, t, _inten(v) if with_inten else None, target=target)


def test_zero_area_vertices_have_no_quadric():
    """Row 0 of collapsed_rows has only zero-area faces: A = 0 and Q = 0, so its collapses cost 0 with error 0."""
    v, t = scs.collapsed_rows()
    st = so.setup(v, t, None, math.inf, 1.0)
    assert all(st["A"][x] == 0.0 and not any(st["Q"][x]) for x in range(6))
    (_, _, _, _, stats), _ = compare(v, t, _inten(v))
    assert stats[3] > 0


@pytest.mark.parametrize("with_inten", [False, True])
@pytest.mark.parametrize("scale", [1e-20, 1e20])
def test_scaled_keys(scale, with_inten):
    """The same meshes at 1e-20 (errors below FLT_MIN: subnormal or zero float32 keys) and at 1e20 (errors above
    FLT_MAX: finite in float64, infinite keys), so many keys tie in their float part and the tie order decides."""
    for v, t in (scs.bumpy_grid(), scs.sphere_mesh(10, 3.3, jitter=0.1)[:2]):
        v = (v.astype(np.float64) * scale).astype(np.float32)
        e = np.array(_first_errors(v, t))
        assert ((0 < e) & (e < FLT_MIN)).any() if scale < 1 else ((FLT_MAX < e) & (e < math.inf)).any()
        (_, _, _, _, stats), _ = compare(v, t, _inten(v) if with_inten else None, target=len(t) // 5)
        assert stats[8] == 0 and stats[3] > 0


def _first_errors(v, t):
    """The errors of the input's admissible edges (the oracle's first pass)."""
    st = so.setup(v, t, None, math.inf, 1.0)
    vf = so.adjacency(st["tris"], len(v))
    out = [so.evaluate(st, vf, f, k) for f in range(len(t)) for k in range(3)]
    return [r[0] for r in out if r is not None]


# ---- arguments --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sheet():
    return scs.sheet_mesh(depth=4)[:2]


@pytest.mark.parametrize("bw", [0.0, 0.25, 1.0, 4.0, 1000.0])
def test_boundary_weight(sheet, bw):
    for v, t in (sheet, scs.grid(8, jitter=0.2, seed=4)):
        compare(v, t, _inten(v), target=len(t) // 10, boundaryWeight=bw)


def test_boundary_weight_moves_the_result(sheet):
    """boundaryWeight reaches the kernels: 0 and 1000 give other outputs than the default on the sheet."""
    v, t = sheet
    out = [cs.SimplifyMesh(v, t, targetTriangles=len(t) // 10, boundaryWeight=bw)[0] for bw in (0.0, 1.0, 1000.0)]
    assert not np.array_equal(out[0], out[1]) and not np.array_equal(out[2], out[1])


@pytest.mark.parametrize("max_error", [0.0, 1e-3, 0.01, 0.05, 0.2])
def test_max_error(sheet, max_error):
    for v, t in (sheet, scs.bumpy_grid(seed=3)):
        (_, _, _, info, stats), _ = compare(v, t, maxError=max_error)
        assert stats[8] == 1 and info[0] <= max_error


def test_every_target():
    v, t = scs.bumpy_grid(seed=1)
    inten = _inten(v)
    T0 = len(t)
    for target in range(T0 + 2, -1, -1):
        (_, gt, _, _, stats), _ = compare(v, t, inten, target=target)
        if target >= T0:
            assert stats[2] == 0 and len(gt) == T0
        elif stats[8] == 0:
            assert target - 1 <= len(gt) <= target


def test_target_at_or_above_input():
    v, t = scs.box()
    for target in (len(t), len(t) + 1, 10 * len(t)):
        (gv, gt, _, _, stats), _ = compare(v, t, _inten(v), target=target)
        assert stats[8] == 0 and stats[2] == 0 and stats[3] == 0
        assert np.array_equal(gt, t) and np.array_equal(gv, v)


# ---- layout -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_permuted_ids(seed):
    for v, t in (scs.sphere_mesh(10, 3.3)[:2], scs.bumpy_grid(seed=seed)):
        pv, pt, pi = scs.permuted(v, t, seed, _inten(v))
        compare(pv, pt, pi, target=len(t) // 4)


def test_unused_vertices_with_nan():
    for v, t in (scs.bumpy_grid(seed=2), scs.box()):
        inten = _inten(v)
        uv, ut, ui = scs.with_unused(v, t, inten=inten)
        assert np.isnan(uv).any() and len(uv) == 11 * len(v)
        for i in (None, ui):
            (gv, _, _, _, stats), _ = compare(uv, ut, i, target=len(t) // 4)
            assert stats[8] == 0 and not np.isnan(gv).any()


def test_components():
    parts = [scs.sphere_mesh(10, 3.3)[:2], scs.torus_mesh(12, 3.4, 1.4)[:2], scs.bowtie(), scs.fan(21),
             scs.grid(6, jitter=0.2)]
    v, t = scs.components(*parts)
    inten = _inten(v)
    for target in (0, len(t) // 5):
        (_, _, _, _, stats), _ = compare(v, t, inten, target=target)
        assert stats[1] == 1


# (V, T): V and 3T on both sides of the 256-thread block edges, V at 2^k and 2^k + 1 (the corner sort's radix bits)
SIZES = [(256, 85), (257, 86), (255, 253), (256, 254), (257, 255), (512, 256), (513, 257), (1024, 341), (1025, 342)]


@pytest.mark.parametrize("V,T", SIZES)
def test_block_edges(V, T):
    v, t = scs.strip(T, seed=T)
    pad = np.random.default_rng(V).uniform(-3, 3, (V - len(v), 3)).astype(np.float32)
    v = np.concatenate([v, pad])
    assert len(v) == V and len(t) == T
    inten = _inten(v)
    for target in (0, T // 3):
        compare(v, t, inten, target=target)


def test_truncated_outputs_with_intensity():
    v, t = scs.bumpy_grid(seed=4)
    inten = _inten(v)
    target = len(t) // 3
    full, ref = compare(v, t, inten, target=target)
    nv, nt = len(full[0]), len(full[1])
    W, U = nv // 2, nt // 3
    bufs = [cs.DeviceBuffer(v.nbytes), cs.DeviceBuffer(t.nbytes), cs.DeviceBuffer(inten.nbytes),
            cs.DeviceBuffer(12 * W), cs.DeviceBuffer(4 * W), cs.DeviceBuffer(12 * U)]
    try:
        for b, a in zip(bufs, (v, np.ascontiguousarray(t, np.int32), inten)):
            b.upload(a)
        stats, info = np.zeros(9, np.int64), np.zeros(1)
        n = cs.lib().cs_simplify_mesh(bufs[0].ptr, bufs[2].ptr, len(v), bufs[1].ptr, len(t), target, math.inf, 1.0,
                                      bufs[3].ptr, bufs[4].ptr, W, bufs[5].ptr, U,
                                      info.ctypes.data_as(ctypes.c_void_p), stats.ctypes.data_as(ctypes.c_void_p),
                                      None)
        assert n == nt and list(stats[:6]) == ref["stats"][:6] and stats[6] == W and stats[7] == U
        assert stats[8] == ref["stats"][8] and info[0] == ref["info"]
        assert np.array_equal(_bits(bufs[3].download(np.float32, 3 * W), np.float32),
                              _bits(full[0][:W].ravel(), np.float32))
        assert np.array_equal(_bits(bufs[4].download(np.float32, W), np.float32), _bits(full[2][:W], np.float32))
        assert np.array_equal(bufs[5].download(np.int32, 3 * U).reshape(U, 3), full[1][:U])
    finally:
        for b in bufs:
            b.free()


# ---- fans and flat grids: how many edges a pass selects ---------------------------------------------------------------
@pytest.mark.parametrize("closed", [False, True])
def test_fan_one_collapse_per_pass(closed):
    v, t = scs.fan(64 if closed else 65, closed=closed)
    assert len(t) == 64
    (_, _, _, _, stats), _ = compare(v, t, _inten(v))
    assert stats[2] == stats[3] > 0


def test_fan_reaches_the_pass_cap():
    """Too large for the oracle (its closed rings make it cubic in the fan's size): the call's structure only."""
    v, t = scs.fan(FAN_CAP_TRIANGLES + 1)
    T0 = len(t)
    gv, gt, _, _, stats, _ = cs.SimplifyMesh(v, t)
    assert stats[8] == 3 and stats[2] == so.MAX_PASSES and stats[3] == so.MAX_PASSES
    assert T0 - 2 * stats[3] <= stats[5] <= T0 - stats[3] and len(gt) == stats[5]
    # still a fan: the centre (vertex 0, the lowest id, which every collapse at it keeps) is in every face
    assert (gt == 0).any(axis=1).all()
    assert so.manifold_apart_from(gt, []) and so.boundary_loops(gt) == 1


@pytest.mark.parametrize("n", sorted(FLAT_PASS_BOUND))
def test_flat_grid_reaches_its_budget(n):
    v, t = scs.grid(n)
    target = len(t) // 10
    _, gt, _, _, stats, _ = cs.SimplifyMesh(v, t, targetTriangles=target)
    print("flat %d x %d: %d -> %d triangles, status %d, %d passes, %d collapses"
          % (n, n, len(t), len(gt), stats[8], stats[2], stats[3]))
    assert stats[8] == 0 and target - 1 <= len(gt) <= target
    assert stats[2] <= FLAT_PASS_BOUND[n]
    if n <= 40:                # the oracle takes about 20 s at 64 x 64
        compare(v, t, target=target)
