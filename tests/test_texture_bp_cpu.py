"""CPU checks of cs_texture_mesh_bp: (a) on random paths the kept labelling reaches the exact minimum of E that dynamic
programming gives, and the messages converge; (b) on the island case ICM keeps a higher E and BP reaches the minimum;
(c) with maxBpSweeps 0 the oracle is cs_texture_mesh_photo's on every photo case; (d) E_final <= E_kept <= E_0; (e)
each oracle mutation of rule 4b changes some case's output, so a kernel with the same slip would fail the GPU
comparison in test_texture_bp_gpu.py; (f) the argument checks, the header, and the SASS of the photo call's kernels."""
import ctypes
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
from cudasift_b200 import build
import texture_bp_cases as bc
import texture_bp_oracle as bo
import texture_cases as tc
import texture_oracle as to
import texture_photo_cases as pc
import texture_photo_oracle as tpo
from test_bundle_intrinsics_cpu import _sass
from test_texture_cpu import IMG, KS, RS, TS

CS_E_ARG = -2
_memo = {}


def _case(name):
    if name not in _memo:
        _memo[name] = {"scene": lambda: tc._case(*tc.scene_views()[:4], *tc.scene_mesh(jitter=0.3), lam=0.5),
                       **bc.CASES}[name]()
    return _memo[name]


def _run(c, **over):
    return bo.texture_bp(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], **(c["kw"] | over))


def _ref(name, **over):
    k = (name, tuple(sorted(over.items())))
    if k not in _memo:
        _memo[k] = _run(_case(name), **over)
    return _memo[k]


# ---- (a) exact on paths ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_random_paths_reach_the_minimum(seed):
    rng = np.random.default_rng(300 + seed)
    for _ in range(50):
        n = int(rng.integers(2, 30))
        lam = float(rng.uniform(0.1, 2.0))
        tris, nbr, col, cands = bc.random_path(n, rng)
        start = np.array([c[0][1] for c in cands], np.int64)
        label = start.copy()
        e0 = to.energy(label, cands, nbr, lam)
        ek, st = bo.belief_propagation(label, e0, cands, nbr, tris, col, lam, 4 * n + 8)
        best = to.energy(bc.viterbi(cands, lam), cands, nbr, lam)
        assert st[2] == 0 and st[0] <= 2 * n + 2, (n, st)
        assert ek == to.energy(label, cands, nbr, lam)
        assert ek <= best + 1e-12 * max(1.0, best), (n, lam, ek, best)
        assert st[3] == int((label != start).sum())


# ---- (b) the island -------------------------------------------------------------------------------------------------
def test_island_icm_stays_and_bp_reaches_the_minimum():
    c = _case("island")
    icm, bp = _ref("island", maxBpSweeps=0), _ref("island")
    order = c["order"]
    assert icm["info"][1] == icm["info"][0] == 1.0 and icm["stats"][6] == 0
    a, b = ISLAND_D(icm)
    assert (np.abs(np.asarray(a) - 0.3) < 0.12).all() and sum(a) < 2 * 0.5 and min(b) > 0.1
    best = to.energy(bc.viterbi([bp["cands"][f] for f in order], 0.5)[np.argsort(order)], bp["cands"], bp["nbr"], 0.5)
    assert bp["info"][2] == bp["info"][1] == best < icm["info"][1]
    assert bp["stats"][16:] == [bp["stats"][16], bp["stats"][17], 0, 3] and (bp["labels"] == 0).all()
    assert bp["ret"] == 1 and icm["ret"] == 3


def ISLAND_D(r):
    """D of the other view on the run, and on the rest of the strip."""
    D, _, _ = bo.data_terms(r["cands"])
    order = bc.path_order(r["nbr"])
    run = set(order[bc.ISLAND[0]:bc.ISLAND[1]])
    return [D[f, 1] for f in order if f in run], [D[f, 1] for f in order if f not in run]


# ---- (c) no sweeps is the photo call --------------------------------------------------------------------------------
def test_no_sweeps_is_the_photo_call():
    for name in sorted(pc.CASES):
        c = pc.CASES[name]()
        a = tpo.texture_photo(c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], **c["kw"])
        b = _run(c, maxBpSweeps=0)
        assert b["stats"][:16] == a["stats"] and b["stats"][16:] == [0] * 4, name
        for k in ("ret", "labels", "uv", "atlas", "charts", "faceChart"):
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), (name, k)
        assert b["info"] == list(a["info"]) + [a["info"][0]]


# ---- (d) the energies are ordered -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["scene", "strip", "island"])
def test_energies_are_ordered(name):
    r = _ref(name)
    e0, e1, ek = r["info"]
    assert e1 <= ek <= e0, r["info"]
    print("%s: E %.4f -> BP %.4f -> ICM %.4f, stats %s" % (name, e0, ek, e1, r["stats"][16:]))


def test_vectorised_energy_is_rule_4s():
    for name in ("scene", "strip"):
        r = _ref(name)
        D, A, _ = bo.data_terms(r["cands"])
        for lab in (r["labels"].astype(np.int64), r["start"], r["kept"]):
            assert bo.energy(lab, D, A, r["nbr"], 0.5) == to.energy(lab, r["cands"], r["nbr"], 0.5)


# ---- (e) sensitivity ------------------------------------------------------------------------------------------------
def _jacobi(D, A, m, nbr, kp, msg, col, colours, lam):
    old = msg.copy()
    new = msg.copy()
    n = 0
    for c in range(colours):
        work = old.copy()
        n += bo.colour_step(D, A, m, nbr, kp, work, col, c, lam)
        into = np.nonzero(col != c)[0]
        changed = (work[into] != old[into]).any((1, 2))
        new[into[changed]] = work[into[changed]]
    msg[:] = new
    return n


def _subtracting(D, msg, F, k):
    full = ((D[F] + msg[F, 0]) + msg[F, 1]) + msg[F, 2]
    return full - msg[F, k]


def _highest_rank(D, A, m, msg):
    b = ((D + msg[:, 0]) + msg[:, 1]) + msg[:, 2]
    r = np.array([max((i for i in range(MC) if b[f, i] == b[f].min()), default=0) for f in range(len(m))])
    return np.where(m > 0, A[np.arange(len(m)), r], -1), r


MC = bo.MCAND
MUTATIONS = {
    "jacobi_schedule": ("step", _jacobi),
    "exclusion_by_subtraction": ("excluded", _subtracting),
    "no_normalisation": ("normalise", lambda M, mg: np.where(np.arange(MC)[None, :] < mg[:, None], M, 0.0)),
    "highest_rank_ties": ("decode", _highest_rank),
    "keep_on_equal": ("keep", lambda e, best: e <= best),
    "stop_on_unchanged_labels": ("converged", lambda changed, moved: not moved),
    "no_icm_polish": ("polish", lambda after, kept: kept),
}
SENSITIVE = [("scene", {}), ("island", {}), ("strip", {}), ("scene", dict(maxBpSweeps=1)),
             ("scene", dict(lam=5.0)), ("equal_q", {})]


def _outputs(r):
    return [np.asarray(r[k]).tobytes() for k in ("ret", "stats", "info", "labels", "faceChart", "charts", "uv",
                                                 "atlas")]


def _sensitive_case(name):
    if name == "equal_q":
        if name not in _memo:
            _memo[name] = pc.CASES[name]()
        return _memo[name]
    return _case(name)


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_every_mutation_is_seen(mutation, monkeypatch):
    name, fn = MUTATIONS[mutation]
    changed = []
    for key, over in SENSITIVE:
        c = _sensitive_case(key)
        ref = _outputs(_run(c, **over))
        with monkeypatch.context() as m:
            m.setattr(bo, name, fn)
            out = _outputs(_run(c, **over))
        if out != ref:
            changed.append((key, over))
            break
    print("%s: changes %s" % (mutation, changed))
    assert changed, mutation


# ---- (f) argument checks, header, SASS ------------------------------------------------------------------------------
def _call(sweeps=32, T=4, lam=0.5, dataTerm=1, **kw):
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    charts = np.zeros((4, 8), np.int32)
    return cs.lib().cs_texture_mesh_bp(IMG, 2, p(KS), p(RS), p(TS), kw.get("verts", 0x1000), 4, 0x2000, T, dataTerm,
                                       3.0, 4.0, sweeps, lam, 75.0, 0.01, 2, 1024, 100, 0x400000, 4,
                                       kw.get("uv", 0x10000), 0x20000, None, p(charts), 4, None, None, None)


def _rejects(r, *words):
    msg = cs.lib().cs_last_error().decode()
    assert r == CS_E_ARG, (r, msg)
    assert msg.startswith("cs_texture_mesh_bp: invalid argument (CS_E_ARG)"), msg
    for w in words:
        assert w in msg, (w, msg)


def test_argument_checks():
    for s in (-1, 1001, -(1 << 31)):
        _rejects(_call(sweeps=s), "maxBpSweeps")
    _rejects(_call(dataTerm=2), "dataTerm")
    _rejects(_call(lam=-1.0), "lambda")
    _rejects(_call(verts=0x1002), "d_vertices")
    _rejects(_call(T=-1), "numTriangles")
    for s in (0, 1, 1000):
        _rejects(_call(sweeps=s, uv=0x1000), "overlap")


def test_empty_mesh_makes_no_cuda_call():
    stats = np.full(20, -1, np.int64)
    info = np.full(3, -1.0)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    r = cs.lib().cs_texture_mesh_bp(IMG, 2, p(KS), p(RS), p(TS), None, 0, None, 0, 1, 3.0, 4.0, 32, 0.5, 75.0, 0.01,
                                    2, 1024, 100, None, 0, None, None, None, None, 0, p(info), p(stats), None)
    assert r == 0 and (stats == 0).all() and (info == 0).all()


def test_header_declares_the_call():
    hdr = open(os.path.join(os.path.dirname(cs.__file__), "..", "include", "cudasift_b200.h")).read()
    assert "int cs_texture_mesh_bp(" in hdr
    assert "15 + 2 G + rounds + colours x sweeps + (colours + 3) x BP sweeps" in hdr and "196 bytes per face" in hdr
    f = cs.lib().cs_texture_mesh_bp
    assert len(f.argtypes) == 29 and f.argtypes[12] is ctypes.c_int and f.argtypes[13] is ctypes.c_double
    with pytest.raises(ValueError):
        cs.TextureMeshBP([], [], [], [], np.zeros((0, 3)), np.zeros((0, 3)), dataTerm="sharpness")


# sha256 of the normalised `cuobjdump -sass` of the photo call's two kernels in the parent of cs_texture_mesh_bp, from
# nvcc 12.9 (V12.9.86) with the library's flags: the BP stage leaves them as they were.
SASS = {"texture_photo_candidate_kernel": "960498530f7ad9b0b9d8d044935734db7f17eb8784ba29c8c8dcad875056bccb",
        "texture_outlier_kernel": "96cd850b851308d46cd3f44895426a4f038ace2e5b3ed2ddb5f217744b757dc9"}


def test_photo_kernels_are_unchanged():
    nvcc = build.nvcc_path()
    if nvcc is None or "V12.9.86" not in subprocess.run([nvcc, "--version"], stdout=subprocess.PIPE,
                                                        text=True).stdout:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    build.build_library()
    fs = _sass(os.path.join(build.OBJDIR, "texture.o"))
    for name, digest in SASS.items():
        key = [f for f in fs if re.search(r"\d+%sE" % name, f)]
        assert len(key) == 1, (name, sorted(fs))
        assert hashlib.sha256("\n".join(fs[key[0]]).encode()).hexdigest() == digest, name
