"""Poisson meshing against pinned bytes (tests/golden/mesh_pinned.npz, from tests/golden/make_mesh_pinned.py): every
stored case's vertices, triangles, vertex intensities and chi by sha256 digest, and its info and stats, bit for bit,
for cs_poisson_mesh and cs_poisson_mesh_screened on the sphere, the torus and the open sheet at depths 5 to 8, with
intensities, trimming, point weights 1, 4 and 16, and every status."""
import importlib.util
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _generator():
    spec = importlib.util.spec_from_file_location("make_mesh_pinned", os.path.join(GOLDEN, "make_mesh_pinned.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def pinned():
    with np.load(os.path.join(GOLDEN, "mesh_pinned.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("call", ["dirichlet", "screened"])
def test_mesh_matches_pinned_bytes(cs, pinned, call):
    gen = _generator()
    cases = json.loads(str(pinned["cases"]))
    assert cases == gen.cases()
    statuses = set()
    for i, c in enumerate(cases):
        if c["call"] != call:
            continue
        want = {k[len("c%d_" % i):]: v for k, v in pinned.items() if k.startswith("c%d_" % i)}
        got = gen.run(cs, c)
        assert set(got) == set(want), (c, sorted(got), sorted(want))
        for k, v in got.items():
            w = want[k]
            assert v.dtype == w.dtype and v.shape == w.shape and v.tobytes() == w.tobytes(), (c, k, v, w)
        statuses.add(int(want["stats"][9]))
    # the Dirichlet call reaches every status; the screened call has no status 2
    assert statuses == ({0, 1, 2, 3} if call == "dirichlet" else {0, 1, 3}), statuses
