"""The cooperative solvers against pinned bytes (tests/golden/solvers_pinned.npz, from
tests/golden/make_solvers_pinned.py): every stored case's outputs by sha256 digest, its costs and statistics, bit for
bit.  The cases run every instantiation of bundle adjustment's kernel (camera block 6 or 9, trivial or robust loss)
with per-member errors and inlier bytes, rotation averaging under the squared loss and Geman-McClure, and global
positioning under the trivial loss and Cauchy, each on a small and a larger scene."""
import importlib.util
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _generator():
    spec = importlib.util.spec_from_file_location("make_solvers_pinned", os.path.join(GOLDEN, "make_solvers_pinned.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def pinned():
    with np.load(os.path.join(GOLDEN, "solvers_pinned.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("solver", ["bundle", "rotavg", "globalpos"])
def test_solver_matches_pinned_bytes(cs, pinned, solver):
    gen = _generator()
    cases = json.loads(str(pinned["cases"]))
    assert cases == gen.cases()
    ran = 0
    for i, c in enumerate(cases):
        if c["solver"] != solver:
            continue
        want = {k[len("c%d_" % i):]: v for k, v in pinned.items() if k.startswith("c%d_" % i)}
        got = gen.run(cs, c)
        assert set(got) == set(want), (c, sorted(got), sorted(want))
        for k, v in got.items():
            assert np.array_equal(v, want[k]), (c, k, v, want[k])
        ran += 1
    assert ran >= 4
