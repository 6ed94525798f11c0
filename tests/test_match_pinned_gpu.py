"""The tensor-core matcher against pinned bytes (tests/golden/match_pinned.npz, from tests/golden/make_match_pinned.py):
every stored case's outputs and statistics, bit for bit.  The cases run MatchSiftData, mutual, two-nearest-neighbour,
ratio (with and without the cross-check) and batched ratio matching in mode 2, on sizes that are not multiples of 32 or
128, fewer than 32 candidates, 100 rows against 60 000 candidates, rows that fall back to the exact scan and the
bad-input gate."""
import importlib.util
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _generator():
    spec = importlib.util.spec_from_file_location("make_match_pinned", os.path.join(GOLDEN, "make_match_pinned.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def pinned():
    with np.load(os.path.join(GOLDEN, "match_pinned.npz")) as z:
        return {k: z[k] for k in z.files}


def test_tensor_matcher_matches_pinned_bytes(cs, pinned):
    gen = _generator()
    cases = json.loads(str(pinned["cases"]))
    assert {c["kind"] for c in cases} == {"match", "mutual", "knn", "ratio", "batch"}
    for i, c in enumerate(cases):
        got = gen.run(cs, c)
        want = {k[len("c%d_" % i):]: v for k, v in pinned.items() if k.startswith("c%d_" % i)}
        assert set(got) == set(want), (c["kind"], c["name"])
        for k, v in got.items():
            assert np.array_equal(v, want[k]), (c["kind"], c["name"], c.get("cross"), k, v, want[k])
