"""Guided matching against pinned bytes (tests/golden/guided_pinned.npz, from tests/golden/make_guided_pinned.py): every
stored case's cs_match_knn2_guided lists, cs_match_guided pairs (with and without the cross-check) and
cs_match_guided_stats, bit for bit.  The cases run F and H at 1, 4 and 16 px on planted 1 000 x 1 200 and
5 000 x 5 000 views, rows that scan every candidate (positions beyond 1e12 px, |pw| < 1e-12, a threshold of 1e5 px),
non-finite positions and models that admit nothing."""
import importlib.util
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _generator():
    spec = importlib.util.spec_from_file_location("make_guided_pinned", os.path.join(GOLDEN, "make_guided_pinned.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def pinned():
    with np.load(os.path.join(GOLDEN, "guided_pinned.npz")) as z:
        return {k: z[k] for k in z.files}


def test_guided_matcher_matches_pinned_bytes(cs, pinned):
    gen = _generator()
    cases = json.loads(str(pinned["cases"]))
    assert {c["kind"] for c in cases} == {"knn", "guided"} and len(cases) == 63
    for i, c in enumerate(cases):
        got = gen.run(cs, c)
        want = {k[len("c%d_" % i):]: v for k, v in pinned.items() if k.startswith("c%d_" % i)}
        assert set(got) == set(want), (c["kind"], c["name"])
        for k, v in got.items():
            assert np.array_equal(v, want[k]), (c["kind"], c["name"], c["model"], c["t"], c.get("cross"), k, v, want[k])
