"""Verification against pinned bytes (tests/golden/verify_pinned.npz, from tests/golden/make_verify_pinned.py): every
stored case's model, inlier count, inlier list digest and statistics, and the models entry points' slot digests and
normalisation, bit for bit.  The cases cover F and H on general and planar scenes, E on sideways and forward motion,
too few pairs for each model, and both branches of the refit's keep rule (refit kept and dropped) for each model."""
import importlib.util
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _generator():
    spec = importlib.util.spec_from_file_location("make_verify_pinned", os.path.join(GOLDEN, "make_verify_pinned.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def pinned():
    with np.load(os.path.join(GOLDEN, "verify_pinned.npz")) as z:
        return {k: z[k] for k in z.files}


def _same(got, want, where):
    for k, v in got.items():
        assert np.array_equal(v, want[k]), (where, k, v, want[k])


def test_single_calls_match_pinned_bytes(cs, pinned):
    gen = _generator()
    cases = json.loads(str(pinned["cases"]))
    assert len(cases) >= 27
    for i, c in enumerate(cases):
        _same(gen.run(cs, c), {k: pinned["c%d_%s" % (i, k)] for k in ("model", "count", "inliers", "stats")}, c)


def test_models_entry_points_match_pinned_bytes(cs, pinned):
    gen = _generator()
    for i, c in enumerate(json.loads(str(pinned["models_cases"]))):
        _same(gen.run_models(cs, c), {k: pinned["m%d_%s" % (i, k)] for k in ("slots", "counts", "norm", "valid")}, c)
