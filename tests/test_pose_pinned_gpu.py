"""Absolute pose against pinned bytes (tests/golden/pose_pinned.npz, from tests/golden/make_pose_pinned.py): every
stored case's poses, counts, statistics and per-feature output digests, and the models entry point's slot digest and
slot counts, bit for bit.  The cases cover single jobs from 30 to 5 000 correspondences, one mixed batch (empty jobs,
invalid pointOf entries, NaN points and positions, too few correspondences) with and without per-feature outputs, and
both branches of the refinement's keep rule (refinement kept and dropped)."""
import importlib.util
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _generator():
    spec = importlib.util.spec_from_file_location("make_pose_pinned", os.path.join(GOLDEN, "make_pose_pinned.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def pinned():
    with np.load(os.path.join(GOLDEN, "pose_pinned.npz")) as z:
        return {k: z[k] for k in z.files}


def _stored(pinned, prefix):
    return {k[len(prefix):]: v for k, v in pinned.items() if k.startswith(prefix)}


def _same(got, want, where):
    assert set(got) == set(want), (where, sorted(got), sorted(want))
    for k, v in got.items():
        assert np.array_equal(v, want[k]), (where, k, v, want[k])


def test_batch_calls_match_pinned_bytes(cs, pinned):
    gen = _generator()
    cases = json.loads(str(pinned["cases"]))
    assert len(cases) >= 9 and json.loads(str(pinned["kept_branches"])) == [0, 1]
    for i, c in enumerate(cases):
        _same(gen.run(cs, c), _stored(pinned, "c%d_" % i), c)


def test_models_entry_point_matches_pinned_bytes(cs, pinned):
    gen = _generator()
    for i, c in enumerate(json.loads(str(pinned["models_cases"]))):
        _same(gen.run_models(cs, c), _stored(pinned, "m%d_" % i), c)
