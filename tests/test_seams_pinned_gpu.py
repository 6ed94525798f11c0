"""Seam levelling against pinned bytes (tests/golden/seams_pinned.npz, from tests/golden/make_seams_pinned.py): every
stored case's info and stats bit for bit and, for valid input, its levelled atlas (and corner offsets for
cs_level_texture_seams) by sha256 digest, for cs_level_texture_seams and cs_level_texture_seams_local on every valid
case of tests/seam_cases.py and its scale case, the ramp past 2048 x 256 free texels, the vignetted texture scene (flat
and jittered, the local call at stripWidth 1, 7 and 20) and every status."""
import importlib.util
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _generator():
    spec = importlib.util.spec_from_file_location("make_seams_pinned", os.path.join(GOLDEN, "make_seams_pinned.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def pinned():
    with np.load(os.path.join(GOLDEN, "seams_pinned.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("call", ["global", "local"])
def test_seams_match_pinned_bytes(cs, pinned, call):
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
        if "inputs" in want:                      # the scene's inputs come from cs_texture_mesh
            assert got["inputs"].tobytes() == want["inputs"].tobytes(), ("texturing changed the inputs", c)
        for k, v in got.items():
            w = want[k]
            assert v.dtype == w.dtype and v.shape == w.shape and v.tobytes() == w.tobytes(), (c, k, v, w)
        statuses.add(int(want["stats"][7]))
    assert statuses == {0, 1, 2, 3}, statuses
