"""CPU checks of ranked batch extraction: the entry points exist, cs_extractor_create_ranked and cs_rank_records
reject bad arguments before any CUDA call, and the Python wrapper passes its arguments through unchanged."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("cs_extractor_create_ranked", "cs_extractor_candidates", "cs_rank_records")
CS_E_ARG = -2
MAX_CANDIDATES = 1 << 18


def test_symbols_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for name in NEW:
        assert name in declared and name in exported, name
        assert hasattr(cs.lib(), name)
    assert build.SOURCES.count("rank.cu") == 1


def _create(w=640, h=480, octaves=5, maxPts=100, up=0, batch=1, maxCand=1000):
    return cs.lib().cs_extractor_create_ranked(w, h, octaves, maxPts, up, batch, maxCand)


@pytest.mark.parametrize("maxPts,maxCand", [(0, 1000), (-5, 1000), (101, 100), (1, 0), (1000, MAX_CANDIDATES + 1),
                                            (1, 1 << 30)])
def test_create_ranked_rejects_bad_capacities(maxPts, maxCand):
    """Invalid capacities fail with CS_E_ARG whether or not a device is present: the check precedes any CUDA call."""
    assert _create(maxPts=maxPts, maxCand=maxCand) is None
    msg = cs.lib().cs_last_error().decode()
    assert "invalid argument" in msg and "CS_E_ARG" in msg, msg


def test_create_ranked_accepts_the_limits():
    """Valid capacities pass the argument check: without a device the failure is a CUDA one, with a device it works."""
    for maxPts, maxCand in ((1, 1), (100, 100), (1, MAX_CANDIDATES)):
        cs.lib().cs_set_tuning(b"no such key", 0)    # leaves a known message in cs_last_error
        h = _create(w=64, h=48, maxPts=maxPts, maxCand=maxCand)
        if h:
            cs.lib().cs_extractor_destroy(h)
        else:
            assert "invalid argument" not in cs.lib().cs_last_error().decode()


def test_create_ranked_rejects_legacy_pipeline():
    cs.set_tuning("legacy", 1)
    try:
        assert _create() is None
        msg = cs.lib().cs_last_error().decode()
        assert "CS_E_ARG" in msg and "legacy" in msg, msg
    finally:
        cs.set_tuning("legacy", 0)


def test_rank_records_rejects_bad_arguments():
    L = cs.lib()
    buf = np.zeros(2 * 576 + 16, np.uint8)
    base = buf.ctypes.data
    a16 = base + (-base) % 16                     # 16-byte aligned host addresses: rejected before they are used
    assert L.cs_rank_records(a16, -1, a16, 10) == CS_E_ARG
    assert L.cs_rank_records(a16, 1, a16, 0) == CS_E_ARG
    assert L.cs_rank_records(a16, MAX_CANDIDATES + 1, a16, 10) == CS_E_ARG
    assert L.cs_rank_records(a16 + 4, 1, a16, 10) == CS_E_ARG
    assert L.cs_rank_records(a16, 1, a16 + 8, 10) == CS_E_ARG
    assert L.cs_rank_records(None, 1, a16, 10) == CS_E_ARG
    assert L.cs_rank_records(None, 0, None, 10) == 0   # nothing to rank
    with pytest.raises(ValueError):
        cs.rank_records(np.zeros(3, cs.SIFT_DTYPE), 0)
    assert len(cs.rank_records(np.zeros(0, cs.SIFT_DTYPE), 5)) == 0


class _FakeLib:
    """Records the calls the wrapper makes instead of reaching the library."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            return {"cs_extractor_create_batch": 1111, "cs_extractor_create_ranked": 2222,
                    "cs_extractor_candidates": 77}.get(name, 0)
        return f


def test_python_wrapper_maps_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    plain = cs.Extractor(1920, 1080, 5, 512, False, batch=4)
    assert plain.handle == 1111 and fake.calls[-1] == ("cs_extractor_create_batch", (1920, 1080, 5, 512, 0, 4))
    ranked = cs.Extractor(1280, 960, 4, 1000, True, batch=16, maxCandidates=32768)
    assert ranked.handle == 2222
    assert fake.calls[-1] == ("cs_extractor_create_ranked", (1280, 960, 4, 1000, 1, 16, 32768))
    assert ranked.maxPts == 1000 and ranked.maxCandidates == 32768
    assert ranked.candidates(3) == 77 and fake.calls[-1] == ("cs_extractor_candidates", (2222, 3))
    fake.calls.clear()
    plain.close(); ranked.close()
    assert [c[0] for c in fake.calls] == ["cs_extractor_destroy"] * 2


def test_python_wrapper_raises_on_rejection():
    with pytest.raises(cs.CudaSiftError, match="invalid argument"):
        cs.Extractor(640, 480, 5, 1000, False, batch=2, maxCandidates=999)
