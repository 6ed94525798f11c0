"""CPU checks of mutual matching: the entry points exist, cs_match_mutual and cs_match_mutual_host reject bad
arguments before any CUDA call, and the Python wrappers pass their arguments through unchanged."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import cudasift_b200 as cs
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("cs_match_mutual", "cs_match_mutual_host")
CS_E_ARG = -2
REC = 576


def test_symbols_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for name in NEW:
        assert name in declared and name in exported, name
        assert hasattr(cs.lib(), name)
    assert "MatchSiftDataMutual" in cs.__all__ and "match_mutual_host" in cs.__all__
    assert build.SOURCES.count("match_mutual.cu") == 1


def _bad_calls(base):
    """(description, args without ms) of every invalid call; base is a 16-byte aligned address with room for two
    sets of 4 records and 8 pairs.  The pointers are never dereferenced: the checks come first."""
    s1, s2, pairs = base, base + 4 * REC, base + 8 * REC
    return [
        ("n1 < 0", (s1, -1, s2, 4, 0.0, 1.0, pairs, 4, 0)),
        ("n2 < 0", (s1, 4, s2, -3, 0.0, 1.0, pairs, 4, 0)),
        ("NULL set 1", (None, 4, s2, 4, 0.0, 1.0, pairs, 4, 0)),
        ("NULL set 2", (s1, 4, None, 4, 0.0, 1.0, pairs, 4, 0)),
        ("maxPairs < 0", (s1, 4, s2, 4, 0.0, 1.0, pairs, -1, 0)),
        ("NULL pairs", (s1, 4, s2, 4, 0.0, 1.0, None, 4, 0)),
        ("mode -1", (s1, 4, s2, 4, 0.0, 1.0, pairs, 4, -1)),
        ("mode 3", (s1, 4, s2, 4, 0.0, 1.0, pairs, 4, 3)),
        ("same set twice", (s1, 4, s1, 4, 0.0, 1.0, pairs, 4, 0)),
        ("set 2 starts inside set 1", (s1, 4, s1 + 3 * REC, 4, 0.0, 1.0, pairs, 4, 0)),
        ("set 1 starts inside set 2", (s2 + REC, 2, s2, 2, 0.0, 1.0, pairs, 4, 0)),
        ("pairs unaligned", (s1, 4, s2, 4, 0.0, 1.0, pairs + 4, 4, 0)),
        ("pairs inside set 1", (s1, 4, s2, 4, 0.0, 1.0, s1 + 8, 4, 0)),
        ("pairs run into set 2", (s1, 4, s2, 4, 0.0, 1.0, s2 - 8, 4, 0)),
    ]


@pytest.mark.parametrize("entry", NEW)
def test_invalid_arguments_return_cs_e_arg(entry):
    """Every invalid argument fails with CS_E_ARG whether or not a device is present."""
    buf = np.zeros(8 * REC + 8 * 8 + 16, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    f = getattr(cs.lib(), entry)
    for what, args in _bad_calls(base):
        ms = ctypes.c_double(-1.0)
        assert f(*args, ctypes.byref(ms)) == CS_E_ARG, (entry, what)
        msg = cs.lib().cs_last_error().decode()
        assert "invalid argument" in msg and "CS_E_ARG" in msg, (entry, what, msg)
        assert ms.value == 0.0, (entry, what)
    if entry == "cs_match_mutual":        # the device pairs buffer is written as int2
        assert f(base, 4, base + 4 * REC, 4, 0.0, 1.0, base + 8 * REC + 4, 4, 0, None) == CS_E_ARG


@pytest.mark.parametrize("entry", NEW)
def test_empty_sets_write_nothing(entry):
    """n1 == 0 or n2 == 0 returns 0 before any CUDA call (matching.cu:1095-1096); adjacent sets do not overlap, and
    an empty set may be NULL, as may the pairs buffer when maxPairs is 0."""
    buf = np.zeros(8 * REC + 16, np.uint8)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    f = getattr(cs.lib(), entry)
    assert f(base, 0, base + 4 * REC, 4, 0.0, 1.0, None, 0, 0, None) == 0
    assert f(base, 4, None, 0, 0.0, 1.0, None, 0, 1, None) == 0
    assert f(None, 0, None, 0, 0.0, 1.0, None, 0, 2, None) == 0
    assert not buf.any()


class _FakeLib:
    """Records the calls the wrappers make instead of reaching the library."""

    def __init__(self, pairs=3):
        self.calls = []
        self.pairs = pairs

    def __getattr__(self, name):
        def f(*args):
            self.calls.append((name, args))
            if name == "cs_device_alloc":
                return 4096
            if name in NEW:
                return self.pairs
            return 0
        return f


def test_device_wrapper_maps_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    d1, d2 = cs.SiftData(), cs.SiftData()
    d1._buf, d2._buf = cs.DeviceBuffer(64), cs.DeviceBuffer(64)
    d1.numPts, d2.numPts = 7, 5
    pairs, ms = cs.MatchSiftDataMutual(d1, d2, minScore=0.85, maxAmbiguity=0.95, mode=2)
    call = [c for c in fake.calls if c[0] == "cs_match_mutual"]
    assert len(call) == 1
    a = call[0][1]
    assert a[0] == d1.d_data and a[1] == 7 and a[2] == d2.d_data and a[3] == 5
    assert a[4] == pytest.approx(0.85) and a[5] == pytest.approx(0.95)
    assert a[6] == 4096 and a[7] == 5 and a[8] == 2          # room for min(n1, n2) pairs
    assert pairs.shape == (3, 2) and pairs.dtype == np.int32
    fake.calls.clear()
    cs.MatchSiftDataMutual(d1, d2)
    a = [c for c in fake.calls if c[0] == "cs_match_mutual"][0][1]
    assert a[4] == 0.0 and a[5] == float("inf") and a[8] == 0
    d1._buf = d2._buf = None


def test_host_wrapper_maps_arguments(monkeypatch):
    fake = _FakeLib(pairs=2)
    monkeypatch.setattr(cs, "lib", lambda: fake)
    s1, s2 = np.zeros(9, cs.SIFT_DTYPE), np.zeros(4, cs.SIFT_DTYPE)
    o1, o2, pairs, ms = cs.match_mutual_host(s1, s2, minScore=0.5, maxAmbiguity=0.8, mode=1)
    (name, a), = fake.calls
    assert name == "cs_match_mutual_host"
    assert a[1] == 9 and a[3] == 4 and a[4] == pytest.approx(0.5) and a[5] == pytest.approx(0.8)
    assert a[7] == 4 and a[8] == 1
    assert o1 is not s1 and o2 is not s2 and len(o1) == 9 and len(o2) == 4
    assert pairs.shape == (2, 2) and pairs.dtype == np.int32


def test_python_wrapper_raises_on_rejection():
    with pytest.raises(cs.CudaSiftError, match="invalid argument"):
        cs.match_mutual_host(np.zeros(3, cs.SIFT_DTYPE), np.zeros(3, cs.SIFT_DTYPE), mode=5)
