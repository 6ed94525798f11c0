"""CPU checks of feature tracks (cs_build_tracks): the entry point is declared, exported and typed, every invalid
argument is rejected with the offending list or image named before any CUDA call, calls without pairs return 0
without a device, the numpy statement (tracks_oracle) agrees with scipy's connected components and states the
header's rules on small hand-made cases, and the Python wrapper builds its tables and sizes its buffers."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.csgraph

import cudasift_b200 as cs
import tracks_oracle as to
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_E_ARG = -2


def test_symbol_declared_exported_and_typed():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE, text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert "cs_build_tracks" in declared and "cs_build_tracks" in exported
    assert "typedef struct cs_track_list" in header
    f = cs.lib().cs_build_tracks
    assert f.restype is ctypes.c_int and len(f.argtypes) == 13
    assert ctypes.sizeof(cs.TrackList) == 24
    assert [n for n, _ in cs.TrackList._fields_] == ["image1", "image2", "pairs", "numPairs"]
    assert "BuildTracks" in cs.__all__ and "TrackList" in cs.__all__ and callable(cs.BuildTracks)


class Arena:
    """Host memory laid out as on the device: three pair lists of 4 pairs, then d_trackOf (16 ints), d_offsets (5
    ints) and d_members (8 pairs), 8-byte aligned.  Nothing is dereferenced: every case fails its checks."""

    def __init__(self):
        self.buf = np.zeros(3 * 32 + 64 + 32 + 64 + 64, np.uint8)
        base = self.buf.ctypes.data + (-self.buf.ctypes.data) % 16
        self.pairs = [base + 32 * k for k in range(3)]
        self.trackOf = base + 96
        self.offsets = base + 96 + 64
        self.members = base + 96 + 64 + 32

    def lists(self):
        return [dict(image1=0, image2=1, pairs=self.pairs[0], numPairs=4),
                dict(image1=1, image2=1, pairs=self.pairs[1], numPairs=4),
                dict(image1=2, image2=0, pairs=self.pairs[2], numPairs=4)]

    def common(self):
        return dict(sizes=[6, 5, 5], minLength=2, trackOf=self.trackOf, offsets=self.offsets, maxTracks=4,
                    members=self.members, maxMembers=8)


def _call(lists, common):
    sizes = np.array(common["sizes"], np.int32)
    lt = (cs.TrackList * max(len(lists), 1))(*[cs.TrackList(x["image1"], x["image2"], x["pairs"], x["numPairs"])
                                               for x in lists])
    stats = np.full(8, 7, np.int64)
    ms = ctypes.c_double(-1.0)
    r = cs.lib().cs_build_tracks(sizes.ctypes.data if common.get("sizesPtr", 1) else None,
                                 common.get("numImages", len(sizes)), lt if common.get("listsPtr", 1) else None,
                                 common.get("numLists", len(lists)), common["minLength"], 1, common["trackOf"],
                                 common["offsets"], common["maxTracks"], common["members"], common["maxMembers"],
                                 stats.ctypes.data, ctypes.byref(ms))
    return r, ms.value, stats


def _expect(r, ms, stats, what, name):
    assert r == CS_E_ARG, (what, r)
    msg = cs.lib().cs_last_error().decode()
    assert "invalid argument" in msg and "CS_E_ARG" in msg, (what, msg)
    if name:
        assert name in msg, (what, msg)
    assert ms == 0.0 and (stats == 7).all(), what


def test_rejects_every_invalid_argument():
    a = Arena()
    big = 1 << 30
    cases = [
        ("numImages < 0", {}, dict(numImages=-1), "numImages"),
        ("numImages 2^24 + 1", {}, dict(numImages=(1 << 24) + 1), "numImages"),
        ("numLists < 0", {}, dict(numLists=-1), "numLists"),
        ("numLists 2^24 + 1", {}, dict(numLists=(1 << 24) + 1), "numLists"),
        ("NULL imageSizes", {}, dict(sizesPtr=0), "imageSizes"),
        ("NULL lists", {}, dict(listsPtr=0), "lists"),
        ("negative size", {}, dict(sizes=[6, -1, 5]), "imageSizes[1]"),
        ("N above INT_MAX", {}, dict(sizes=[big, big, 5]), "imageSizes[1]"),
        ("image1 out of range", {1: dict(image1=3)}, {}, "lists[1]"),
        ("image2 negative", {2: dict(image2=-1)}, {}, "lists[2]"),
        ("numPairs < 0", {0: dict(numPairs=-1)}, {}, "lists[0]"),
        ("NULL pairs", {2: dict(pairs=None)}, {}, "lists[2]"),
        ("pairs unaligned", {1: dict(pairs=a.pairs[1] + 4)}, {}, "lists[1]"),
        ("pair total above INT_MAX", {1: dict(numPairs=big), 2: dict(numPairs=big)}, {}, "lists[2]"),
        ("minLength 1", {}, dict(minLength=1), "minLength"),
        ("maxTracks < 0", {}, dict(maxTracks=-1), "maxTracks"),
        ("maxMembers < 0", {}, dict(maxMembers=-1), "maxMembers"),
        ("NULL offsets", {}, dict(offsets=None), "d_offsets"),
        ("NULL members", {}, dict(members=None), "d_members"),
        ("trackOf unaligned", {}, dict(trackOf=a.trackOf + 2), "d_trackOf"),
        ("members unaligned", {}, dict(members=a.members + 4), "d_members"),
        ("members over a list", {}, dict(members=a.pairs[1] + 8, maxMembers=2), "d_members and lists[1].pairs"),
        ("trackOf over a list", {}, dict(trackOf=a.pairs[2]), "d_trackOf and lists[2].pairs"),
        ("offsets over members", {}, dict(offsets=a.members + 24), "d_offsets and d_members"),
        ("offsets' last entry over members", {}, dict(offsets=a.members - 16), "d_offsets and d_members"),
        ("trackOf over offsets", {}, dict(trackOf=a.offsets - 8), "d_trackOf and d_offsets"),
    ]
    for what, lch, cch, name in cases:
        lists, common = a.lists(), a.common()
        for k, f in lch.items():
            lists[k].update(f)
        common.update(cch)
        _expect(*_call(lists, common), what, name)
    assert not a.buf.any()
    # touching ranges and lists over each other (read only) pass the checks; every list empty: no device needed
    lists, common = a.lists(), a.common()
    for x in lists:
        x["numPairs"] = 0
    common.update(trackOf=None, offsets=None, maxTracks=0, members=a.pairs[0], maxMembers=12)
    r, ms, stats = _call(lists, common)
    assert r == 0 and ms == 0.0 and not stats.any()


def test_no_pairs_returns_zero_before_any_cuda_call():
    ms = ctypes.c_double(-1.0)
    stats = np.full(8, 7, np.int64)
    L = cs.lib()
    assert L.cs_build_tracks(None, 0, None, 0, 2, 1, None, None, 0, None, 0, stats.ctypes.data, ctypes.byref(ms)) == 0
    assert ms.value == 0.0 and not stats.any()
    sizes = np.array([3, 0, 4], np.int32)
    lt = (cs.TrackList * 2)(cs.TrackList(0, 2, None, 0), cs.TrackList(1, 1, None, 0))
    stats[:] = 7
    assert L.cs_build_tracks(sizes.ctypes.data, 3, lt, 2, 3, 0, None, None, 0, None, 0, stats.ctypes.data, None) == 0
    assert not stats.any()
    assert L.cs_build_tracks(sizes.ctypes.data, 3, lt, 0, 2, 1, None, None, 0, None, 0, None, None) == 0
    # image indices are checked on empty lists as well
    lt[1] = cs.TrackList(1, 3, None, 0)
    _expect(*_call([dict(image1=0, image2=2, pairs=None, numPairs=0), dict(image1=1, image2=3, pairs=None,
                                                                             numPairs=0)],
                   dict(sizes=[3, 0, 4], minLength=2, trackOf=None, offsets=None, maxTracks=0, members=None,
                        maxMembers=0)), "image2 out of range", "lists[1]")


@pytest.mark.parametrize("seed", range(6))
def test_oracle_components_equal_scipy(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 3000))
    m = int(rng.integers(0, 3 * n))
    u, v = rng.integers(0, n, m), rng.integers(0, n, m)
    label = to.components(n, u, v)
    k, lab = scipy.sparse.csgraph.connected_components(
        scipy.sparse.coo_matrix((np.ones(m), (u, v)), shape=(n, n)), directed=False)
    # the same partition, each labelled by its smallest id
    assert len(np.unique(label)) == k
    first = np.full(k, n)
    np.minimum.at(first, lab, np.arange(n))
    assert np.array_equal(label, first[lab])


def test_oracle_components_path_descending():
    n = 1 << 16
    k = np.arange(n - 2, -1, -1)
    assert (to.components(n, k, k + 1) == 0).all()


def test_oracle_states_the_rules():
    """Images of 3, 0, 4, 1 and 2 features (global ids 0-2, 3-6, 7, 8-9)."""
    sizes = [3, 0, 4, 1, 2]
    lists = [(0, 2, [[0, 1], [2, 3], [3, 0], [-1, 0], [0, 1]]),     # two invalid pairs and a repeated one
             (2, 4, [[1, 1], [3, 0]]),
             (3, 0, [[0, 2]]),
             (2, 2, [[0, 2]]),                                      # joins two features of image 2: a conflict
             (4, 4, [[0, 0]])]                                      # a feature joined with itself
    T, off, mem, tof, st = to.build_tracks(sizes, lists, 2, True)
    # components, by global id: {0, 4, 9}, {2, 6, 7, 8} and {3, 5}, the last with two features of image 2
    assert list(st) == [8, 2, 9, 3, 1, 0, 2, 7]
    assert T == 2 and list(off) == [0, 3, 7]
    assert mem.tolist() == [[0, 0], [2, 1], [4, 1], [0, 2], [2, 3], [3, 0], [4, 0]]
    assert tof.tolist() == [0, -1, 1, -1, 0, -1, 1, 1, 1, 0]
    T, off, mem, tof, st = to.build_tracks(sizes, lists, 2, False)
    assert T == 3 and list(off) == [0, 3, 7, 9] and mem[7:].tolist() == [[2, 0], [2, 2]] and tof[3] == 2
    T, off, mem, tof, st = to.build_tracks(sizes, lists, 4, False, maxTracks=0, maxMembers=3)
    assert T == 1 and list(off) == [0] and len(mem) == 3 and list(st[4:]) == [0, 2, 1, 4]


class _FakeLib:
    def __init__(self, T=2, M=5):
        self.calls, self.T, self.M, self.uploads = [], T, M, {}

    def __getattr__(self, name):
        def f(*args):
            if name == "cs_build_tracks":
                S, nl = args[1], args[3]
                sizes = list((ctypes.c_int * S).from_address(args[0].value)) if S else []
                lists = [cs.TrackList.from_address(args[2] + k * ctypes.sizeof(cs.TrackList)) for k in range(nl)]
                stats = (ctypes.c_longlong * 8).from_address(args[11].value)
                stats[6], stats[7] = self.T, self.M
                self.calls.append((name, args, sizes, [(x.image1, x.image2, x.pairs, x.numPairs) for x in lists]))
                return self.T
            self.calls.append((name, args, None, None))
            if name == "cs_device_alloc":
                return 4096 * (1 + len(self.calls))
            if name == "cs_memcpy_h2d":
                self.uploads[args[0]] = ctypes.string_at(args[1].value, args[2])
            return 0
        return f


def test_wrapper_maps_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    p0 = np.array([[0, 1], [2, 3]], np.int32)
    p2 = np.array([[4, 0], [1, 1], [0, 0]], np.int64)                  # converted to int32
    lists = [(0, 1, p0), (1, 2, np.zeros((0, 2), np.int32)), (2, 0, p2)]
    offsets, members, trackOf, stats, ms = cs.BuildTracks([5, 4, 6], lists, minLength=3, dropConflicting=False)
    (name, a, sizes, table), = [c for c in fake.calls if c[0] == "cs_build_tracks"]
    assert sizes == [5, 4, 6] and a[1] == 3 and a[3] == 3 and a[4] == 3 and a[5] == 0
    allocs = [c[1][0] for c in fake.calls if c[0] == "cs_device_alloc"]
    N, P = 15, 5
    maxMembers = min(N, 2 * P)
    assert allocs == [8 * P, 4 * N, 4 * (maxMembers // 3 + 1), 8 * maxMembers]
    assert a[8] == maxMembers // 3 and a[10] == maxMembers
    base = table[0][2]
    assert [t[:2] for t in table] == [(0, 1), (1, 2), (2, 0)] and [t[3] for t in table] == [2, 0, 3]
    assert table[1][2] is None and table[2][2] - base == 16
    assert fake.uploads[base] == np.concatenate([p0, p2.astype(np.int32)]).tobytes()
    assert offsets.shape == (3,) and members.shape == (5, 2) and trackOf.shape == (15,)
    assert offsets.dtype == members.dtype == trackOf.dtype == np.int32 and stats.dtype == np.int64
    fake.calls.clear()
    fake.T, fake.M = 0, 0
    offsets, members, trackOf, stats, _ = cs.BuildTracks([0, 0], [])
    (name, a, sizes, table), = [c for c in fake.calls if c[0] == "cs_build_tracks"]
    assert a[2] is None and a[3] == 0 and a[6] is None and a[8] == 0 and a[9] is None and a[10] == 0
    assert offsets.shape == (1,) and members.shape == (0, 2) and trackOf.shape == (0,)
