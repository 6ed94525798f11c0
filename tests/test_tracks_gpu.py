"""GPU checks of feature tracks (cs_build_tracks): every case against the numpy statement (tests/tracks_oracle.py)
byte for byte -- offsets, members, trackOf and the eight statistics -- on random collections with jagged, empty and
1-feature images, self-paired images and invalid pairs, minLength 2, 3 and above the largest component, and
dropConflicting on and off; a 2^22-feature path given in descending order, a star of one feature against 10^5, a
complete graph over 32 images and about 5 * 10^7 pairs; truncation with a sentinel past each limit; invariance under
permuted lists and pairs, swapped roles and duplicated lists; repeated calls; the header's launch count; interleaving
with guided, ratio and verify calls; and the collection chain from batched extraction to tracks."""
import ctypes
import itertools

import numpy as np
import pytest

import tracks_oracle as to
from cudasift_b200.synth import synth_image
from test_guided_batch_gpu import _batch as guided_batch
from test_guided_batch_gpu import _mixed, _sift_data
from test_match_batch_gpu import SENTINEL, Sets

pytestmark = pytest.mark.gpu
LAUNCHES = 8


class Lists:
    """Pair lists [(a, b, pairs)] in one device buffer."""

    def __init__(self, cs, lists):
        self.lists = [(int(a), int(b), np.ascontiguousarray(np.asarray(p, np.int32).reshape(-1, 2))) for a, b, p in lists]
        counts = [len(p) for _, _, p in self.lists]
        self.off = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int64)
        self.buf = cs.DeviceBuffer(max(int(self.off[-1]), 1) * 8)
        if self.off[-1]:
            self.buf.upload(np.concatenate([p for _, _, p in self.lists]))
        self.table = (cs.TrackList * max(len(self.lists), 1))(*[
            cs.TrackList(a, b, self.buf.ptr + 8 * int(self.off[q]) if len(p) else None, len(p))
            for q, (a, b, p) in enumerate(self.lists)])

    def free(self):
        self.buf.free()


def run(cs, sizes, L, minLength=2, drop=1, maxTracks=None, maxMembers=None):
    """One call with room for every output (or the given limits) and one sentinel entry past each buffer.  Returns
    (T, offsets, members, trackOf, stats, ms) with the sentinels still attached: offsets [maxTracks + 2], members
    [maxMembers + 1, 2], trackOf [N + 1]."""
    sizes = np.asarray(sizes, np.int32)
    N = int(sizes.sum(dtype=np.int64))
    P = int(L.off[-1])
    mm = min(N, 2 * P) if maxMembers is None else maxMembers
    mt = mm // minLength if maxTracks is None else maxTracks
    bufs = [cs.DeviceBuffer(4 * (N + 1)), cs.DeviceBuffer(4 * (mt + 2)), cs.DeviceBuffer(8 * (mm + 1))]
    try:
        for b in bufs:
            b.upload(np.full(b.nbytes // 4, SENTINEL, np.int32))
        stats, ms = np.full(8, 7, np.int64), ctypes.c_double(0.0)
        T = cs.lib().cs_build_tracks(sizes.ctypes.data, len(sizes), L.table, len(L.lists), minLength, drop,
                                     bufs[0].ptr, bufs[1].ptr, mt, bufs[2].ptr, mm, stats.ctypes.data,
                                     ctypes.byref(ms))
        assert T >= 0, cs.lib().cs_last_error().decode()
        trackOf = bufs[0].download(np.int32, N + 1)
        offsets = bufs[1].download(np.int32, mt + 2)
        members = bufs[2].download(np.int32, 2 * (mm + 1)).reshape(-1, 2)
    finally:
        for b in bufs:
            b.free()
    return T, offsets, members, trackOf, stats, ms.value, mt, mm


def check(cs, sizes, lists, minLength=2, drop=1, maxTracks=None, maxMembers=None, L=None):
    """The call against the oracle, byte for byte, with the sentinels untouched.  Returns the call's outputs."""
    own = L is None
    L = Lists(cs, lists) if own else L
    try:
        T, offsets, members, trackOf, stats, ms, mt, mm = run(cs, sizes, L, minLength, drop, maxTracks, maxMembers)
    finally:
        if own:
            L.free()
    wT, wOff, wMem, wOf, wSt = to.build_tracks(sizes, lists, minLength, bool(drop), mt, mm)
    assert T == wT and stats.tolist() == wSt.tolist(), (T, stats, wSt)
    k, m = len(wOff), len(wMem)
    assert offsets[:k].tobytes() == wOff.tobytes() and (offsets[k:] == SENTINEL).all()
    assert members[:m].tobytes() == wMem.tobytes() and (members[m:] == SENTINEL).all()
    assert trackOf[:-1].tobytes() == wOf.tobytes() and trackOf[-1] == SENTINEL
    assert ms > 0 or int(L.off[-1]) == 0
    return T, offsets[:k], members[:m], trackOf[:-1], stats


def collection(seed, numImages=40, numLists=120, tracks=400):
    """Jagged images (an empty one and a 1-feature one among them), pair lists between random images and images paired
    with themselves, planted multi-view tracks, random pairs that make conflicts, and invalid pairs (out of range and
    negative)."""
    rng = np.random.default_rng(seed)
    sizes = rng.integers(20, 400, numImages)
    sizes[3], sizes[7] = 0, 1
    # planted tracks: each a feature in each of 2..8 distinct images
    views = {}
    for t in range(tracks):
        imgs = rng.choice(np.flatnonzero(sizes > 0), int(rng.integers(2, 9)), replace=False)
        feats = [int(rng.integers(0, sizes[a])) for a in imgs]
        for (a, f), (b, g) in itertools.combinations(zip(imgs, feats), 2):
            views.setdefault((int(a), int(b)), []).append((f, g))
    lists = [(a, b, p) for (a, b), p in views.items()]
    for _ in range(numLists):
        a, b = (int(x) for x in rng.integers(0, numImages, 2))
        if rng.random() < 0.15:
            b = a
        k = int(rng.integers(0, 24))
        p = np.stack([rng.integers(0, max(sizes[a], 1), k), rng.integers(0, max(sizes[b], 1), k)], 1)
        if k:
            p[rng.integers(0, k)] = (int(sizes[a]), 0)                     # out of range
            p[rng.integers(0, k)] = (0, -1 - int(rng.integers(0, 5)))     # negative
        lists.append((a, b, p))
    lists.append((3, 7, [[0, 0], [1, 0]]))                                # the empty image: both invalid
    lists.append((7, 7, [[0, 0]]))                                        # a feature joined with itself
    perm = rng.permutation(len(lists))
    return sizes, [lists[q] for q in perm]


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("minLength", [2, 3, 10 ** 6])
@pytest.mark.parametrize("drop", [0, 1])
def test_random_collections(cs, seed, minLength, drop):
    sizes, lists = collection(seed)
    T, _, _, _, stats = check(cs, sizes, lists, minLength, drop)
    assert stats[1] > 50 and stats[3] > 100
    if minLength < 10 ** 6:
        assert T > 50 and stats[4] > 0
    else:
        assert T == 0 and stats[4] == 0 and stats[5] == stats[3]


def test_path_descending(cs):
    """The path 0 - 1 - ... - 2^22 - 1 in one image paired with itself, pairs in descending order: the deepest hooks.
    With dropConflicting it is one conflicting component and no track."""
    n = 1 << 22
    k = np.arange(n - 2, -1, -1, dtype=np.int32)
    lists = [(0, 0, np.stack([k + 1, k], 1))]
    L = Lists(cs, lists)
    try:
        T, off, mem, tof, st = check(cs, [n], lists, 2, 0, L=L)
        assert T == 1 and list(off) == [0, n] and (tof == 0).all()
        T, off, _, tof, st = check(cs, [n], lists, 2, 1, L=L)
        assert T == 0 and list(off) == [0] and st.tolist() == [n - 1, 0, n, 1, 1, 0, 0, 0] and (tof == -1).all()
    finally:
        L.free()


def test_path_across_images(cs):
    """The same depth across 64 images of 2^16 features, feature f of image a against feature f of image a + 1, given
    from the last image down: 2^16 tracks of 64 views."""
    n, m = 1 << 16, 64
    f = np.arange(n, dtype=np.int32)
    lists = [(a + 1, a, np.stack([f[::-1], f[::-1]], 1)) for a in range(m - 2, -1, -1)]
    T, off, mem, _, _ = check(cs, [n] * m, lists)
    assert T == n and (np.diff(off) == m).all() and mem[:m].tolist() == [[a, 0] for a in range(m)]


def test_star(cs):
    """One feature against 10^5 others: every hook lands on the same root.  The component holds 10^5 features of
    image 1, so it conflicts: one track without dropConflicting, none with it."""
    n = 100000
    lists = [(1, 0, np.stack([np.arange(n), np.zeros(n, int)], 1))]
    T, off, mem, _, st = check(cs, [1, n], lists, 2, 0)
    assert T == 1 and list(off) == [0, n + 1] and st[3] == 1 and st[4] == 1
    T, off, _, _, st = check(cs, [1, n], lists, 2, 1)
    assert T == 0 and list(off) == [0] and st[4] == 1
    T, _, _, _, st = check(cs, [1, n, 5], lists + [(1, 2, [[0, 0]]), (2, 2, [[1, 3]])], 3, 1)
    assert T == 0 and st[4] == 1 and st[5] == 1                           # image 1 twice in the star; one short pair


def test_complete_graph_over_32_images(cs):
    """Every pair of 32 images joins feature f with feature f (f < 50): 50 tracks of 32 views, and image 31's
    feature 50 + a joined with feature 50 + a of one other image a."""
    m, k = 32, 50
    f = np.arange(k)
    lists = [(a, b, np.stack([f, f], 1)) for a, b in itertools.combinations(range(m), 2)]
    lists += [(a, 31, [[50 + a, 50 + a]]) for a in range(31)]
    T, off, _, tof, st = check(cs, [k + 31] * m, lists)
    assert T == k + 31 and (np.diff(off)[:k] == m).all() and st[0] == k * m * (m - 1) // 2 + 31


def test_fifty_million_pairs(cs):
    """About 5 * 10^7 pairs in 2 000 lists of 25 000 over 500 images of 20 000 features."""
    rng = np.random.default_rng(17)
    n, s, P = 500, 20000, 25000
    lists = [(int(a), int(b), rng.integers(0, s, (P, 2), dtype=np.int32)) for a, b in rng.integers(0, n, (2000, 2))]
    _, _, _, _, st = check(cs, [s] * n, lists, 2, 0)
    assert st[0] == 2000 * P and st[3] >= 1


def test_truncation(cs):
    sizes, lists = collection(3)
    T, off, mem, _, st = check(cs, sizes, lists)
    M = int(st[7])
    for mt, mm in ((0, 0), (1, 1), (T // 2, M // 3), (T - 1, M - 1), (T, M), (T + 5, M + 5)):
        check(cs, sizes, lists, 2, 1, mt, mm)


def test_invariance(cs):
    """Permuted lists, permuted pairs, swapped roles and duplicated lists give the same bytes, and so does a second
    call."""
    sizes, lists = collection(4)
    ref = check(cs, sizes, lists)
    rng = np.random.default_rng(8)
    variants = {
        "lists permuted": [lists[q] for q in rng.permutation(len(lists))],
        "pairs permuted": [(a, b, np.asarray(p)[rng.permutation(len(p))]) for a, b, p in lists],
        "roles swapped": [(b, a, np.asarray(p).reshape(-1, 2)[:, ::-1]) if q % 2 else (a, b, p)
                          for q, (a, b, p) in enumerate(lists)],
        "lists duplicated": lists + lists[::3],
        "same": lists,
    }
    for what, v in variants.items():
        got = check(cs, sizes, v)
        assert got[0] == ref[0], what
        for x, y in zip(got[1:4], ref[1:4]):
            assert x.tobytes() == y.tobytes(), what
        assert got[4][2:].tolist() == ref[4][2:].tolist(), what


def test_launch_count(cs):
    sizes, lists = collection(5)
    L = Lists(cs, lists)
    big = Lists(cs, lists * 20)
    try:
        lib = cs.lib()
        for x in (L, big):
            before = lib.cs_launch_count()
            run(cs, sizes, x)
            assert lib.cs_launch_count() - before == LAUNCHES
        empty = Lists(cs, [(0, 1, np.zeros((0, 2)))])
        before = lib.cs_launch_count()
        T, off, _, tof, st, _, _, _ = run(cs, sizes, empty)
        empty.free()
        assert lib.cs_launch_count() == before and T == 0 and not st.any() and off[0] == 0 and (off[1:] == SENTINEL).all()
        assert (tof[:-1] == -1).all() and tof[-1] == SENTINEL
    finally:
        L.free()
        big.free()


def test_interleaving_with_other_calls(cs):
    """Tracks between guided batch, ratio and verify calls: both sides give the bytes they give alone."""
    arrays, jobs = _mixed()
    S = Sets(cs, arrays)
    keep = []
    sizes, lists = collection(6)
    try:
        (p0, n0), (p1, n1) = S.sets[0], S.sets[1]
        d0, d1 = _sift_data(cs, p0, n0, keep), _sift_data(cs, p1, n1, keep)

        def others():
            c, s, a = guided_batch(cs, S.sets, jobs, 4.0, 1)
            r, _ = cs.MatchSiftDataRatio(d0, d1)
            v = cs.VerifyPairs(d0, d1, r, "fundamental", 512, 4.0, 3)
            return c.tobytes(), s.tobytes(), [x.tobytes() for x in a], r.tobytes(), v[0].tobytes(), v[1].tobytes()

        want = others()
        first = check(cs, sizes, lists)
        assert others() == want
        again = check(cs, sizes, lists)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(first[1:], again[1:])) and first[0] == again[0]
        assert others() == want
    finally:
        S.free()


def test_end_to_end_collection(cs):
    """The six shifted views of the guided batch's chain test: ranked batch extraction (N = 1000), the ratio batch over
    the 15 pairs, the verify batch (F), the jobs with at least 30 inliers, the guided batch, then BuildTracks on the
    guided pairs: equal to the oracle, with at least one track over all six views."""
    w, h = 960, 540
    img = synth_image(w, h, seed=9)
    shifts = [(0, 0), (3, 5), (-4, 6), (8, -2), (-6, -7), (10, 9)]
    views = [np.ascontiguousarray(np.roll(img, s, axis=(0, 1))) for s in shifts]
    pitch = cs.iAlignUp(w, 128)
    cis = [cs.CudaImage().Allocate(w, h, pitch, False, None, v) for v in views]
    for ci in cis:
        ci.Download()
    ex = cs.Extractor(w, h, 5, 1000, False, batch=6, maxCandidates=16384)
    datas = []
    try:
        ex.submit_device_batch([ci.d_data for ci in cis], pitch, 1.0, 3.0, 0.0)
        counts = ex.wait_batch(6)
        for i in range(6):
            d = cs.SiftData()
            cs.InitSiftData(d, int(counts[i]))
            d._buf.upload(ex.device_points_at(i, int(counts[i])))
            d.numPts = int(counts[i])
            datas.append(d)
    finally:
        ex.close()
    try:
        pairs_idx = list(itertools.combinations(range(6), 2))
        ratio, _, _ = cs.MatchSiftDataRatioBatch(datas, pairs_idx)
        Mv, inl, _, _ = cs.VerifyPairsBatch([(datas[a], datas[b], ratio[k], k) for k, (a, b) in enumerate(pairs_idx)],
                                            "fundamental", 1024, 4.0)
        keep = [k for k in range(len(pairs_idx)) if len(inl[k]) >= 30]
        assert len(keep) >= 10
        jobs = [pairs_idx[k] for k in keep]
        guided, _, _ = cs.MatchSiftDataGuidedBatch(datas, jobs, "fundamental", Mv[keep], 4.0)
        sizes = [d.numPts for d in datas]
        lists = [(a, b, g) for (a, b), g in zip(jobs, guided)]
        offsets, members, trackOf, stats, ms = cs.BuildTracks(sizes, lists)
        T, wOff, wMem, wOf, wSt = to.build_tracks(sizes, lists)
        assert ms > 0 and offsets.tobytes() == wOff.tobytes() and members.tobytes() == wMem.tobytes()
        assert trackOf.tobytes() == wOf.tobytes() and stats.tolist() == wSt.tolist()
        views_per_track = [len(np.unique(members[offsets[t]:offsets[t + 1], 0])) for t in range(T)]
        assert T > 100 and max(views_per_track) == 6
    finally:
        for d in datas:
            cs.FreeSiftData(d)
