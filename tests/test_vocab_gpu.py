"""GPU checks of the vocabulary and retrieval calls: cs_vocab_assign against cs_match_knn2's j1 and the CPU statement
(tests/knn_oracle.c) on extracted and synthetic records, an empty set, the bad-input gate, 2^18 words and several
waves; cs_vocab_train word for word and trace against tests/vocab_oracle.py, determinism, the stop rule and empty
words; cs_retrieve_pairs against the oracle (idf to 1 ulp, the rest exact) with its edge cases; and the retrieval chain
on a synthetic collection against the exhaustive ratio + verification recipe."""
import ctypes
import itertools

import numpy as np
import pytest

import knn_oracle
import vocab_oracle as vo
from cudasift_b200.synth import synth_descriptors, synth_image

pytestmark = pytest.mark.gpu
REC = 576


def _records(desc):
    """Vocabulary records: the descriptors, every other field 0."""
    r = np.zeros(len(desc), synth_descriptors(1, 0).dtype)
    r["data"] = desc
    return r


class _Sets:
    """Record arrays on the device as SiftData (one buffer each)."""

    def __init__(self, cs, arrays):
        self.datas = []
        for a in arrays:
            d = cs.InitSiftData(cs.SiftData(), max(len(a), 1))
            if len(a):
                d._buf.upload(a)
            d.numPts = len(a)
            self.datas.append(d)

    def free(self, cs):
        for d in self.datas:
            cs.FreeSiftData(d)


def _extract(cs, views, maxPts=1000):
    """Ranked batch extraction of float32 views (one size, at most 32): host record arrays."""
    h, w = views[0].shape
    pitch = cs.iAlignUp(w, 128)
    cis = [cs.CudaImage().Allocate(w, h, pitch, False, None, v) for v in views]
    for ci in cis:
        ci.Download()
    ex = cs.Extractor(w, h, 5, maxPts, False, batch=len(views), maxCandidates=16384)
    try:
        ex.submit_device_batch([ci.d_data for ci in cis], pitch, 1.0, 3.0, 0.0)
        counts = ex.wait_batch(len(views))
        return [ex.device_points_at(i, int(counts[i])).copy() for i in range(len(views))]
    finally:
        ex.close()


def _assign_check(cs, arrays, vocab, oracle=True):
    S = _Sets(cs, arrays)
    V = _Sets(cs, [vocab])
    try:
        L = cs.lib()
        before = L.cs_launch_count()
        wordOf, stats, ms = cs.AssignWords(S.datas, V.datas[0])
        launches = L.cs_launch_count() - before
        base = 0
        for a in arrays:
            n = len(a)
            if n:
                gi, _, _ = cs.match_knn2(a, vocab, mode=2)
                assert wordOf[base:base + n].tobytes() == gi[:, 0].tobytes()
                if oracle:
                    oi, _ = knn_oracle.match_knn2(a, vocab)
                    assert wordOf[base:base + n].tobytes() == oi[:, 0].tobytes()
            base += n
        assert base == len(wordOf)
        return wordOf, stats, launches
    finally:
        S.free(cs)
        V.free(cs)


def test_assign_equals_knn2(cs):
    """Extracted records, synthetic ones, an empty set and a set with a NaN (gated): j1 of cs_match_knn2 and of the
    CPU statement, bit for bit; 5 launches per wave."""
    img = synth_image(960, 540, seed=31)
    ext = _extract(cs, [img])[0]
    vocab = _records(synth_descriptors(3000, 5, sift_like=True)["data"])
    gated = synth_descriptors(300, 7)
    gated["data"][17, 3] = np.nan
    arrays = [ext, synth_descriptors(1000, 1), np.zeros(0, ext.dtype), gated, synth_descriptors(257, 2, sift_like=True),
              np.zeros(64, ext.dtype)]                                       # all-zero rows: word -1
    wordOf, stats, launches = _assign_check(cs, arrays, vocab)
    assert stats[4] == 1 and launches == 5 * int(stats[4])
    assert stats[3] == 1 and stats[2] >= 300                                  # the gated set went the exact way
    nan_row = len(arrays[0]) + len(arrays[1]) + 17                          # no positive score either
    assert (wordOf[-64:] == -1).all() and wordOf[nan_row] == -1
    assert (np.delete(wordOf[:-64], nan_row) >= 0).all()


def test_assign_2p18_words(cs):
    vocab = _records(synth_descriptors(1 << 18, 11)["data"])
    _, stats, launches = _assign_check(cs, [synth_descriptors(400, 12)], vocab)
    assert launches == 5 * int(stats[4]) and stats[4] == 1


def _assign_waves(ns, numWords):
    """The wave rule of cs_match_ratio_batch (crossCheck 0) over the jobs (a, vocabulary): per distinct set 516 bytes
    per row rounded up to 128 rows, per direction 160 bytes per row rounded up to 128 rows plus 24 per row."""
    set_b = lambda n: -(-n // 128) * 128 * 516
    dir_b = lambda n: -(-n // 128) * 128 * 160 + 24 * n
    waves, total = 0, 0
    for n in ns:
        if n == 0:
            continue
        cost = dir_b(n) + set_b(n)
        if waves == 0 or total + cost > 256 << 20:
            waves, total = waves + 1, set_b(numWords)
        total += cost
    return waves


def test_assign_several_waves(cs):
    ns = [30000] * 16
    arrays = [synth_descriptors(n, 40 + k) for k, n in enumerate(ns)]
    vocab = _records(synth_descriptors(65536, 39)["data"])
    waves = _assign_waves(ns, 65536)
    assert waves >= 2
    _, stats, launches = _assign_check(cs, arrays, vocab, oracle=False)
    assert stats[4] == waves and launches == 5 * waves


def _training_set(cs):
    views = [synth_image(960, 540, seed=200 + k) for k in range(24)]
    recs = _extract(cs, views)
    desc = np.concatenate([r["data"] for r in recs])[:20000]
    assert len(desc) == 20000
    return recs, desc


def _assign_host(desc, words):
    idx, sc = knn_oracle.match_knn2(_records(desc), _records(words))
    return idx[:, 0], sc[:, 0]


def test_train_against_oracle(cs):
    """20 000 extracted descriptors, 512 words, 8 iterations: the words after every iteration equal the oracle's
    update of the same assignment, bit for bit, and the trace equals the oracle's; two calls give the same bytes."""
    _, desc = _training_set(cs)
    S = _Sets(cs, [_records(desc[:7000]), _records(desc[7000:])])
    try:
        runs = []
        for t in range(9):
            vocab, trace, stats, _ = cs.TrainVocabulary(S.datas, 512, t, seed=3)
            runs.append((vocab._buf.download(synth_descriptors(1, 0).dtype, 512), trace, stats))
            cs.FreeSiftData(vocab)
        start = desc[vo.start_draws(3, len(desc), 512)]
        assert runs[0][0]["data"].tobytes() == start.tobytes() and not runs[0][1].size
        for t in range(8):
            words, trace, stats = runs[t + 1]
            prev = runs[t][0]["data"]
            wordOf, best = _assign_host(desc, prev)
            V = _Sets(cs, [_records(prev)])
            dev, _, _ = cs.AssignWords(S.datas, V.datas[0])
            V.free(cs)
            assert dev.tobytes() == wordOf.tobytes(), t
            want, empty = vo.update(desc, prev, wordOf)
            assert words["data"].tobytes() == want.tobytes(), t
            assert trace[t, 1] == empty and trace[t, 3] == vo.mean_best(wordOf, best), t
            rest = words.copy()
            rest["data"] = 0
            assert not rest.view(np.uint8).any()
        # the whole trace of the 8-iteration call against the oracle loop on the host assignment
        assign = lambda w: (*_assign_host(desc, w), 0)
        ow, otrace, it, stopped = vo.kmeans(desc, 512, 8, 3, assign)
        words, trace, stats = runs[8]
        assert ow.tobytes() == words["data"].tobytes()
        assert np.array_equal(trace[:, [0, 1, 3]], otrace[:, [0, 1, 3]]) and stats[0] == it and stats[1] == stopped
        assert stats[2] == 20000
        again, trace2, stats2, _ = cs.TrainVocabulary(S.datas, 512, 8, seed=3)
        assert again._buf.download(np.uint8, 512 * REC).tobytes() == runs[8][0].tobytes()
        assert trace2.tobytes() == trace.tobytes() and stats2.tobytes() == stats.tobytes()
        cs.FreeSiftData(again)
    finally:
        S.free(cs)


def test_train_stop_rule_and_empty_words(cs):
    """8 distinct descriptors each repeated 250 times and 16 words: the start draws repeat descriptors, the tie rule
    empties the higher copies, and the second assignment repeats the first, so the loop stops."""
    base = synth_descriptors(8, 90)["data"]
    desc = np.repeat(base, 250, axis=0)
    S = _Sets(cs, [_records(desc)])
    try:
        L = cs.lib()
        before = L.cs_launch_count()
        vocab, trace, stats, _ = cs.TrainVocabulary(S.datas, 16, 20, seed=1)
        launches = L.cs_launch_count() - before
        assert stats[1] == 1 and stats[0] == len(trace) and stats[0] < 20
        drawn = len({tuple(v) for v in desc[vo.start_draws(1, len(desc), 16)].tolist()})
        assert trace[0, 1] == 16 - drawn > 0 and trace[-1, 0] == 0 and trace[-1, 1] == trace[-2, 1]
        assert launches == stats[3] == 1 + 6 * stats[0] + 2 * (stats[0] - 1)
        assign = lambda w: (*_assign_host(desc, w), 0)
        ow, otrace, it, stopped = vo.kmeans(desc, 16, 20, 1, assign)
        got = vocab._buf.download(synth_descriptors(1, 0).dtype, 16)["data"]
        assert got.tobytes() == ow.tobytes() and it == stats[0] and stopped == 1
        assert np.array_equal(trace[:, [0, 1, 3]], otrace[:, [0, 1, 3]])
        cs.FreeSiftData(vocab)
    finally:
        S.free(cs)


def _zipf_words(I, per, numWords, seed, a=1.2):
    rng = np.random.default_rng(seed)
    sizes = rng.integers(per // 2, per + 1, I)
    ranks = np.arange(1, numWords + 1, dtype=np.float64) ** -a
    p = ranks / ranks.sum()
    perm = rng.permutation(numWords)
    words = perm[rng.choice(numWords, int(sizes.sum()), p=p)].astype(np.int32)
    return sizes.astype(np.int32), words


def _retrieve_c(cs, sizes, words, numWords, topK, maxPairs):
    I, N = len(sizes), len(words)
    bufs = [cs.DeviceBuffer(max(N, 1) * 4), cs.DeviceBuffer(max(I * topK, 1) * 4), cs.DeviceBuffer(max(I * topK, 1) * 8),
            cs.DeviceBuffer(numWords * 8), cs.DeviceBuffer(max(maxPairs + 1, 1) * 8)]
    try:
        bufs[0].upload(words)
        bufs[4].upload(np.full(2 * (maxPairs + 1), -7, np.int32))
        stats, ms = np.zeros(7, np.int64), ctypes.c_double(0.0)
        L = cs.lib()
        before = L.cs_launch_count()
        P = L.cs_retrieve_pairs(sizes.ctypes.data, I, bufs[0].ptr, numWords, topK, bufs[1].ptr, bufs[2].ptr,
                                bufs[3].ptr, bufs[4].ptr, maxPairs, stats.ctypes.data, ctypes.byref(ms))
        assert P >= 0, L.cs_last_error().decode()
        launches = L.cs_launch_count() - before
        nb = bufs[1].download(np.int32, I * topK).reshape(I, topK)
        sc = bufs[2].download(np.float64, I * topK).reshape(I, topK)
        idf = bufs[3].download(np.float64, numWords)
        pairs = bufs[4].download(np.int32, 2 * (maxPairs + 1)).reshape(-1, 2)
    finally:
        for b in bufs:
            b.free()
    return P, nb, sc, idf, pairs, stats, launches


def _retrieve_check(cs, sizes, words, numWords, topK, maxPairs=None):
    I = len(sizes)
    maxPairs = I * topK if maxPairs is None else maxPairs
    P, nb, sc, idf, pairs, stats, launches = _retrieve_c(cs, sizes, words, numWords, topK, maxPairs)
    tf, df, Np = vo.bag_of_words(sizes, words, numWords)
    host = vo.idf(df, Np)
    assert np.all(np.abs(idf - host) <= np.spacing(np.maximum(np.abs(host), 1e-300)))
    onb, osc, opairs, q, S, _, ost = vo.retrieve(sizes, words, numWords, topK, idf_w=idf)
    assert nb.tobytes() == onb.tobytes() and sc.tobytes() == osc.tobytes()
    assert P == len(opairs) and stats[5] == P
    w = min(P, maxPairs)
    assert pairs[:w].tobytes() == opairs[:w].tobytes() and (pairs[w:] == -7).all()
    assert (stats[0], stats[1], stats[2], stats[3]) == (ost["Nprime"], ost["postings"], ost["sumDf2"], ost["updates"])
    per = max(1, min(I, (256 << 20) // (8 * I)))
    waves = -(-I // per)
    assert stats[4] == waves and launches == 6 + 2 * waves
    return nb, sc, opairs, stats


def test_retrieve_against_oracle(cs):
    sizes, words = _zipf_words(300, 400, 2000, 5)
    words[:50] = -1                                                           # ignored features
    sizes[7] = 0                                                              # an image without features
    words = words[:int(sizes.sum())]
    # image 9 repeats image 3's words, image 12 has only ignored ones
    base = np.concatenate([[0], np.cumsum(sizes)])
    w3 = words[base[3]:base[4]]
    parts = [words[base[a]:base[a + 1]] for a in range(len(sizes))]
    parts[9], parts[12] = w3.copy(), np.full(len(parts[12]), 5000, np.int32)
    sizes = np.array([len(p) for p in parts], np.int32)
    words = np.concatenate(parts).astype(np.int32)
    nb, sc, pairs, stats = _retrieve_check(cs, sizes, words, 2000, 20)
    assert (nb[7] == -1).all() and (nb[12] == -1).all() and stats[6] == 50 + len(parts[12])
    # identical images: equal scores with every third image, the lower index first
    for a in range(len(sizes)):
        if a not in (3, 9):
            row = list(nb[a])
            if 3 in row and 9 in row:
                assert row.index(3) < row.index(9)
    assert 9 in nb[3] and 3 in nb[9]
    _retrieve_check(cs, sizes[:10], words[:int(sizes[:10].sum())], 2000, 16)   # topK >= numImages
    _retrieve_check(cs, sizes, words, 2000, 20, maxPairs=100)                 # truncation
    _retrieve_check(cs, sizes, words, 2000, 1)


def test_retrieve_several_waves(cs):
    sizes, words = _zipf_words(6000, 30, 20000, 8, a=0.9)
    _, _, _, stats = _retrieve_check(cs, sizes, words, 20000, 10)
    assert stats[4] == 2


def test_retrieval_chain_recalls_the_exhaustive_pairs(cs):
    """4 scenes x 8 views (960 x 540 windows of a 1920 x 1080 scene at overlapping offsets), ranked extraction of 1000
    features, a 4096-word vocabulary and topK 8: every pair the exhaustive recipe verifies (ratio batch over all 496
    pairs, F with at least 30 inliers) is in the retrieved pair table, which has at most 32 x 8 pairs."""
    views = []
    for scene in range(4):
        img = synth_image(1920, 1080, seed=scene)
        for k in range(8):
            x, y = 120 * k, 60 * k
            views.append(np.ascontiguousarray(img[y:y + 540, x:x + 960]))
    recs = _extract(cs, views)
    S = _Sets(cs, recs)
    try:
        vocab, trace, _, _ = cs.TrainVocabulary(S.datas, 4096, 10)
        wordOf, _, _ = cs.AssignWords(S.datas, vocab)
        nb, sc, pairs, stats, _ = cs.RetrievePairs([d.numPts for d in S.datas], wordOf, 4096, topK=8)
        assert len(pairs) <= 32 * 8
        allp = list(itertools.combinations(range(32), 2))
        ratio, _, _ = cs.MatchSiftDataRatioBatch(S.datas, allp)
        jobs = [(S.datas[a], S.datas[b], ratio[k], k) for k, (a, b) in enumerate(allp)]
        _, _, vst, _ = cs.VerifyPairsBatch(jobs, "fundamental", 1024, 4.0)
        accepted = {allp[k] for k in range(len(allp)) if vst[k, 7] >= 30}
        retrieved = {tuple(p) for p in pairs.tolist()}
        assert accepted and accepted <= retrieved, sorted(accepted - retrieved)
        cs.FreeSiftData(vocab)
    finally:
        S.free(cs)
