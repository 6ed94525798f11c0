"""cs_vocab_assign, cs_vocab_train and cs_retrieve_pairs without a device: the symbols, every argument check and the
name it reports, the calls that make no CUDA call, the wrappers through a fake library, and the numpy statement itself
(planted clusters, planted neighbours, the q-weight scores against a float64 tf-idf product)."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

import vocab_oracle as vo
import cudasift_b200 as cs
from cudasift_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_E_ARG = -2
REC = 576
NEW = ("cs_vocab_assign", "cs_vocab_train", "cs_retrieve_pairs")


def test_symbols_declared_exported_and_typed():
    header = open(os.path.join(ROOT, "include", "cudasift_b200.h")).read()
    declared = set(re.findall(r"\b(cs_[a-z0-9_]+)\s*\(", header))
    out = subprocess.run(["nm", "-D", "--defined-only", build.build_library()], stdout=subprocess.PIPE,
                         text=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.strip()}
    for name in NEW:
        assert name in declared and name in exported, name
        assert getattr(cs.lib(), name).restype is ctypes.c_int
    assert len(cs.lib().cs_vocab_assign.argtypes) == 7 and len(cs.lib().cs_vocab_train.argtypes) == 9
    assert len(cs.lib().cs_retrieve_pairs.argtypes) == 12
    for name in ("TrainVocabulary", "AssignWords", "RetrievePairs"):
        assert name in cs.__all__ and hasattr(cs, name)


class Arena:
    """Host memory laid out as on the device: two sets of 4 records, a vocabulary of 4 records and the outputs.
    Nothing is dereferenced: every case fails its checks or has nothing to do."""

    def __init__(self):
        self.buf = np.zeros(12 * REC + 8192, np.uint8)
        base = self.buf.ctypes.data + (-self.buf.ctypes.data) % 256
        self.pts = [base, base + 4 * REC]
        self.vocab = base + 8 * REC
        o = base + 12 * REC
        self.wordOf, self.nb, self.sc, self.idf, self.pairs = o, o + 256, o + 512, o + 1024, o + 2048


def _sets(specs):
    return (cs.MatchSet * max(len(specs), 1))(*[cs.MatchSet(p, n) for p, n in specs])


def _assign(a, **kw):
    c = dict(sets=[(a.pts[0], 4), (a.pts[1], 4)], S=2, vocab=a.vocab, W=4, wordOf=a.wordOf)
    c.update(kw)
    stats, ms = np.full(5, 7, np.uint64), ctypes.c_double(-1.0)
    r = cs.lib().cs_vocab_assign(_sets(c["sets"]) if c.get("setsPtr", 1) else None, c["S"], c["vocab"], c["W"],
                                 c["wordOf"], stats.ctypes.data, ctypes.byref(ms))
    return r, ms.value, stats


def _train(a, **kw):
    c = dict(sets=[(a.pts[0], 4), (a.pts[1], 4)], S=2, W=4, it=5, vocab=a.vocab)
    c.update(kw)
    trace, stats, ms = np.full(4 * 8, 5.0), np.full(4, 7, np.int64), ctypes.c_double(-1.0)
    r = cs.lib().cs_vocab_train(_sets(c["sets"]), c["S"], c["W"], c["it"], 0, c["vocab"], trace.ctypes.data,
                                stats.ctypes.data, ctypes.byref(ms))
    return r, ms.value, stats


def _retrieve(a, **kw):
    c = dict(sizes=[4, 4], I=2, wordOf=a.wordOf, W=100, K=8, nb=a.nb, sc=a.sc, idf=a.idf, pairs=a.pairs, maxPairs=16)
    c.update(kw)
    sizes = np.ascontiguousarray(c["sizes"], np.int32)
    stats, ms = np.full(7, 7, np.int64), ctypes.c_double(-1.0)
    r = cs.lib().cs_retrieve_pairs(sizes.ctypes.data if c.get("sizesPtr", 1) else None, c["I"], c["wordOf"], c["W"],
                                   c["K"], c["nb"], c["sc"], c["idf"], c["pairs"], c["maxPairs"], stats.ctypes.data,
                                   ctypes.byref(ms))
    return r, ms.value, stats


def _rejects(call, a, cases):
    for what, kw, name in cases:
        r, ms, stats = call(a, **kw)
        assert r == CS_E_ARG, (what, r)
        msg = cs.lib().cs_last_error().decode()
        assert "invalid argument" in msg and name in msg, (what, name, msg)
        assert ms == 0.0 and (stats == 7).all(), what
    assert not a.buf.any()


def test_assign_rejects_every_invalid_argument():
    a = Arena()
    _rejects(_assign, a, [
        ("numSets < 0", dict(S=-1), "numSets"),
        ("numSets > 65536", dict(S=65537), "numSets"),
        ("NULL sets", dict(setsPtr=0), "sets"),
        ("a set with n < 0", dict(sets=[(a.pts[0], 4), (a.pts[1], -1)]), "sets[1]"),
        ("a set without records", dict(sets=[(None, 4), (a.pts[1], 4)]), "sets[0]"),
        ("sizes past INT_MAX", dict(sets=[(a.pts[0], 2 ** 31 - 1), (a.pts[1], 4)]), "sets[1]"),
        ("numWords 0", dict(W=0), "numWords"),
        ("numWords 2^18 + 1", dict(W=(1 << 18) + 1), "numWords"),
        ("NULL vocab", dict(vocab=None), "d_vocab"),
        ("vocab unaligned", dict(vocab=a.vocab + 8), "d_vocab"),
        ("NULL wordOf", dict(wordOf=None), "d_wordOf"),
        ("wordOf unaligned", dict(wordOf=a.wordOf + 2), "d_wordOf"),
        ("wordOf over the vocabulary", dict(wordOf=a.vocab + 64), "d_wordOf and d_vocab"),
        ("wordOf over a set", dict(wordOf=a.pts[1] + 8), "d_wordOf and sets[1].pts"),
    ])


def test_train_rejects_every_invalid_argument():
    a = Arena()
    _rejects(_train, a, [
        ("numSets < 0", dict(S=-1), "numSets"),
        ("numWords 0", dict(W=0), "numWords"),
        ("numWords above M", dict(W=9), "numWords"),
        ("no features", dict(sets=[(None, 0), (None, 0)]), "numWords"),
        ("maxIterations -1", dict(it=-1), "maxIterations"),
        ("maxIterations 1001", dict(it=1001), "maxIterations"),
        ("NULL vocab", dict(vocab=None), "d_vocab"),
        ("vocab unaligned", dict(vocab=a.vocab + 4), "d_vocab"),
        ("vocab over a set", dict(vocab=a.pts[0] + 16 * 16), "d_vocab and sets[0].pts"),
    ])


def test_retrieve_rejects_every_invalid_argument():
    a = Arena()
    _rejects(_retrieve, a, [
        ("numImages < 0", dict(I=-1), "numImages"),
        ("numImages > 65536", dict(I=65537), "numImages"),
        ("NULL imageSizes", dict(sizesPtr=0), "imageSizes"),
        ("a negative size", dict(sizes=[4, -1]), "imageSizes[1]"),
        ("sizes past INT_MAX", dict(sizes=[2 ** 31 - 1, 4]), "imageSizes[1]"),
        ("numWords 0", dict(W=0), "numWords"),
        ("topK 0", dict(K=0), "topK"),
        ("topK 1025", dict(K=1025), "topK"),
        ("maxPairs < 0", dict(maxPairs=-1), "maxPairs"),
        ("NULL wordOf", dict(wordOf=None), "d_wordOf"),
        ("NULL neighbours", dict(nb=None), "d_neighbours"),
        ("NULL pairs", dict(pairs=None), "d_pairs"),
        ("neighbours unaligned", dict(nb=a.nb + 2), "d_neighbours"),
        ("scores unaligned", dict(sc=a.sc + 4), "d_scores"),
        ("idf unaligned", dict(idf=a.idf + 4), "d_idf"),
        ("neighbours over wordOf", dict(nb=a.wordOf + 16), "d_wordOf and d_neighbours"),
        ("scores over neighbours", dict(sc=a.nb + 8), "d_neighbours and d_scores"),
        ("idf over scores", dict(idf=a.sc + 64), "d_scores and d_idf"),
        ("pairs over idf", dict(pairs=a.idf + 8), "d_idf and d_pairs"),
    ])


def test_calls_without_features_make_no_cuda_call():
    """No features: the assignment and the retrieval return 0 with zero statistics and touch nothing (this holds
    without a device); a training call without features is an argument error."""
    a = Arena()
    r, ms, stats = _assign(a, sets=[(None, 0), (None, 0)], wordOf=None)
    assert r == 0 and ms == 0.0 and not stats.any()
    r, ms, stats = _assign(a, S=0, sets=[], wordOf=None)
    assert r == 0 and not stats.any()
    r, ms, stats = _retrieve(a, sizes=[0, 0], wordOf=None)
    assert r == 0 and ms == 0.0 and not stats.any()
    r, ms, stats = _retrieve(a, I=0, sizes=[0], nb=None, sc=None)
    assert r == 0 and not stats.any()
    assert not a.buf.any()


class _FakeLib:
    def __init__(self):
        self.calls = []

    def cs_device_alloc(self, n):
        return 4096 * (len(self.calls) + 1)

    def cs_device_free(self, p):
        return 0

    def cs_memcpy_h2d(self, dst, src, n):
        return 0

    def cs_memcpy_d2h(self, dst, src, n):
        return 0

    def cs_vocab_train(self, *args):
        self.calls.append(("train", args))
        stats = np.ctypeslib.as_array(ctypes.cast(args[7], ctypes.POINTER(ctypes.c_longlong)), (4,))
        stats[:] = [3, 1, 100, 20]
        return 3

    def cs_vocab_assign(self, *args):
        self.calls.append(("assign", args))
        return 0

    def cs_retrieve_pairs(self, *args):
        self.calls.append(("retrieve", args))
        return 0


class _Data:
    def __init__(self, n):
        self.d_data, self.numPts = 1 << 20, n


def test_wrappers_build_their_arguments(monkeypatch):
    fake = _FakeLib()
    monkeypatch.setattr(cs, "lib", lambda: fake)
    datas = [_Data(40), _Data(0), _Data(60)]
    vocab, trace, stats, _ = cs.TrainVocabulary(datas, 16)
    kind, args = fake.calls[-1]
    assert kind == "train" and args[1] == 3 and args[2] == 16 and args[3] == 10 and args[4] == 0
    assert vocab.numPts == 16 and trace.shape == (3, 4) and list(stats) == [3, 1, 100, 20]
    cs.TrainVocabulary(datas, 8, maxIterations=0, seed=5)
    kind, args = fake.calls[-1]
    assert args[3] == 0 and args[4] == 5 and args[6] is None
    wordOf, st, _ = cs.AssignWords(datas, vocab)
    kind, args = fake.calls[-1]
    assert kind == "assign" and args[1] == 3 and args[3] == 16 and wordOf.shape == (100,) and st.shape == (5,)
    nb, sc, pairs, st, _ = cs.RetrievePairs([40, 0, 60], np.zeros(100, np.int32), 16, topK=4)
    kind, args = fake.calls[-1]
    assert kind == "retrieve" and args[1] == 3 and args[3] == 16 and args[4] == 4 and args[7] is None
    assert args[9] == 12 and nb.shape == (3, 4) and sc.shape == (3, 4) and pairs.shape == (0, 2)
    with pytest.raises(ValueError):
        cs.RetrievePairs([40, 0, 60], np.zeros(99, np.int32), 16)


# ------------------------------------------------------------------------------ the statement itself
def _assign_float64(desc, words):
    s = desc.astype(np.float64) @ words.astype(np.float64).T
    w = np.argmax(s, axis=1)
    return np.where(s.max(axis=1) > 0, w, -1), s.max(axis=1).astype(np.float32), 0


def test_oracle_kmeans_recovers_planted_clusters():
    """6 tight clusters and 24 words: every word keeps members of one cluster only, every cluster keeps a word, each
    word with members converges onto its centre, and the loop stops on no change."""
    rng = np.random.default_rng(4)
    centres = rng.random((6, 128))
    centres /= np.linalg.norm(centres, axis=1, keepdims=True)
    label = rng.integers(0, 6, 3000)
    desc = centres[label] + rng.normal(0, 0.005, (3000, 128))
    desc = (desc / np.linalg.norm(desc, axis=1, keepdims=True)).astype(np.float32)
    words, trace, it, stopped = vo.kmeans(desc, 24, 50, 1, lambda w: _assign_float64(desc, w))
    wordOf = _assign_float64(desc, words)[0]
    assert all(len(set(label[wordOf == k])) <= 1 for k in range(24))
    assert set(label[wordOf >= 0]) == set(range(6)) and (wordOf >= 0).all()
    used = np.unique(wordOf)
    assert np.abs(np.sort(words[used] @ centres.T, axis=1)[:, -1] - 1).max() < 1e-3
    assert stopped == 1 and trace[-1, 0] == 0 and trace[0, 0] == 3000


def test_oracle_start_draws_follow_the_counter_rule():
    from verify_oracle import GOLDEN, splitmix64
    d = vo.start_draws(11, 1000, 50)
    assert len(set(d.tolist())) == 50
    x = splitmix64(np.uint64(11) + GOLDEN * np.uint64(0))
    assert d[0] == int((int(x) >> 32) * 1000 >> 32)


def test_oracle_retrieval_returns_planted_neighbours():
    """Ten groups of five images, each group drawing from its own 40 words: the neighbours of an image are the other
    four of its group (topK 4), and the pair table is the groups' 10 x 10 pairs."""
    rng = np.random.default_rng(2)
    sizes, words = [], []
    for a in range(50):
        g = a // 5
        w = rng.integers(40 * g, 40 * g + 40, 60)
        sizes.append(len(w))
        words.append(w)
    sizes, words = np.array(sizes), np.concatenate(words).astype(np.int32)
    nb, sc, pairs, q, S, iw, stats = vo.retrieve(sizes, words, 400, 4)
    for a in range(50):
        assert sorted(nb[a].tolist()) == [b for b in range(5 * (a // 5), 5 * (a // 5) + 5) if b != a]
        assert (np.diff(sc[a]) <= 0).all() and (sc[a] > 0).all()
    assert len(pairs) == 100 and stats["Nprime"] == 50


def test_oracle_scores_match_a_float64_tfidf_product():
    """The q-weight scores 2^-44 equal the cosine of scipy.sparse float64 tf-idf vectors to within 2^-20 relative."""
    import scipy.sparse as sp
    rng = np.random.default_rng(9)
    I, W = 120, 3000
    sizes = rng.integers(50, 400, I)
    p = np.arange(1, W + 1) ** -1.1
    words = rng.choice(W, int(sizes.sum()), p=p / p.sum()).astype(np.int32)
    tf, df, Np = vo.bag_of_words(sizes, words, W)
    iw = vo.idf(df, Np)
    S = vo.scores(vo.weights(tf, iw), W).toarray().astype(np.float64) * vo.SCORE_SCALE
    rows = np.repeat(np.arange(I), sizes)
    T = sp.csr_matrix((np.ones(len(words)), (rows, words)), shape=(I, W))
    X = T.multiply(iw[None, :]).tocsr()
    n = np.sqrt(np.asarray(X.multiply(X).sum(axis=1)).ravel())
    C = (X @ X.T).toarray() / np.outer(n, n)
    # relative to the similarity scale (1 for identical vectors), over the pairs that can be listed (b != a)
    off = ~np.eye(I, dtype=bool)
    assert (C[off] > 1e-3).sum() > I and np.abs(S[off] - C[off]).max() <= 2.0 ** -20
