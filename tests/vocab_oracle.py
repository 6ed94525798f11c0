"""A numpy statement of cs_vocab_train and cs_retrieve_pairs (csrc/vocab.cu) for the tests: the start draws, the word
update, the trace's mean score, the bag of words, idf, the fixed-point weights q, the integer scores, the top-k order and
the pair table.  The word of a descriptor comes from tests/knn_oracle.c (j1 of cs_match_knn2), which states the FMA
chain.

TEST INFRASTRUCTURE ONLY."""
import numpy as np

from verify_oracle import GOLDEN, splitmix64

Q_SCALE = 2.0 ** 22
SCORE_SCALE = 2.0 ** -44


# ------------------------------------------------------------------------------ training
def start_draws(seed, M, numWords):
    """The first numWords distinct idx = ((splitmix64(seed + GOLDEN * counter) >> 32) * M) >> 32, counter 0, 1, ..."""
    out, seen, ctr = [], set(), 0
    while len(out) < numWords:
        block = np.arange(ctr, ctr + 4096, dtype=np.uint64)
        with np.errstate(over="ignore"):
            x = splitmix64(np.uint64(seed) + GOLDEN * block)
        idx = ((x >> np.uint64(32)) * np.uint64(M)) >> np.uint64(32)
        for v in idx.tolist():
            if v not in seen:
                seen.add(v)
                out.append(v)
                if len(out) == numWords:
                    break
        ctr += 4096
    return np.array(out, np.int64)


def update(desc, words, wordOf):
    """The word update: per word with members, s = the members' descriptors summed per component in float64 in
    ascending index, norm = the 128 squares summed in ascending component, float32(s / sqrt(norm)); a word without
    members (or norm 0) keeps its descriptor.  Returns (new words, words without members)."""
    desc = np.asarray(desc, np.float32)
    out = np.array(words, np.float32, copy=True)
    order = np.argsort(wordOf, kind="stable")
    w_sorted = wordOf[order]
    empty = 0
    starts = np.searchsorted(w_sorted, np.arange(len(words)), "left")
    ends = np.searchsorted(w_sorted, np.arange(len(words)), "right")
    for k in range(len(words)):
        b, e = starts[k], ends[k]
        if b == e:
            empty += 1
            continue
        s = np.cumsum(desc[order[b:e]].astype(np.float64), axis=0)[-1]     # sequential, ascending index
        sq = s * s
        n = np.cumsum(sq)[-1]                                              # ascending component
        if n > 0.0:
            out[k] = (s / np.sqrt(n)).astype(np.float32)
    return out, empty


def mean_best(wordOf, best):
    """The trace's mean best score: tiles of 1024, thread t sums tile + 4t .. 4t + 3 from 0, the tree s = 128 .. 1, the
    tiles in ascending order, over the assigned count."""
    M = len(wordOf)
    v = np.where(wordOf >= 0, np.asarray(best, np.float64), 0.0)
    T = -(-M // 1024)
    x = np.zeros(T * 1024)
    x[:M] = v
    x = x.reshape(T, 256, 4)
    y = ((x[:, :, 0] + x[:, :, 1]) + x[:, :, 2]) + x[:, :, 3]
    s = 128
    while s >= 1:
        y = y[:, :s] + y[:, s:2 * s]
        s //= 2
    total = 0.0
    for t in y[:, 0]:
        total += float(t)
    n = int((wordOf >= 0).sum())
    return total / n if n else 0.0


def kmeans(desc, numWords, maxIterations, seed, assign):
    """The whole loop; assign(words) -> (wordOf, best score, fallback rows).  Returns (words, trace, iterations,
    stopped)."""
    desc = np.asarray(desc, np.float32)
    words = desc[start_draws(seed, len(desc), numWords)].copy()
    trace = np.zeros((maxIterations, 4))
    prev, stopped, it = None, 0, 0
    for t in range(maxIterations):
        wordOf, best, fb = assign(words)
        changed = len(wordOf) if prev is None else int((wordOf != prev).sum())
        trace[t, 0], trace[t, 2], trace[t, 3] = changed, fb, mean_best(wordOf, best)
        it = t + 1
        if changed == 0:
            trace[t, 1] = trace[t - 1, 1] if t else 0
            stopped = 1
            break
        words, trace[t, 1] = update(desc, words, wordOf)
        prev = wordOf
    return words, trace[:it], it, stopped


# ------------------------------------------------------------------------------ retrieval
def bag_of_words(imageSizes, wordOf, numWords):
    """tf as a dict per image {word: count} over the valid words, the df array and N'."""
    bases = np.concatenate([[0], np.cumsum(imageSizes)]).astype(np.int64)
    tf = []
    for a in range(len(imageSizes)):
        w = np.asarray(wordOf[bases[a]:bases[a + 1]])
        w = w[(w >= 0) & (w < numWords)]
        u, c = np.unique(w, return_counts=True)
        tf.append(dict(zip(u.tolist(), c.tolist())))
    df = np.zeros(numWords, np.int64)
    for d in tf:
        for w in d:
            df[w] += 1
    return tf, df, sum(1 for d in tf if d)


def idf(df, Nprime):
    out = np.zeros(len(df))
    nz = df > 0
    out[nz] = np.log(float(Nprime) / df[nz].astype(np.float64))
    return out


def weights(tf, idf_w):
    """q per image as {word: int}: x = tf idf, norm summed in ascending word, rint(x / sqrt(norm) 2^22)."""
    out = []
    for d in tf:
        ws = sorted(d)
        x = np.array([float(d[w]) * idf_w[w] for w in ws])
        n = np.cumsum(x * x)[-1] if len(x) else 0.0
        if n > 0.0:
            q = np.rint((x / np.sqrt(n)) * Q_SCALE).astype(np.int64)
        else:
            q = np.zeros(len(ws), np.int64)
        out.append(dict(zip(ws, q.tolist())))
    return out


def q_matrix(q, numWords):
    """q as an int64 scipy.sparse CSR matrix [I, numWords]."""
    import scipy.sparse as sp
    rows = [a for a, d in enumerate(q) for _ in d]
    cols = [w for d in q for w in d]
    vals = [v for d in q for v in d.values()]
    return sp.csr_matrix((np.array(vals, np.int64), (np.array(rows, np.int64), np.array(cols, np.int64))),
                         shape=(len(q), numWords))


def scores(q, numWords):
    """The exact int64 score matrix (scipy.sparse CSR [I, I], diagonal included): an integer product."""
    Q = q_matrix(q, numWords)
    return (Q @ Q.T).tocsr()


def topk(S, topK):
    """neighbours [I, topK] (-1 padded) and similarities [I, topK]: b != a with score > 0, score desc then b asc."""
    I = S.shape[0]
    nb, sc = np.full((I, topK), -1, np.int32), np.zeros((I, topK))
    for a in range(I):
        lo, hi = S.indptr[a], S.indptr[a + 1]
        b, s = S.indices[lo:hi], S.data[lo:hi]
        keep = (b != a) & (s > 0)
        b, s = b[keep], s[keep]
        order = np.lexsort((b, -s))[:topK]
        nb[a, :len(order)] = b[order]
        sc[a, :len(order)] = s[order].astype(np.float64) * SCORE_SCALE
    return nb, sc


def pairs(nb):
    """{min, max} of every listed neighbour, deduplicated, ascending."""
    s = set()
    for a in range(len(nb)):
        for b in nb[a]:
            if b >= 0:
                s.add((min(a, int(b)), max(a, int(b))))
    return np.array(sorted(s), np.int32).reshape(-1, 2)


def retrieve(imageSizes, wordOf, numWords, topK, idf_w=None):
    """(neighbours, similarities, pairs, q, S, idf, stats dict); idf_w (for example the device's) replaces the host
    log when given."""
    tf, df, Np = bag_of_words(imageSizes, wordOf, numWords)
    iw = idf(df, Np) if idf_w is None else np.asarray(idf_w, np.float64)
    q = weights(tf, iw)
    S = scores(q, numWords)
    nb, sc = topk(S, topK)
    dfq = np.zeros(numWords, np.int64)
    for d in q:
        for w, v in d.items():
            if v:
                dfq[w] += 1
    stats = dict(Nprime=Np, postings=sum(len(d) for d in tf), sumDf2=int((df * df).sum()), updates=int((dfq * dfq).sum()))
    return nb, sc, pairs(nb), q, S, iw, stats
