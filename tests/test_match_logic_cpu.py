"""CPU restatement (numpy) of the tensor matcher's decision logic (csrc/match_tc.cu: epilogue top-3
tracking + t3_resolve_kernel's reference rule), checked against the oracle's exact MatchSiftData.  It pins the argument
that makes one approximate GEMM pass sufficient: with |approx - exact| <= eps and delta = 2*eps,

  * per (row, partition) the three largest 4-candidate group maxima g1 >= g2 >= g3 and the ids of the
    first two are enough to certify that every candidate that can still decide the row lies in those
    two groups;
  * re-scoring only those groups exactly and applying the reference's update rule and 8-way merge
    reproduces score / match / ambiguity bit for bit; rows that cannot be certified are detected.

The approximate scores here carry the split-FP16 input error only (float64 accumulation); the tensor
cores' accumulation error is inside the same eps budget (T3_C1) and is exercised on the GPU."""
import numpy as np

import oracle
from cudasift_b200.synth import synth_descriptors

T3_C1, T3_C2, SCALE = 4.0e-5, 1.0e-9, 4096.0


def exact_scores(a, b):
    acc = np.zeros((a.shape[0], b.shape[0]), np.float32)
    for k in range(128):            # matching.cu:338-351: sequential FMA chain from 0
        acc = (np.outer(a[:, k].astype(np.float64), b[:, k].astype(np.float64)) + acc.astype(np.float64)).astype(np.float32)
    return acc


def split(x):
    xs = x.astype(np.float32) * np.float32(SCALE)
    hi = xs.astype(np.float16)
    lo = (xs - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def emulate(s1, s2):
    a, b = s1["data"], s2["data"]
    n1, n2v = len(a), (len(b) // 32) * 32
    b = b[:n2v]
    ex = exact_scores(a, b)
    ah, al = split(a)
    bh, bl = split(b)
    approx = ((ah @ bh.T) + (ah @ bl.T) + (al @ bh.T)) / (SCALE * SCALE)
    na = np.sqrt((a.astype(np.float64) ** 2).sum(1)) * 1.0001
    bmax = (np.sqrt((b.astype(np.float64) ** 2).sum(1)) * 1.0001).max()
    gm = approx.reshape(n1, n2v // 4, 4).max(-1)                  # group maxima; group g is in partition g % 8
    out = dict(score=np.zeros(n1, np.float32), match=np.full(n1, -1, np.int32), ambiguity=np.zeros(n1, np.float32))
    uncertified = np.zeros(n1, bool)
    nchains = 0
    for r in range(n1):
        delta = 2.0 * (T3_C1 * na[r] * bmax + T3_C2 * (na[r] + bmax))
        G, S, Th, I1, I2 = np.zeros(8), np.zeros(8), np.zeros(8), [-1] * 8, [-1] * 8
        for p in range(8):
            ids = np.arange(p, n2v // 4, 8)
            v = gm[r, ids]
            order = np.argsort(-v, kind="stable")[:3]             # stable: the first of equal maxima comes first
            top = [(v[o], ids[o]) for o in order if v[o] > 0.0]
            if len(top) > 0: G[p], I1[p] = top[0]
            if len(top) > 1: S[p], I2[p] = top[1]
            if len(top) > 2: Th[p] = top[2][0]
        pool = sorted(list(G) + [S[0]], reverse=True)
        L = pool[1]
        if not (L > 2.0 * delta):
            uncertified[r] = True
            continue
        cand, ok = [], True
        for p in range(8):
            if G[p] < L - delta:
                continue                                          # cannot be first or second
            low = (min(L, G[p]) if p == 0 else G[p]) - delta       # partition 0 also supplies its second best (Q9)
            if not (Th[p] <= 0.0 or Th[p] < low):
                ok = False
            cand.append(I1[p])
            if I2[p] >= 0 and S[p] >= low:
                cand.append(I2[p])
        if not ok:
            uncertified[r] = True
            continue
        pmx, psec0, pidx = np.zeros(8, np.float32), np.float32(0), [-1] * 8
        for g in cand:
            for j in range(4):
                p2, sc, p = 4 * g + j, ex[r, 4 * g + j], g % 8
                nchains += 1
                if not sc > 0:
                    continue
                if sc > pmx[p]:
                    if p == 0: psec0 = pmx[0]
                    pmx[p], pidx[p] = sc, p2
                else:
                    if sc == pmx[p]: pidx[p] = min(pidx[p], p2)
                    if p == 0: psec0 = max(psec0, sc)
        mx, sec, idx = pmx[0], psec0, pidx[0]
        for y in range(8):                                        # matching.cu:378-390
            if idx != pidx[y]:
                if pmx[y] > mx: sec, mx, idx = max(mx, sec), pmx[y], pidx[y]
                elif pmx[y] > sec: sec = pmx[y]
        out["score"][r], out["match"][r] = mx, idx
        out["ambiguity"][r] = np.float32(sec) / (np.float32(mx) + np.float32(1e-6))
    return out, uncertified, nchains


def _check(s1, s2):
    got, unc, nchains = emulate(s1, s2)
    want = oracle.match(s1, s2, threads=4)
    ok = ~unc
    for f in ("score", "match", "ambiguity"):
        assert np.array_equal(got[f][ok], want[f][ok]), f
    return unc, nchains


def test_logic_random_sets():
    s1, s2 = synth_descriptors(384, 1), synth_descriptors(1000, 2)     # 1000 % 32 != 0: tail ignored (Q7)
    unc, nchains = _check(s1, s2)
    assert unc.mean() < 0.02
    assert nchains < 16 * len(s1)                                      # a handful of exact chains per row


def test_logic_flags_what_it_cannot_decide():
    s1, s2 = synth_descriptors(128, 21), synth_descriptors(640, 22)
    s2["data"][32] = s2["data"][0]; s2["data"][64] = s2["data"][0]     # three equal group maxima in partition 0
    s1["data"][:16] = s2["data"][0] * 0.999 + s1["data"][:16] * 0.001
    s1["data"][20] *= -1                                               # no positive score at all (Q11)
    s1["data"][21] = s2["data"][40]; s2["data"][7] = s2["data"][40]; s2["data"][33] = s2["data"][40]   # ties across partitions (Q10)
    unc, _ = _check(s1, s2)
    assert unc[:16].all() and unc[20]
    assert not unc[21]                                                 # duplicates in different partitions are decidable
