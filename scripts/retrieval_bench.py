"""Image retrieval on the GPU (cs_vocab_train, cs_vocab_assign, cs_retrieve_pairs) against host arms.

(a) training: the ranked features of synthetic 1080p images, numWords words, a fixed iteration count: time per
    iteration, the assignment's Gpair/s and the fallback rows; host arm scipy.cluster.vq.kmeans2 on the same data.
(b) assignment of the same descriptors against a larger vocabulary: time, Gpair/s, fallback rows.
(c) retrieval on seeded Zipf word lists: time, sum df^2, score updates per second; host arm scipy.sparse + argpartition.
Prints the card name and power limit, then one JSON line per measurement."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cudasift_b200 as cs                      # noqa: E402
from cudasift_b200.synth import synth_image      # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    return out.splitlines()[0] if out else "unknown"


def extract(n, maxPts):
    w, h = 1920, 1080
    pitch = cs.iAlignUp(w, 128)
    datas = []
    ex = cs.Extractor(w, h, 5, maxPts, False, batch=16, maxCandidates=32768)
    try:
        for b0 in range(0, n, 16):
            views = [synth_image(w, h, seed=5000 + k) for k in range(b0, min(n, b0 + 16))]
            cis = [cs.CudaImage().Allocate(w, h, pitch, False, None, v) for v in views]
            for ci in cis:
                ci.Download()
            ex.submit_device_batch([ci.d_data for ci in cis], pitch, 1.0, 3.0, 0.0)
            counts = ex.wait_batch(len(views))
            for i in range(len(views)):
                d = cs.InitSiftData(cs.SiftData(), int(counts[i]))
                d._buf.upload(ex.device_points_at(i, int(counts[i])))
                d.numPts = int(counts[i])
                datas.append(d)
    finally:
        ex.close()
    return datas


def zipf_lists(I, per, W, seed, a=1.0):
    rng = np.random.default_rng(seed)
    p = np.arange(1, W + 1, dtype=np.float64) ** -a
    p /= p.sum()
    words = rng.permutation(W)[rng.choice(W, I * per, p=p)].astype(np.int32)
    return np.full(I, per, np.int32), words


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--features", type=int, default=2000)
    ap.add_argument("--words", type=int, default=16384)
    ap.add_argument("--iterations", type=int, default=10)
    ap.add_argument("--assign-words", type=int, default=65536)
    ap.add_argument("--retrieve", type=int, nargs="*", default=[1000, 10000])
    ap.add_argument("--retrieve-words", type=int, default=65536)
    ap.add_argument("--host", action="store_true", help="also run the host arms")
    args = ap.parse_args()
    cs.InitCuda(0)
    print("card:", card(), flush=True)
    datas = extract(args.images, args.features)
    M = sum(d.numPts for d in datas)
    cs.TrainVocabulary(datas, args.words, 1)                        # warm-up
    vocab, trace, stats, ms = cs.TrainVocabulary(datas, args.words, args.iterations)
    it = int(stats[0])
    print(json.dumps({"bench": "train", "descriptors": M, "words": args.words, "iterations": it,
                      "ms_per_iteration": ms / it, "gpair_per_s": M * args.words * it / (ms * 1e-3) / 1e9,
                      "fallback_rows": trace[:, 2].tolist(), "empty_words": trace[:, 1].tolist()}), flush=True)
    if args.host:
        from scipy.cluster.vq import kmeans2
        X = np.concatenate([d._buf.download(cs.SIFT_DTYPE, d.numPts)["data"] for d in datas]).astype(np.float32)
        t0 = time.perf_counter()
        kmeans2(X, args.words, iter=args.iterations, minit="random", seed=0)
        print(json.dumps({"bench": "train_host_kmeans2", "s": time.perf_counter() - t0}), flush=True)
    cs.FreeSiftData(vocab)
    big, _, _, _ = cs.TrainVocabulary(datas, args.assign_words, 0)  # start words: a vocabulary of the right size
    cs.AssignWords(datas, big)
    wordOf, st, ms = cs.AssignWords(datas, big)
    print(json.dumps({"bench": "assign", "descriptors": M, "words": args.assign_words, "ms": ms,
                      "gpair_per_s": M * args.assign_words / (ms * 1e-3) / 1e9, "fallback_rows": int(st[2]),
                      "waves": int(st[4])}), flush=True)
    cs.FreeSiftData(big)
    for I in args.retrieve:
        sizes, words = zipf_lists(I, 2000, args.retrieve_words, I)
        cs.RetrievePairs(sizes, words, args.retrieve_words, topK=50)
        nb, sc, pairs, st, ms = cs.RetrievePairs(sizes, words, args.retrieve_words, topK=50)
        rec = {"bench": "retrieve", "images": I, "words_per_image": 2000, "vocabulary": args.retrieve_words, "ms": ms,
               "sum_df2": int(st[2]), "updates": int(st[3]), "updates_per_s": int(st[3]) / (ms * 1e-3),
               "waves": int(st[4]), "pairs": int(st[5])}
        print(json.dumps(rec), flush=True)
        if args.host and I <= 10000:
            import scipy.sparse as sp
            t0 = time.perf_counter()
            rows = np.repeat(np.arange(I), sizes)
            T = sp.csr_matrix((np.ones(len(words)), (rows, words)), shape=(I, args.retrieve_words))
            df = np.asarray((T > 0).sum(axis=0)).ravel()
            idf = np.log(I / np.maximum(df, 1))
            X = T.multiply(idf[None, :]).tocsr()
            n = np.sqrt(np.asarray(X.multiply(X).sum(axis=1)).ravel())
            X = sp.diags(1 / np.maximum(n, 1e-300)) @ X
            S = (X @ X.T).toarray()
            np.fill_diagonal(S, 0)
            np.argpartition(-S, 50, axis=1)[:, :50]
            print(json.dumps({"bench": "retrieve_host_scipy", "images": I, "s": time.perf_counter() - t0}), flush=True)


if __name__ == "__main__":
    main()
