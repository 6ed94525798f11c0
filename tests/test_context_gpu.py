"""GPU check of the per-device context: the matchers, the verifier and the ranking stage share one set of buffers per
device, grown on demand.  Calls of every kind and of three sizes are interleaved on one device, larger after smaller
and smaller after larger, and every output must be byte for byte what the same call gives alone in a fresh process.

Run as a script (`python test_context_gpu.py KIND SIZE OUT.npz`), this file makes one such call and saves its outputs."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

pytestmark = pytest.mark.gpu

# (n1, n2): "tiny" takes the exact paths in mode 0, the others the tensor-core paths
SIZES = {"tiny": (90, 70), "small": (300, 260), "large": (2600, 3100)}
KINDS = ("match", "mutual", "mutual_host", "knn2", "ratio", "ratio_host", "verify", "verify_host", "rank")
# the order of the interleaved run: every size follows a larger and a smaller one
ROUNDS = ("small", "large", "tiny", "large", "small")
H = np.array([[1.02, 0.03, 15.0], [-0.02, 0.98, -9.0], [1e-5, -2e-5, 1.0]])


def inputs(size):
    """Two record sets where half of set 1 has a noisy copy in set 2 (at a shuffled row, with its position mapped by H),
    and the pair list of those copies plus a quarter as many random pairs."""
    from cudasift_b200.synth import synth_descriptors
    n1, n2 = SIZES[size]
    rng = np.random.default_rng(n1 * 7 + n2)
    s1, s2 = synth_descriptors(n1, n1), synth_descriptors(n2, n2 + 1)
    s1["sharpness"] = rng.uniform(-30, 30, n1).astype(np.float32)
    m = min(n1, n2) // 2
    rows = rng.permutation(n2)[:m]
    d = s1["data"][:m] + rng.normal(0, 0.01, (m, 128)).astype(np.float32)
    s2["data"][rows] = d / np.linalg.norm(d, axis=1, keepdims=True)
    x = np.column_stack([s1["xpos"][:m], s1["ypos"][:m], np.ones(m)]) @ H.T
    s2["xpos"][rows] = (x[:, 0] / x[:, 2] + rng.normal(0, 0.5, m)).astype(np.float32)
    s2["ypos"][rows] = (x[:, 1] / x[:, 2] + rng.normal(0, 0.5, m)).astype(np.float32)
    k = m // 4
    pairs = np.vstack([np.column_stack([np.arange(m), rows]),
                       np.column_stack([rng.integers(0, n1, k), rng.integers(0, n2, k)])]).astype(np.int32)
    return s1, s2, pairs


def _device(cs, recs):
    d = cs.SiftData()
    cs.InitSiftData(d, len(recs), host=True)
    d._buf.upload(recs)
    d.numPts = len(recs)
    return d


def run(cs, kind, size):
    """One call; returns its outputs (results and the statistics it leaves) as a dict of arrays."""
    s1, s2, pairs = inputs(size)
    n1, n2 = len(s1), len(s2)
    out = {}
    if kind in ("match", "mutual", "ratio", "verify"):
        d1, d2 = _device(cs, s1), _device(cs, s2)
        if kind == "match":
            cs.MatchSiftData(d1, d2)
            out["host1"] = d1.h_data
        elif kind == "mutual":
            out["pairs"], _ = cs.MatchSiftDataMutual(d1, d2)
        elif kind == "ratio":
            out["pairs"], _ = cs.MatchSiftDataRatio(d1, d2)
        else:
            out["model"], out["inliers"], _ = cs.VerifyPairs(d1, d2, pairs, "fundamental", numLoops=1024)
        out["dev1"], out["dev2"] = d1._buf.download(cs.SIFT_DTYPE, n1), d2._buf.download(cs.SIFT_DTYPE, n2)
        cs.FreeSiftData(d1)
        cs.FreeSiftData(d2)
    elif kind == "mutual_host":
        out["rec1"], out["rec2"], out["pairs"], _ = cs.match_mutual_host(s1, s2)
    elif kind == "knn2":
        out["idx"], out["score"], _ = cs.match_knn2(s1, s2)
    elif kind == "ratio_host":
        out["pairs"], _ = cs.match_ratio_host(s1, s2, crossCheck=False)
    elif kind == "verify_host":
        out["model"], out["inliers"], _ = cs.verify_pairs_host(s1, s2, pairs, "homography", numLoops=1024)
    elif kind == "rank":
        out["ranked"] = cs.rank_records(s1, n1 // 3)
    if kind.startswith("verify"):
        out["stats"] = np.array(cs.verify_stats(), np.int64)
    elif kind != "rank":
        out["stats"] = np.array(cs.match_stats(), np.uint64)
    return {k: np.ascontiguousarray(v) for k, v in out.items()}


def alone(kind, size, tmp_path):
    """The same call as the only one of a fresh process."""
    path = str(tmp_path / ("%s_%s.npz" % (kind, size)))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), kind, size, path], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout
    with np.load(path) as f:
        return {k: f[k] for k in f.files}


def test_interleaved_calls_match_calls_alone(cs, tmp_path):
    got = {}
    for i, size in enumerate(ROUNDS):
        kinds = KINDS[i:] + KINDS[:i]                      # a different neighbour for every kind in every round
        for kind in kinds:
            got.setdefault((kind, size), []).append(run(cs, kind, size))
    for (kind, size), runs in got.items():
        want = alone(kind, size, tmp_path)
        if "pairs" in want:
            assert len(want["pairs"]) > min(SIZES[size]) // 4, (kind, size)     # the inputs do produce pairs
        if kind.startswith("verify"):
            assert len(want["inliers"]) > 0, (kind, size)
        for r in runs:
            assert sorted(r) == sorted(want), (kind, size)
            for k in want:
                assert r[k].dtype == want[k].dtype and r[k].shape == want[k].shape, (kind, size, k)
                assert r[k].tobytes() == want[k].tobytes(), (kind, size, k)


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    import cudasift_b200

    cudasift_b200.InitCuda(0)
    np.savez(sys.argv[3], **run(cudasift_b200, sys.argv[1], sys.argv[2]))
