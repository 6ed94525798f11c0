"""The stage-timing lines of CUDASIFT_MATCH_TIMING=1: one mutual, knn, guided, ratio-batch, guided-batch, verify and
verify-batch call in a child process, every line in the common form "<header> [us]: name t name t ...", and each
benchmark script's parser returning every stage of its call."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

pytestmark = pytest.mark.gpu

T3 = ["prep", "gemm", "resolve", "exact-fallback", "reverse-gemm", "reverse-resolve", "reverse-exact-fallback", "pairs"]
GUIDED = ["prep", "index", "knn", "pairs"]
RATIO_BATCH = ["prep", "gemm", "resolve", "exact-fallback", "pairs"]
GUIDED_BATCH = ["prep", "index", "knn", "pairs"]
VERIFY = ["flags", "compact", "norm", "hyp", "score", "argmax", "refit", "write"]


def _mark(text):
    sys.stderr.write(text + "\n")
    sys.stderr.flush()


def _child():
    """The seven calls, each followed by the marker line its script's parser expects."""
    import cudasift_b200 as cs
    from cudasift_b200.synth import synth_descriptors

    cs.InitCuda(0)
    s1, s2 = synth_descriptors(512, 1), synth_descriptors(640, 2)
    H = np.eye(3)
    pairs = np.stack([np.arange(300), np.arange(300)], axis=1).astype(np.int32)
    cs.match_mutual_host(s1, s2, mode=2)
    _mark("size mutual")
    cs.match_ratio_host(s1, s2, crossCheck=True, mode=2)
    _mark("size knn")
    cs.match_guided_host(s1, s2, "homography", H, thresh=400.0)
    _mark("input guided")
    cs.verify_pairs_host(s1, s2, pairs, "fundamental", numLoops=256)
    _mark("input verify")

    datas = []
    for s in (s1, s2):
        d = cs.InitSiftData(cs.SiftData(), len(s))
        d._buf.upload(s)
        d.numPts = len(s)
        datas.append(d)
    _mark("call")
    cs.MatchSiftDataRatioBatch(datas, [(0, 1), (1, 0)])
    _mark("setting ratio-batch")
    _mark("call")
    cs.MatchSiftDataGuidedBatch(datas, [(0, 1), (1, 0)], "homography", [H, H], thresh=400.0)
    _mark("setting guided-batch")
    _mark("call")
    cs.VerifyPairsBatch([(datas[0], datas[1], pairs), (datas[1], datas[0], pairs, 7)], numLoops=256)
    _mark("setting verify-batch")
    for d in datas:
        cs.FreeSiftData(d)


@pytest.fixture(scope="module")
def stderr_text():
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stderr


def test_every_line_in_the_common_form(stderr_text):
    lines = [l for l in stderr_text.splitlines() if " timing " in l]
    headers = {l.split(" timing ")[0] for l in lines}
    assert headers == {"mutual", "knn", "guided", "verify", "ratio-batch", "guided-batch"}, headers
    for l in lines:
        assert re.fullmatch(r"[a-z-]+ timing [^\[]+ \[us\]:( [a-z-]+ \d+\.\d)+", l), l


def test_single_call_parsers(stderr_text):
    import guided_bench
    import knn_bench
    import mutual_bench
    import verify_bench
    assert list(mutual_bench.parse_split(stderr_text)["mutual"]) == T3
    assert list(knn_bench.parse_split(stderr_text)["knn"]["cross-check"]) == T3[:7]
    assert list(guided_bench.parse_split(stderr_text)["guided"]) == GUIDED
    assert list(verify_bench.parse_split(stderr_text)["verify"]) == VERIFY


def test_batch_parsers(stderr_text):
    import guided_batch_bench
    import match_batch_bench
    import verify_batch_bench
    for parse, name, stages in ((match_batch_bench.parse_split, "ratio-batch", RATIO_BATCH),
                                (guided_batch_bench.parse_split, "guided-batch", GUIDED_BATCH),
                                (verify_batch_bench.parse_split, "verify-batch", VERIFY)):
        split = parse(stderr_text)[name]
        assert split.pop("waves") == 1, (name, split)
        assert list(split) == stages, name


if __name__ == "__main__":
    _child()
