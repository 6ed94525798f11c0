#!/usr/bin/env python
"""Pinned bytes of geometric verification: for a fixed set of planted scenes, the model (E, R and t for the essential
call), the inlier count, a sha256 of the inlier list and every statistic of cs_verify_pairs / cs_verify_essential;
for one scene per model, sha256 digests of the slot models and counts of cs_verify_models /
cs_verify_essential_models and the five normalisation values.  The tolerance tests cannot see a changed last bit; this
file can.  Cases that reach both branches of the refit's keep rule (stats[6]) are found by a seed search and stored
with the rest.

Runs on a GPU with whatever library CUDASIFT_B200_LIB names (else the tree's own build):

  python tests/golden/make_verify_pinned.py      -> tests/golden/verify_pinned.npz

tests/test_verify_pinned_gpu.py replays the stored cases and compares.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "verify_pinned.npz")

H, F, E = 1, 2, 3                      # CS_GEOM_HOMOGRAPHY, CS_GEOM_FUNDAMENTAL, the essential call
THRESH = 2.0


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def scene(case):
    """(x1, x2 float32 [n, 2], pairs int32 [n, 2]) of a case."""
    if case["model"] == E:
        from test_essential_gpu import planted
        x1, x2, pairs = planted(max(case["n"], 200), case["scene_seed"], case["scene"], sigma=case["sigma"],
                                outliers=case["outliers"])[:3]
    else:
        from test_verify_gpu import planted
        x1, x2, pairs = planted(max(case["n"], 200), case["scene_seed"], case["scene"] == "plane", sigma=case["sigma"],
                                outliers=case["outliers"])[:3]
    return x1, x2, pairs[:case["n"]]


class _Dev:
    """Device copies of a case's records and pairs, and room for its inliers."""

    def __init__(self, cs, x1, x2, pairs):
        self.cs = cs
        r = []
        for xy in (x1, x2):
            rec = np.zeros(len(xy), cs.SIFT_DTYPE)
            rec["xpos"], rec["ypos"] = xy[:, 0], xy[:, 1]
            r.append(rec)
        self.n1, self.n2, self.k = len(x1), len(x2), len(pairs)
        self.b = [cs.DeviceBuffer(max(r[0].nbytes, 576)), cs.DeviceBuffer(max(r[1].nbytes, 576)),
                  cs.DeviceBuffer(max(8 * self.k, 8)), cs.DeviceBuffer(max(8 * self.k, 8))]
        self.b[0].upload(r[0])
        self.b[1].upload(r[1])
        if self.k:
            self.b[2].upload(np.ascontiguousarray(pairs, np.int32))

    def free(self):
        for b in self.b:
            b.free()


def _intrinsics():
    from test_essential_cpu import K1, K2
    return np.ascontiguousarray(K1, np.float64), np.ascontiguousarray(K2, np.float64)


def run(cs, case):
    """The pinned outputs of one single call: {model bytes, count, inlier digest, stats}."""
    L = cs.lib()
    d = _Dev(cs, *scene(case))
    try:
        if case["model"] == E:
            k1, k2 = _intrinsics()
            E_, R, t = np.zeros(9), np.zeros(9), np.zeros(3)
            m = L.cs_verify_essential(d.b[0].ptr, d.n1, d.b[1].ptr, d.n2, d.b[2].ptr, d.k, k1.ctypes.data,
                                      k2.ctypes.data, case["loops"], THRESH, case["seed"], E_.ctypes.data, R.ctypes.data,
                                      t.ctypes.data, d.b[3].ptr, d.k, None)
            assert m >= 0, L.cs_last_error()
            model = np.concatenate([E_, R, t])
            stats = np.array(cs.essential_stats(), np.int64)
        else:
            model = np.zeros(9)
            m = L.cs_verify_pairs(d.b[0].ptr, d.n1, d.b[1].ptr, d.n2, d.b[2].ptr, d.k, case["model"], case["loops"],
                                  THRESH, case["seed"], model.ctypes.data, d.b[3].ptr, d.k, None)
            assert m >= 0, L.cs_last_error()
            stats = np.array(cs.verify_stats(), np.int64)
        inl = d.b[3].download(np.int32, 2 * m) if m else np.zeros(0, np.int32)
    finally:
        d.free()
    return {"model": model.view(np.uint64), "count": np.int64(m), "inliers": np.array(_sha(inl)), "stats": stats}


def run_models(cs, case):
    """The pinned outputs of the models entry point: {slot digest, count digest, normalisation, valid pairs}."""
    L = cs.lib()
    per = 10 if case["model"] == E else 3
    M, C, N = np.zeros((per * case["loops"], 9)), np.zeros(per * case["loops"], np.int32), np.zeros(5)
    d = _Dev(cs, *scene(case))
    try:
        if case["model"] == E:
            k1, k2 = _intrinsics()
            v = L.cs_verify_essential_models(d.b[0].ptr, d.n1, d.b[1].ptr, d.n2, d.b[2].ptr, d.k, k1.ctypes.data,
                                             k2.ctypes.data, case["loops"], THRESH, case["seed"], M.ctypes.data,
                                             C.ctypes.data, N.ctypes.data)
        else:
            v = L.cs_verify_models(d.b[0].ptr, d.n1, d.b[1].ptr, d.n2, d.b[2].ptr, d.k, case["model"], case["loops"],
                                   THRESH, case["seed"], M.ctypes.data, C.ctypes.data, N.ctypes.data)
        assert v >= 0, L.cs_last_error()
    finally:
        d.free()
    return {"slots": np.array(_sha(M)), "counts": np.array(_sha(C)), "norm": N.view(np.uint64), "valid": np.int64(v)}


def _case(model, scene_, n, loops, seed=0, scene_seed=21, sigma=0.5, outliers=0.4):
    return {"model": model, "scene": scene_, "n": n, "loops": loops, "seed": seed, "scene_seed": scene_seed,
            "sigma": sigma, "outliers": outliers}


def fixed_cases():
    cases = []
    for model in (F, H):
        for scene_ in ("general", "plane"):
            for n in (1000, 5000):
                for loops in (1024, 4096):
                    cases.append(_case(model, scene_, n, loops, seed=n + loops))
    for motion in ("sideways", "forward"):
        for n in (1000, 5000):
            for loops in (1024, 4096):
                cases.append(_case(E, motion, n, loops, seed=n + loops))
    for model, n in ((H, 3), (F, 6), (E, 4)):                # fewer pairs than a sample: no winner, zero model
        cases.append(_case(model, "plane" if model == H else "general" if model == F else "sideways", n, 256))
    return cases


def keep_rule_cases(cs, tries=200):
    """Per model, the first seeds of a small noisy scene whose refit is kept (stats[6] = 1) and dropped (0)."""
    cases = []
    for model, scene_ in ((F, "general"), (H, "plane"), (E, "sideways")):
        found = {}
        for seed in range(tries):
            c = _case(model, scene_, 200, 32, seed=seed, scene_seed=1000 + seed, sigma=2.0, outliers=0.5)
            kept = int(run(cs, c)["stats"][6])
            if kept not in found:
                found[kept] = c
            if len(found) == 2:
                break
        print("keep rule, model %d: branches %s" % (model, sorted(found)))
        cases += [found[k] for k in sorted(found)]
    return cases


def models_cases():
    return [_case(F, "general", 1000, 256, seed=7), _case(H, "plane", 1000, 256, seed=7),
            _case(E, "sideways", 1000, 256, seed=7)]


def main():
    import cudasift_b200 as cs
    cs.InitCuda(0)
    cases = fixed_cases() + keep_rule_cases(cs)
    mcases = models_cases()
    out = {"cases": np.array(json.dumps(cases)), "models_cases": np.array(json.dumps(mcases))}
    for i, c in enumerate(cases):
        for k, v in run(cs, c).items():
            out["c%d_%s" % (i, k)] = v
    for i, c in enumerate(mcases):
        for k, v in run_models(cs, c).items():
            out["m%d_%s" % (i, k)] = v
    kept = {m: sorted({int(out["c%d_stats" % i][6]) for i, c in enumerate(cases) if c["model"] == m}) for m in (F, H, E)}
    out["kept_branches"] = np.array(json.dumps(kept))
    print("cases %d, models cases %d, refit kept branches per model %s" % (len(cases), len(mcases), kept))
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
