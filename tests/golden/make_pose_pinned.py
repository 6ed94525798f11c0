#!/usr/bin/env python
"""Pinned bytes of absolute pose: for a fixed set of scenes, the pose (R, t), the count, every statistic and sha256
digests of the per-feature errors and inlier bytes of cs_absolute_pose_batch, for single jobs and for one mixed batch
(empty jobs, invalid pointOf entries, NaN points and positions, too few correspondences) with and without per-feature
outputs; for single jobs, a sha256 digest of every slot's pose and the slot counts of cs_absolute_pose_models.  The
oracle tests compare poses to a tolerance and cannot see a changed last bit; this file can.  Cases that reach both
branches of the refinement's keep rule (stats[6]) are found by a seed search and stored with the rest.

Runs on a GPU with whatever library CUDASIFT_B200_LIB names (else the tree's own build):

  python tests/golden/make_pose_pinned.py      -> tests/golden/pose_pinned.npz

tests/test_pose_pinned_gpu.py replays the stored cases and compares.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "pose_pinned.npz")


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def scene(case):
    """(xys, pointOfs, points, Ks) of a case: pose_cases.batch of its sizes, the jobs listed in empty cut to no records;
    with invalid, every job of at least 20 records gets 3 out-of-range pointOf entries, 2 naming a NaN point and 2 NaN
    positions."""
    import pose_cases as pc
    xys, pofs, pts, Ks, _, _ = pc.batch(case["scene_seed"], case["sizes"], noise=case["noise"])
    for p in case["empty"]:
        xys[p], pofs[p] = xys[p][:0], pofs[p][:0]
    if case["invalid"]:
        nan_point = len(pts)
        pts = np.concatenate([pts, [[np.nan, 0.0, 0.0]]])
        for xy, pof in zip(xys, pofs):
            if len(xy) >= 20:
                pof[:3] = 10 ** 6
                pof[3:5] = nan_point
                xy[5:7, 0] = np.nan
    return xys, pofs, pts, Ks


def _batch(cs, case):
    from test_pose_gpu import Batch
    xys, pofs, pts, Ks = scene(case)
    return Batch(cs, xys, pofs, pts), Ks


def run(cs, case):
    """The pinned outputs of one batch call: {posed jobs, R and t bytes, counts, stats, error and inlier digests}."""
    b, Ks = _batch(cs, case)
    seeds = np.arange(len(case["sizes"])) * 7 + case["seed"]
    try:
        r, R, t, counts, errors, inlier, stats, _ = b.run(Ks, case["loops"], case["maxError"], seeds,
                                                         outputs=case["outputs"])
    finally:
        b.free()
    out = {"posed": np.int64(r), "R": R.view(np.uint64), "t": t.view(np.uint64), "counts": counts, "stats": stats}
    if case["outputs"]:
        out["errors"] = np.array([_sha(e) for e in errors])
        out["inlier"] = np.array([_sha(i.view(np.uint8)) for i in inlier])
    return out


def run_models(cs, case):
    """The pinned outputs of cs_absolute_pose_models for the case's first job: {slot digest, slot counts, valid}."""
    b, Ks = _batch(cs, case)
    try:
        V, R, t, c = b.models(0, Ks[0], case["loops"], case["maxError"], case["seed"])
        assert V >= 0, cs.lib().cs_last_error()
    finally:
        b.free()
    return {"slots": np.array(_sha(np.concatenate([R.ravel(), t.ravel()]))), "counts": c, "valid": np.int64(V)}


def _case(sizes, loops, maxError=4.0, seed=0, scene_seed=21, noise=0.5, invalid=False, outputs=True, empty=()):
    return {"sizes": sizes, "loops": loops, "maxError": maxError, "seed": seed, "scene_seed": scene_seed,
            "noise": noise, "invalid": invalid, "outputs": outputs, "empty": list(empty)}


def fixed_cases():
    cases = []
    for k, (n, loops, err) in enumerate(((30, 256, 4.0), (200, 1024, 4.0), (1000, 256, 2.0), (5000, 1024, 4.0),
                                         (600, 64, 8.0))):
        cases.append(_case([n], loops, err, seed=n + loops, scene_seed=50 + k))
    # job 0 has no records, job 5 only records without a point
    mixed = [0, 2, 40, 3, 600, 0, 2000, 7, 150]
    cases.append(_case(mixed, 256, seed=3, scene_seed=60, invalid=True, empty=[0]))
    cases.append(_case(mixed, 256, seed=3, scene_seed=60, invalid=True, outputs=False, empty=[0]))
    return cases


def keep_rule_cases(cs, tries=200):
    """The first seeds of a small noisy scene whose refinement is kept (stats[6] = 1) and dropped (0)."""
    found = {}
    for seed in range(tries):
        c = _case([40], 32, 2.0, seed=seed, scene_seed=1000 + seed, noise=1.5)
        st = run(cs, c)["stats"][0]
        if st[5] >= 3 and int(st[6]) not in found:
            found[int(st[6])] = c
        if len(found) == 2:
            break
    print("keep rule: branches %s" % sorted(found))
    return [found[k] for k in sorted(found)]


def models_cases():
    return [_case([40], 64, seed=7, scene_seed=70), _case([600], 128, seed=8, scene_seed=71),
            _case([2000], 96, 2.0, seed=9, scene_seed=72, invalid=True)]


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
    kept = sorted({int(out["c%d_stats" % i][p][6]) for i, c in enumerate(cases) for p in range(len(c["sizes"]))
                   if out["c%d_stats" % i][p][5] >= 3})
    out["kept_branches"] = np.array(json.dumps(kept))
    print("cases %d, models cases %d, refinement kept branches %s" % (len(cases), len(mcases), kept))
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
