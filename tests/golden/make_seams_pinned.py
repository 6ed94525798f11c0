#!/usr/bin/env python
"""Pinned bytes of seam levelling: for a fixed set of inputs, sha256 digests of the levelled atlas (and of the corner
offsets for cs_level_texture_seams) and info and stats as they are, for cs_level_texture_seams and
cs_level_texture_seams_local.  Both calls run every valid case of tests/seam_cases.py and its scale case, two invalid
cases (status 2), a one-label case (status 1), maxIterations = 1 (status 3), the ramp of test_seams_local_cpu
stretched past 2048 x 256 free texels with noise on its atlas, and the vignetted texture scene, flat and jittered; the
local call also runs at stripWidth 1 and 7 beside its default 20.  The oracle tests compare the solves to a bound and
cannot see a changed last bit; this file can.

The scene's inputs come from cs_texture_mesh, so their digests are stored too: a texturing change shows as a changed
input, not as a changed seams output.

Every case names its generator and call arguments, so a replay needs nothing else.  Runs on a GPU with whatever
library CUDASIFT_B200_LIB names (else the tree's own build):

  python tests/golden/make_seams_pinned.py      -> tests/golden/seams_pinned.npz

tests/test_seams_pinned_gpu.py replays the stored cases and compares.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "seams_pinned.npz")

LOCAL_ARGS = ("padding", "maxIterations", "tol")     # the seam_cases arguments the local call takes


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


_scenes = {}


def scene(jitter):
    """The vignetted texture scene of test_seams_local_gpu: TextureMesh's atlas, uv, labels and charts, and the global
    call's levelled atlas (the local call's input)."""
    if jitter not in _scenes:
        import cudasift_b200 as cs
        import texture_cases as tc
        from test_seams_local_cpu import vignetted
        imgs, Ks, Rs, ts, _ = tc.scene_views()
        v, t = tc.scene_mesh(jitter=jitter)
        atlas, uv, labels, charts = cs.TextureMesh(vignetted(imgs), Ks, Rs, ts, v, t)[:4]
        glob = cs.LevelTextureSeams(v, t, atlas, uv, labels, charts)[0]
        _scenes[jitter] = dict(v=v, t=t, labels=labels, uv=uv, charts=charts, atlas=atlas, glob=glob, kw={})
    return _scenes[jitter]


def inputs(c):
    """The vertices, triangles, labels, uv, charts and atlas of a case, and the seam_cases arguments it carries."""
    import seam_cases as sc
    g = c["gen"]
    if g == "ramp":
        from test_seams_local_cpu import ramp
        v, t, lab, uv, charts, atlas = ramp(c=32, L=420)
        atlas = atlas + np.random.default_rng(5).uniform(-10, 10, atlas.shape).astype(np.float32)
        d = dict(v=v, t=t, labels=lab, uv=uv, charts=charts, atlas=atlas, kw={})
    elif g == "scene":
        s = scene(c["jitter"])
        d = dict(s, atlas=s["glob"] if c["call"] == "local" else s["atlas"])
    else:
        d = dict(sc.scale() if g == "scale" else sc.CASES[g]())
    if c.get("one_label"):                        # every face of another label than the first seen face's unseen
        lab = np.asarray(d["labels"], np.int32)
        d["labels"] = np.where(lab == lab[lab >= 0][0], lab, -1).astype(np.int32)
    return d


def run(cs, c):
    """The pinned outputs of one case: info and stats as they are, digests of the levelled atlas (and the corner
    offsets) unless the input is invalid, and for the scene the digests of its inputs."""
    d = inputs(c)
    kw = dict(d["kw"])
    if c["call"] == "local":
        kw = {k: v for k, v in kw.items() if k in LOCAL_ARGS}
    kw.update(c["args"])
    args = (d["v"], d["t"], d["atlas"], d["uv"], d["labels"], d["charts"])
    out = {}
    if c["gen"] == "scene":
        out["inputs"] = np.array([_sha(np.asarray(a)) for a in args])
    if c["call"] == "global":
        atlas, corner, info, stats, _ = cs.LevelTextureSeams(*args, **kw)
    else:
        atlas, info, stats, _ = cs.LevelTextureSeamsLocal(*args, **kw)
    out.update({"info": np.asarray(info), "stats": np.asarray(stats)})
    if stats[7] != 2:                             # status 2 leaves the output buffers unwritten
        out["atlas"] = np.array(_sha(atlas))
        if c["call"] == "global":
            out["corner"] = np.array(_sha(corner))
    return out


def cases():
    import seam_cases as sc
    gens = sorted(n for n in sc.CASES if not n.startswith("invalid_")) + ["scale"]
    out = []
    for call in ("global", "local"):
        out += [dict(call=call, gen=g, args={}) for g in gens]
        out += [dict(call=call, gen=g, args={}) for g in ("invalid_gap", "invalid_nan_uv")]
        out += [dict(call=call, gen="solve_smoothness_0", one_label=True, args={}),
                dict(call=call, gen="ramp", args=dict(padding=0, maxIterations=50))]
        out += [dict(call=call, gen="scene", jitter=j, args={}) for j in (0.0, 0.3)]
        out += [dict(call=call, gen="scene", jitter=0.0, args=dict(maxIterations=1))]
    out += [dict(call="local", gen="scene", jitter=j, args=dict(stripWidth=w)) for j in (0.0, 0.3) for w in (1, 7)]
    return out


def main():
    import cudasift_b200 as cs
    cs.InitCuda(0)
    cs_ = cases()
    out = {"cases": np.array(json.dumps(cs_))}
    for i, c in enumerate(cs_):
        for k, v in run(cs, c).items():
            out["c%d_%s" % (i, k)] = v
        print(i, c, "status", out["c%d_stats" % i][7], "stats", list(out["c%d_stats" % i]), flush=True)
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
