#!/usr/bin/env python
"""Pinned bytes of Poisson meshing: for a fixed set of point clouds, sha256 digests of the vertices, triangles, vertex
intensities and chi of cs_poisson_mesh and cs_poisson_mesh_screened, and their info and stats as they are.  The cases
cover the sphere, the torus and the open sheet at depths 5, 6 and 7 under both calls, intensities, trimming, status 1
(no usable point), status 2 (the Dirichlet call on the sheet), status 3 (one iteration), the screened call at point
weights 1, 4 and 16, and a depth-8 sphere of 1 M points.  The oracle tests compare to a tolerance and cannot see a
changed last bit; this file can.

Every case names its generator arguments (cloud, point count, seed, call arguments), so a replay needs nothing else.
Runs on a GPU with whatever library CUDASIFT_B200_LIB names (else the tree's own build):

  python tests/golden/make_mesh_pinned.py      -> tests/golden/mesh_pinned.npz

tests/test_mesh_pinned_gpu.py replays the stored cases and compares.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
OUT = os.path.join(ROOT, "tests", "golden", "mesh_pinned.npz")

INTENSITY = (np.array([0.5, -0.25, 0.75]), 2.0)      # a linear intensity field x . a + c


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def cloud(c):
    """The points, normals and intensities (or None) of a case."""
    import mesh_cases as mc
    import mesh_screened_cases as msc
    make = {"sphere": mc.sphere, "torus": mc.torus, "hemisphere": mc.hemisphere, "sheet": msc.sheet}[c["cloud"]]
    x, n = make(c["points"], seed=c["seed"])
    x, n = x.copy(), n.copy()
    if c.get("nan") == "all":
        x[:] = np.nan
    elif c.get("nan") == "some":                       # refused points among used ones
        x[::7, 1] = np.nan
        n[3::11] = 0.0
    inten = None
    if c.get("intensity"):
        a, c0 = INTENSITY
        inten = (x.astype(np.float64) @ a + c0).astype(np.float32)
    return x, n, inten


def run(cs, c):
    """The pinned outputs of one case: digests of the vertices, triangles, vertex intensities and chi, info and stats as
    they are."""
    x, n, inten = cloud(c)
    f = cs.PoissonMeshScreened if c["call"] == "screened" else cs.PoissonMesh
    verts, tris, vint, info, stats, chi, _ = f(x, n, inten, returnChi=True, **c["args"])
    return {"vertices": np.array(_sha(verts)), "triangles": np.array(_sha(tris)),
            "intensity": np.array("none" if vint is None else _sha(vint)), "chi": np.array(_sha(chi)),
            "info": np.asarray(info), "stats": np.asarray(stats)}


def cases():
    clouds = [dict(cloud="sphere", points=20000, seed=0), dict(cloud="torus", points=20000, seed=0),
              dict(cloud="sheet", points=40000, seed=1)]
    out = []
    for call in ("dirichlet", "screened"):
        out += [dict(call=call, args=dict(depth=d), **cl) for cl in clouds for d in (5, 6, 7)]
        out += [dict(call=call, cloud="sphere", points=40000, seed=5, intensity=True, args=dict(depth=6)),
                dict(call=call, cloud="sphere", points=20000, seed=6, args=dict(depth=6, maxIterations=1, tol=1e-9)),
                dict(call=call, cloud="sphere", points=1000, seed=2, nan="all", args=dict(depth=5)),
                dict(call=call, cloud="sphere", points=20000, seed=2, nan="some", args=dict(depth=5))]
    out += [dict(call="dirichlet", cloud="hemisphere", points=30000, seed=0, args=dict(depth=6, trim=0.5)),
            dict(call="dirichlet", cloud="sphere", points=20000, seed=6, intensity=True, args=dict(depth=5, trim=0.5)),
            dict(call="screened", cloud="sheet", points=40000, seed=1, intensity=True, args=dict(depth=6, trim=0.5))]
    out += [dict(call="screened", cloud="sheet", points=40000, seed=1, args=dict(depth=6, pointWeight=w))
            for w in (1.0, 4.0, 16.0)]
    out += [dict(call="screened", cloud="torus", points=20000, seed=0, args=dict(depth=5, pointWeight=w))
            for w in (1.0, 16.0)]
    out += [dict(call=call, cloud="sphere", points=1_000_000, seed=11, args=dict(depth=8))
            for call in ("dirichlet", "screened")]
    return out


def main():
    import cudasift_b200 as cs
    cs.InitCuda(0)
    cs_ = cases()
    out = {"cases": np.array(json.dumps(cs_))}
    for i, c in enumerate(cs_):
        for k, v in run(cs, c).items():
            out["c%d_%s" % (i, k)] = v
        print(i, c, "status", out["c%d_stats" % i][9], "iterations", out["c%d_stats" % i][2],
              "triangles", out["c%d_stats" % i][6], flush=True)
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
