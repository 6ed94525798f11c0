"""Mesh simplification (cs_simplify_mesh) on the GPU: the depth-9 PoissonMesh sphere (about 6.1 M triangles) reduced to
10 % and to 1 %, and the fused points of the rendered dense scene meshed by PoissonMeshScreened at depth 8 (trim 0.5)
reduced to 10 %.  Per workload: the call's event time (median of --reps calls after one warm-up), the passes, ms per
pass, and the bytes a pass must move at the HBM rate of 3.35 TB/s (bytes_per_pass below, from the counts).  The card's
name and power limit are read in the same run.  One JSON line on stdout."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mesh_bench import HBM, card, scene_points  # noqa: E402


def bytes_per_pass(T, V):
    """Bytes one pass reads and writes once each, at the mean triangle count T of the passes and V vertices: the
    candidate kernel reads the triangles and corner lists (12 + 12 bytes per triangle) and the float64 position,
    quadric and area of every vertex (112) and writes a key and a face count per corner (36 per triangle); the key sort
    (two passes over 8-byte keys, read and written: 96 per triangle); scatter and select read the keys (24 + 24) and
    write the selected keys and counts (36); the minimum keys (8 per vertex, set, scattered and read: 24); the face
    remap reads the triangles twice and the remap (36) and writes the next list (16); the corner keys and their sort
    (12 written, then 4 passes over 8-byte pairs: 96 per triangle)."""
    per_tri = 24 + 36 + 96 + 48 + 36 + 36 + 16 + 12 + 96
    return per_tri * T + (112 + 24) * V


def run(name, v, t, frac, reps):
    import cudasift_b200 as cs
    target = max(1, int(len(t) * frac))
    cs.SimplifyMesh(v, t, targetTriangles=target)
    times = []
    for _ in range(reps):
        gv, gt, _, info, stats, ms = cs.SimplifyMesh(v, t, targetTriangles=target)
        times.append(ms)
    ms = float(np.median(times))
    P = int(stats[2])
    meanT = (len(t) + len(gt)) / 2.0
    b = bytes_per_pass(meanT, len(v))
    per = ms / max(P, 1)
    return {"workload": name, "triangles_in": int(len(t)), "triangles_out": int(len(gt)), "status": int(stats[8]),
            "passes": P, "collapses": int(stats[3]), "frozen": int(stats[1]), "call_ms": round(ms, 2),
            "ms_per_pass": round(per, 3), "bytes_per_pass": int(b),
            "hbm_share": round(b / HBM / (per * 1e-3), 3), "max_error": float(info[0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import cudasift_b200 as cs
    import mesh_cases as mc
    cs.InitCuda(0)
    out = {"card": card(), "workloads": []}
    x, n = mc.sphere(3_000_000, seed=4)
    v, t, _, _, _, _, _ = cs.PoissonMesh(x, n, depth=9)
    for frac in (0.1, 0.01):
        out["workloads"].append(run("sphere depth 9 to %g" % frac, v, t, frac, args.reps))
    xyz, nrm, inten = scene_points()
    v, t, _, _, _, _, _ = cs.PoissonMeshScreened(xyz, nrm, inten, depth=8, trim=0.5)
    out["workloads"].append(run("fused scene depth 8 to 0.1", v, t, 0.1, args.reps))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
