"""Mesh cleaning (cs_clean_mesh) on the GPU, at the defaults: the depth-9 PoissonMesh sphere (about 6.1 M triangles)
with holes of several sizes and islands added (tests/clean_cases.py's punch), and the fused points of the rendered
dense scene meshed by PoissonMeshScreened at depth 8, trim 0.5 and 1.0.  Per workload: the call's event time (median of
--reps calls after one warm-up), the per-stage counts, and the bytes the sorts and passes must move at the HBM rate of
3.35 TB/s (bytes_moved below), and the components and boundary edges before and after.  A
fourth workload times one 256-edge loop, the ear kernel's worst case.  The card's name and power limit are read in the same run.  One JSON line on stdout."""
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

STATS = ["input", "degenerate", "duplicate", "long_edge", "non_manifold_edge", "small_component", "components",
         "components_dropped", "non_manifold_vertices", "loops", "loops_filled", "loops_open", "half_edges_on_no_loop",
         "fill_faces", "vertices", "triangles", "vertices_written", "triangles_written", "status"]


def sort_bytes(n, key_bytes, bits):
    """A cub radix sort of n (key, 4-byte value) pairs over `bits` key bits: ceil(bits / 8) passes, each reading and
    writing every pair once."""
    return n * (key_bytes + 4) * 2 * ((bits + 7) // 8)


def bytes_moved(T, V):
    """Bytes the call must read and write once each at T input triangles and V vertices, as the defaults run it: the
    edge-key sort (3T pairs of 8-byte keys over 32 + vbits bits, read and written per pass) and rule 2's two sorts (T
    pairs over vbits and 32 + vbits bits); the triangles read by the edge keys and rule 2's three passes (4 x 12 per
    triangle) and the keys and corners written (36); the edge-run passes of rules 3 to 6 (five reads of the sorted keys
    and corners, 12 bytes per corner: 180 per triangle); the kept-face and output lists (12 read, 12 written, 12 read
    again per triangle); the vertex passes (24 read and 12 written per vertex, plus 3 x 4 bytes of flags)."""
    vbits = max(1, int(V - 1).bit_length()) if V > 1 else 1
    sorts = sort_bytes(3 * T, 8, 32 + vbits) + sort_bytes(T, 4, vbits) + sort_bytes(T, 8, 32 + vbits)
    return sorts + (48 + 36 + 180 + 36) * T + (24 + 12 + 12) * V


def run(name, v, t, reps, **kw):
    import clean_oracle as co
    import cudasift_b200 as cs
    cs.CleanMesh(v, t, **kw)
    times = []
    for _ in range(reps):
        gv, gt, _, info, stats, ms = cs.CleanMesh(v, t, **kw)
        times.append(ms)
    ms = float(np.median(times))
    b = bytes_moved(len(t), len(v))
    sizes = co.components(t)
    return {"workload": name, "triangles_in": int(len(t)), "call_ms": round(ms, 3), "bytes_moved": int(b),
            "hbm_bound_ms": round(b / HBM * 1e3, 3), "hbm_share": round(b / HBM / (ms * 1e-3), 3),
            "threshold": float(info[2]), "input": {"components": int(len(sizes)),
                                                   "components_under_50": int((sizes < 50).sum()),
                                                   "boundary_edges": co.topology(t)[0]},
            "output": {"components": int(len(co.components(gt))), "boundary_edges": co.topology(gt)[0]},
            "stats": dict(zip(STATS, (int(s) for s in stats)))}


def big_hole():
    """A 100 x 100 grid with a square hole of 64 x 64 cells: one loop of 256 edges, filled at maxHoleEdges 256 by one
    thread (the ear kernel's worst case)."""
    import clean_cases as cc
    v, t = cc.grid(100, drop=cc._cells(18, 18, 64))
    return v, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import clean_cases as cc
    import cudasift_b200 as cs
    import mesh_cases as mc
    cs.InitCuda(0)
    out = {"card": card(), "workloads": []}
    x, n = mc.sphere(3_000_000, seed=4)
    v, t, _, _, _, _, _ = cs.PoissonMesh(x, n, depth=9)
    pv, pt = cc.punch(v, t, seed=1, rings=200, faces=200, islands=5)
    out["workloads"].append(run("sphere depth 9 with holes and islands", pv, pt, args.reps))
    v, t = big_hole()
    out["workloads"].append(run("grid with one 256-edge hole", v, t, args.reps, maxHoleEdges=256))
    xyz, nrm, inten = scene_points()
    for trim in (0.5, 1.0):
        v, t, _, _, _, _, _ = cs.PoissonMeshScreened(xyz, nrm, inten, depth=8, trim=trim)
        out["workloads"].append(run("fused scene depth 8 trim %.1f" % trim, v, t, args.reps))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
