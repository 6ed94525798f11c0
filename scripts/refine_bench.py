"""Photometric mesh refinement (cs_mesh_refine) on the GPU, three workloads on the scene of stereo_cases:
  (a) the jittered scene mesh (refine_cases.scene) seen by 8 views of 640 x 480;
  (b) the texture bench's chain mesh (the scene's points screened-meshed at depth 8, trim 0.5, simplified to 10 %) on
      the same views;
  (c) the jittered scene seen by 16 views of 1920 x 1080.
Per workload: the call's event time, evaluations and accepted steps, E_0 and E_final, the time per evaluation and its
split by kernel (torch.profiler: raster; the per-pair image passes map, score, pair total, image gradient; the face
gather; the vertex kernels), the image passes against their HBM bound at 3.35 TB/s (per pair and evaluation, bytes from
the shapes: map reads the key, writes J, c and a flag, 25 bytes per pixel plus the pair's four bilinear taps, 16;
score reads the window's flags, I and J once, 13, and writes 33; the image gradient reads 33 and writes 8), and the
RMS distance of the vertices to the nearest true rectangle before and after.  The card's name and power limit are read
in the same run.  One JSON line on stdout."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mesh_bench import HBM, card, scene_points  # noqa: E402

SMOOTH = 0.2                     # RefineMesh's default smoothness

GROUPS = {"raster": ("refine_raster",), "image_passes": ("refine_map", "refine_score", "refine_total", "refine_back"),
          "face_gather": ("refine_face",), "vertex": ("refine_thin", "refine_grad", "refine_step")}


def nearest_rms(v, rects):
    """The RMS distance of the points v to the nearest rectangle of the scene."""
    P = np.asarray(v, np.float64)
    best = np.full(len(P), np.inf)
    for r in rects:
        d = P - r["c"]
        du = np.clip(d @ r["u"], -r["hu"], r["hu"])
        dv = np.clip(d @ r["v"], -r["hv"], r["hv"])
        q = r["c"] + du[:, None] * r["u"] + dv[:, None] * r["v"]
        best = np.minimum(best, np.linalg.norm(P - q, axis=1))
    return float(np.sqrt(np.mean(best * best)))


def workloads():
    import cudasift_b200 as cs
    import refine_cases as rc
    a = rc.scene(n=8, width=640, height=480)
    out = [("a scene 8x640x480", a)]
    xyz, nrm, inten = scene_points()
    v, t, vi, _, _, _, _ = cs.PoissonMeshScreened(xyz, nrm, inten, depth=8, trim=0.5)
    gv, gt, _, _, _, _ = cs.SimplifyMesh(v, t, vi, targetTriangles=len(t) // 10)
    out.append(("b chain mesh 8x640x480", dict(a, v=gv, t=gt)))
    out.append(("c scene 16x1920x1080", rc.scene(n=16, width=1920, height=1080)))
    return out


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile
    import cudasift_b200 as cs
    cs.InitCuda(0)
    res = {"card": card(), "hbm_bytes_per_s": HBM, "workloads": []}
    for name, c in workloads():
        args = (c["imgs"], c["Ks"], c["Rs"], c["ts"], c["v"], c["t"], c["pairs"])
        cs.RefineMesh(*args, maxIterations=2)                          # warm-up
        out, info, st, ms = cs.RefineMesh(*args)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            cs.RefineMesh(*args)
            torch.cuda.synchronize()
        split = {k: 0.0 for k in GROUPS}
        for e in prof.key_averages():
            for k, names in GROUPS.items():
                if any(n in e.key for n in names):
                    split[k] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else \
                        e.cuda_time_total / 1e3
        ev = int(st[4])
        npairs = len(c["pairs"])
        pix = float(np.mean([c["imgs"][p[0]].size for p in c["pairs"]])) if npairs else 0.0
        bound_bytes = ev * npairs * pix * (25 + 16 + 13 + 33 + 33 + 8)
        passes_ms = split["image_passes"]
        w = {"workload": name, "faces": len(c["t"]), "vertices": len(c["v"]), "pairs": npairs, "call_ms": ms,
             "evaluations": ev, "accepted": int(st[5]), "free": int(st[1]), "P0": int(st[3]), "status": int(st[7]),
             "E0": float(info[0] + SMOOTH * info[1]), "E_final": float(info[2] + SMOOTH * info[3]), "info": info.tolist(),
             "ms_per_evaluation": ms / max(ev, 1), "stage_ms_per_evaluation": {k: x / max(ev, 1) for k, x in
                                                                               split.items()},
             "image_passes_bound_ms": bound_bytes / HBM * 1e3,
             "image_passes_bound_share": (bound_bytes / HBM * 1e3) / passes_ms if passes_ms > 0 else None,
             "rms_before": nearest_rms(c["v"], c["rects"]), "rms_after": nearest_rms(out, c["rects"])}
        res["workloads"].append(w)
        sys.stderr.write(json.dumps(w) + "\n")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
