"""Mesh texturing (cs_texture_mesh) on the GPU: the chain's mesh (the rendered dense scene fused, screened-meshed at
depth 8 with trim 0.5 and simplified to 10 %, textured from its 8 views of 640 x 480) and a simplified sphere (PoissonMesh
at depth 8 to 10 %) seen by 32 views of 1920 x 1080.  Per workload: the call's event time (median of --reps calls after
one warm-up), the stage split (the library's CUDASIFT_MATCH_TIMING events, from a child process), and three stages
against their HBM bound at 3.35 TB/s (the bytes below, from the counts):
  - depth buffers: the buffers' fill (8 bytes per pixel written) and one atomic read-modify-write (16 bytes) per pixel
    of every image, as if each pixel were covered once;
  - candidates: per face its vertices and indices (48 bytes) and its list (96 bytes), and per candidate pair found the
    4 buffer gathers (a 32-byte sector each; rejected pairs are left out, so this is a lower bound);
  - atlas: every chart texel read and written (8 bytes) and the atlas cleared (4 bytes per texel).
The card's name and power limit are read in the same run.  One JSON line on stdout."""
import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mesh_bench import HBM, card, scene_points  # noqa: E402

STAGES = ("adjacency", "depth", "candidates", "labelling", "charts", "atlas")


def workloads():
    import cudasift_b200 as cs
    import mesh_cases as mc
    import stereo_cases as sc
    import texture_cases as tc
    from cudasift_b200 import synth
    Ks, Rs, ts, views = sc.render(8, 640, 480, seed=2, texels=96)
    xyz, nrm, inten = scene_points()
    v, t, vi, _, _, _, _ = cs.PoissonMeshScreened(xyz, nrm, inten, depth=8, trim=0.5)
    gv, gt, _, _, _, _ = cs.SimplifyMesh(v, t, vi, targetTriangles=len(t) // 10)
    out = [("scene", [w[0] for w in views], Ks, Rs, ts, gv, gt)]
    x, n = mc.sphere(1_000_000, seed=11)
    v, t, _, _, _, _, _ = cs.PoissonMesh(x, n, depth=8)
    gv, gt, _, _, _, _ = cs.SimplifyMesh(v, t, targetTriangles=len(t) // 10)
    Ks, Rs, ts = tc.ring_cameras(32, 1920, 1080, mc.CENTRE, 2.6, seed=5)
    base = synth.synth_image(1920, 1080, seed=9).astype(np.float32)
    imgs = [np.roll(base, 37 * a, axis=1) for a in range(32)]
    out.append(("sphere 32x1080p", imgs, Ks, Rs, ts, gv, gt))
    return out


def child(reps):
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, imgs, Ks, Rs, ts, v, t in workloads():
        sys.stderr.write("workload %s\n" % name)
        sys.stderr.flush()
        for _ in range(reps):
            cs.TextureMesh(imgs, Ks, Rs, ts, v, t)


def parse_split(text):
    out, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"workload (.+)$", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        m = re.match(r"texture timing .*\[us\]:" + "".join(r" %s ([\d.]+)" % s for s in STAGES), line)
        if m and cur:
            out[cur].append([float(v) / 1e3 for v in m.groups()])
    return {k: np.median(np.array(v), 0).tolist() for k, v in out.items() if v}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--child", action="store_true")
    a = ap.parse_args()
    if a.child:
        child(a.reps)
        return
    import cudasift_b200 as cs
    cs.InitCuda(0)
    res = {"card": card(), "hbm_bytes_per_s": HBM, "workloads": []}
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    ch = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reps", "3"], env=env,
                        stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    split = parse_split(ch.stderr) if ch.returncode == 0 else {"error": ch.stderr[-400:]}
    for name, imgs, Ks, Rs, ts, v, t in workloads():
        out = cs.TextureMesh(imgs, Ks, Rs, ts, v, t)                # warm-up
        ms = []
        for _ in range(a.reps):
            out = cs.TextureMesh(imgs, Ks, Rs, ts, v, t)
            ms.append(out[6])
        atlas, uv, labels, charts, info, st, _ = out
        pixels = int(sum(im.size for im in imgs))
        texels = int((charts[:, 3].astype(np.int64) * charts[:, 4]).sum())
        T = len(t)
        b = {"depth": 24 * pixels, "candidates": int(st[2]) * 4 * 32 + (48 + 96) * T,
             "atlas": 8 * texels + 4 * atlas.size}
        w = {"workload": name, "faces": T, "images": len(imgs), "pixels": pixels, "call_ms": float(np.median(ms)),
             "unseen": int(st[1]), "candidate_pairs": int(st[2]), "colours": int(st[3]), "rounds": int(st[4]),
             "sweeps": int(st[5]), "changed": int(st[6]), "charts": int(st[7]), "atlas_rows": int(st[8]),
             "status": int(st[10]), "chart_texels": texels, "energy": [float(info[0]), float(info[1])],
             "bound_bytes": b, "bound_ms": {k: x / HBM * 1e3 for k, x in b.items()}}
        if name in split:
            w["stage_ms"] = dict(zip(STAGES, split[name]))
            w["bound_share"] = {k: w["bound_ms"][k] / w["stage_ms"][k] for k in b if w["stage_ms"][k] > 0}
        res["workloads"].append(w)
        sys.stderr.write(json.dumps(w) + "\n")
    if "error" in split:
        res["split_error"] = split["error"]
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
