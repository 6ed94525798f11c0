"""Local seam levelling (cs_level_texture_seams_local) on the GPU, on the two workloads of scripts/seam_bench.py (the
chain's scene from 8 views of 640 x 480 and the simplified sphere from 32 views of 1920 x 1080), each view given its
own gain, offset and radial falloff (vignetting) so that the seams carry steps the global call cannot remove, and
cs_level_texture_seams run first as a user would.  Per workload: the local call's event time (median of --reps calls
after one warm-up), the stage split (the library's CUDASIFT_MATCH_TIMING events, from a child process), the seam and
free texels and the CG iterations, and the solve's ms per iteration against the HBM bytes one iteration moves at
3.35 TB/s, per free texel:
  - q = A p: z, p_old and diag read (24 bytes), the neighbour codes (16), p and q written (16); the neighbours' z and
    p_old are the same arrays' words, counted once;
  - the update: x, p, r, q and diag read (40), x, r and z written (24);
  so 120 bytes per free texel and iteration.
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

from mesh_bench import HBM, card  # noqa: E402

STAGES = ("check", "seam edges", "domain", "seam texels", "strip", "solve", "output")
BYTES_PER_FREE_TEXEL = 120


def levelled():
    """Per workload: the mesh, TextureMesh's outputs for vignetted views and the global call's atlas."""
    import cudasift_b200 as cs
    from texture_bench import workloads
    out = []
    for name, imgs, Ks, Rs, ts, v, t in workloads():
        rng = np.random.default_rng(7)
        H, W = imgs[0].shape
        yy, xx = np.mgrid[0:H, 0:W]
        r2 = ((xx - W / 2) ** 2 + (yy - H / 2) ** 2) / ((W / 2) ** 2 + (H / 2) ** 2)
        gain, off, fall = (1 + rng.uniform(-0.2, 0.2, len(imgs)), rng.uniform(-20, 20, len(imgs)),
                           rng.uniform(0.1, 0.4, len(imgs)))
        imgs = [np.ascontiguousarray(im * g * (1 - f * r2) + o, np.float32) for im, g, o, f in zip(imgs, gain, off, fall)]
        atlas, uv, labels, charts = cs.TextureMesh(imgs, Ks, Rs, ts, v, t)[:4]
        glob = cs.LevelTextureSeams(v, t, atlas, uv, labels, charts)[0]
        out.append((name, v, t, glob, uv, labels, charts))
    return out


def child(reps, cases):
    import cudasift_b200 as cs
    for name, v, t, atlas, uv, labels, charts in cases:
        sys.stderr.write("workload %s\n" % name)
        sys.stderr.flush()
        for _ in range(reps):
            cs.LevelTextureSeamsLocal(v, t, atlas, uv, labels, charts)


def parse_split(text):
    out, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"workload (.+)$", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        m = re.match(r"seams local timing .*\[us\]:" + "".join(r" %s ([\d.]+)" % s for s in STAGES), line)
        if m and cur:
            out[cur].append([float(x) / 1e3 for x in m.groups()])
    return {k: np.median(np.array(x), 0).tolist() for k, x in out.items() if x}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--child", action="store_true")
    a = ap.parse_args()
    import cudasift_b200 as cs
    cs.InitCuda(0)
    cases = levelled()
    if a.child:
        child(a.reps, cases)
        return
    res = {"card": card(), "hbm_bytes_per_s": HBM, "workloads": []}
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    ch = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reps", "3"], env=env,
                        stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    split = parse_split(ch.stderr) if ch.returncode == 0 else {"error": ch.stderr[-400:]}
    for name, v, t, atlas, uv, labels, charts in cases:
        out = cs.LevelTextureSeamsLocal(v, t, atlas, uv, labels, charts)       # warm-up
        ms = []
        for _ in range(a.reps):
            out = cs.LevelTextureSeamsLocal(v, t, atlas, uv, labels, charts)
            ms.append(out[3])
        _, info, st, _ = out
        N, its = int(st[4]), int(st[6])
        per_it = BYTES_PER_FREE_TEXEL * N
        w = {"workload": name, "faces": len(t), "atlas_texels": int(atlas.size), "call_ms": float(np.median(ms)),
             "stats": [int(x) for x in st], "seam_texels": int(st[3]), "free_texels": N, "iterations": its,
             "info": [float(x) for x in info], "converged_within_1000": int(st[7]) == 0, "bytes_per_iteration": per_it,
             "bound_ms_per_iteration": per_it / HBM * 1e3}
        if name in split:
            w["stage_ms"] = dict(zip(STAGES, split[name]))
            if its:
                w["solve_ms_per_iteration"] = w["stage_ms"]["solve"] / its
                w["bound_share"] = w["bound_ms_per_iteration"] / w["solve_ms_per_iteration"]
        res["workloads"].append(w)
        sys.stderr.write(json.dumps(w) + "\n")
    if "error" in split:
        res["split_error"] = split["error"]
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
