"""Poisson meshing (cs_poisson_mesh, or cs_poisson_mesh_screened with --screened) on the GPU: a sphere of about 1 M and 5 M points and the fused points of the
rendered dense scene, at depth 8 and 9.  Per workload: the call's event time (median of --reps calls after one warm-up),
the splat, solve and extraction split (the library's CUDASIFT_MATCH_TIMING events, from a child process), the CG
iterations, ms per MGPCG iteration (solve time over iterations; the solve also holds the set-up, the true residual and
tau) and the bytes one iteration must move at the HBM rate of 3.35 TB/s (bytes_per_iteration below).  The card's name
and power limit are read in the same run.  One JSON line on stdout."""
import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM = 3.35e12


def bytes_per_iteration(depth, points=0, screened=False):
    """Bytes one MGPCG iteration reads and writes once each (float32 words per node; neighbours assumed cached):
    q = A p (2), the x / r / z update (7), r.z (2), p = z + beta p (3); per level of the V-cycle 4 pre- and 4
    post-half-sweeps (3 each: x and f read, x written), the residual (3), the restriction (1 fine read, 2 coarse
    writes per coarse node) and the prolongation (2 fine, 1 coarse read).  Levels n = N, N / 2, ..., 16 (the smaller
    ones run in one CTA and are left out).  Screened: every half-sweep and the residual also read s (1 more each), A p
    reads the cell starts (1 per node), and the two point passes read g (24 bytes per used point) and write, then read,
    u (8 and 8)."""
    N = 1 << depth
    fine = 4 * (2 + 7 + 2 + 3 + (1 if screened else 0)) * (N + 1) ** 3
    n, lv = N, 0
    sweep = 4 if screened else 3
    while n > 16:
        nodes, coarse = (n + 1) ** 3, (n // 2 + 1) ** 3
        lv += 4 * ((8 * sweep + sweep + 1 + 2) * nodes + (2 + 1) * coarse)
        n //= 2
    return fine + lv + ((2 * 24 + 8 + 8) * points if screened else 0)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             stdout=subprocess.PIPE, text=True, timeout=60).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:                                  # reported, not hidden
        return {"error": str(e)}


def scene_points():
    import cudasift_b200 as cs
    import stereo_cases as sc
    Ks, Rs, ts, views = sc.render(8, 640, 480, seed=2, texels=96)
    images = [v[0] for v in views]
    jobs = [(a, [b for b in np.argsort([abs(b - a) for b in range(8)]) if b != a][:4], 3.0, 12.0) for a in range(8)]
    d, n, c, _, _ = cs.PatchMatchStereo(images, Ks, Rs, ts, jobs)
    dg, ng, cg, _, _ = cs.PatchMatchStereoGeometric(images, Ks, Rs, ts, jobs, d, n)
    xyz, nrm, inten, _, _, _ = cs.FuseDepthMaps(images, Ks, Rs, ts, jobs, dg, ng, cg)
    return xyz, nrm, inten


def workloads():
    import mesh_cases as mc
    s1 = mc.sphere(1_000_000, seed=11)
    s5 = mc.sphere(5_000_000, seed=12)
    sx, sn, si = scene_points()
    return [("sphere 1M", s1[0], s1[1], None, 8), ("sphere 5M", s5[0], s5[1], None, 9),
            ("scene", sx, sn, si, 8), ("scene", sx, sn, si, 9)]


def call(screened):
    import cudasift_b200 as cs
    return cs.PoissonMeshScreened if screened else cs.PoissonMesh


def child(reps, screened):
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, x, n, i, depth in workloads():
        sys.stderr.write("workload %s %d %d\n" % (name, depth, len(x)))
        sys.stderr.flush()
        for _ in range(reps):
            call(screened)(x, n, i, depth=depth)


def parse_split(text):
    out, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"workload (.+) (\d) (\d+)$", line)
        if m:
            cur = "%s d%s" % (m.group(1), m.group(2))
            out[cur] = []
        m = re.match(r"mesh timing .*\[us\]: splat ([\d.]+) solve ([\d.]+) extract ([\d.]+)", line)
        if m and cur:
            out[cur].append([float(v) / 1e3 for v in m.groups()])
    return {k: np.median(np.array(v), 0).tolist() for k, v in out.items() if v}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--child", action="store_true")
    ap.add_argument("--screened", action="store_true", help="cs_poisson_mesh_screened at its default point weight")
    a = ap.parse_args()
    if a.child:
        child(a.reps, a.screened)
        return
    import cudasift_b200 as cs
    cs.InitCuda(0)
    res = {"card": card(), "hbm_bytes_per_s": HBM, "screened": a.screened, "workloads": []}
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    ch = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reps", "3"]
                        + (["--screened"] if a.screened else []), env=env,
                        stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    split = parse_split(ch.stderr) if ch.returncode == 0 else {"error": ch.stderr[-400:]}
    for name, x, n, i, depth in workloads():
        out = call(a.screened)(x, n, i, depth=depth)                  # warm-up
        ms = []
        for _ in range(a.reps):
            out = call(a.screened)(x, n, i, depth=depth)
            ms.append(out[6])
        st = out[4]
        key = "%s d%d" % (name, depth)
        w = {"workload": key, "points": int(len(x)), "used": int(st[0]), "depth": depth, "call_ms": float(np.median(ms)),
             "cg_iterations": int(st[2]), "residual": float(out[3][6]), "vertices": int(st[5]),
             "triangles": int(st[6]), "status": int(st[9]),
             "bytes_per_iteration": bytes_per_iteration(depth, int(st[0]), a.screened)}
        w["hbm_ms_per_iteration"] = w["bytes_per_iteration"] / HBM * 1e3
        if key in split:
            w["splat_ms"], w["solve_ms"], w["extract_ms"] = split[key]
            if st[2] > 0:
                w["solve_ms_per_iteration"] = w["solve_ms"] / int(st[2])
                w["hbm_share"] = w["hbm_ms_per_iteration"] / w["solve_ms_per_iteration"]
        res["workloads"].append(w)
        sys.stderr.write(json.dumps(w) + "\n")
    if "error" in split:
        res["split_error"] = split["error"]
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
