"""Mesh texturing with belief propagation (cs_texture_mesh_bp) against cs_texture_mesh_photo on the GPU, on the two
workloads of scripts/texture_bench.py (the chain's scene and the simplified sphere from 32 views of 1920 x 1080).  Per
workload: both calls at their defaults timed alternately in one run (event time, median of --reps pairs after one
warm-up each), the labelling stage of each from the library's CUDASIFT_MATCH_TIMING events (a child process; for the
BP call it holds the BP and the ICM sweeps); E at the start, ICM's final E (the photo call), BP's kept E and the final E
of the BP call; charts and seam edges (adjacent seen faces with different labels) of both; the BP sweeps run, the
sweep kept and whether the messages converged; and a sweep of bpSweeps over 8, 16, 32, 64 and 128 (call time, kept
and final E, charts, seams), from which the default is chosen.  The card's name and power limit are read in the same
run.  One JSON line on stdout."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mesh_bench import card  # noqa: E402
from texture_bench import STAGES, workloads  # noqa: E402
from texture_photo_bench import parse_split  # noqa: E402

SWEEP = (8, 16, 32, 64, 128)


def calls(cs, bpSweeps=None):
    extra = {} if bpSweeps is None else {"bpSweeps": bpSweeps}
    return {"texture_mesh_photo": lambda *a: cs.TextureMeshPhoto(*a),
            "texture_mesh_bp": lambda *a: cs.TextureMeshBP(*a, **extra)}


def seams(labels, t):
    """Adjacent pairs of seen faces (once per shared edge) whose labels differ."""
    import texture_oracle as to
    nbr = to.adjacency(np.asarray(t, np.int64))
    f = np.repeat(np.arange(len(t)), 3)
    g = nbr.reshape(-1)
    ok = (g > f) & (labels[f] >= 0)
    ok &= labels[np.maximum(g, 0)] >= 0
    return int((ok & (labels[f] != labels[np.maximum(g, 0)])).sum())


def child(reps):
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, imgs, Ks, Rs, ts, v, t in workloads():
        for call, fn in calls(cs).items():
            sys.stderr.write("workload %s/%s\n" % (name, call))
            sys.stderr.flush()
            for _ in range(reps):
                fn(imgs, Ks, Rs, ts, v, t)


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
    res = {"card": card(), "workloads": []}
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    ch = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reps", "3"], env=env,
                        stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    split = parse_split(ch.stderr) if ch.returncode == 0 else {"error": ch.stderr[-400:]}
    for name, imgs, Ks, Rs, ts, v, t in workloads():
        fns = calls(cs)
        out = {k: fn(imgs, Ks, Rs, ts, v, t) for k, fn in fns.items()}        # warm-up
        ms = {k: [] for k in fns}
        for _ in range(a.reps):
            for k, fn in fns.items():
                out[k] = fn(imgs, Ks, Rs, ts, v, t)
                ms[k].append(out[k][6])
        ph, bp = out["texture_mesh_photo"], out["texture_mesh_bp"]
        st = bp[5]
        w = {"workload": name, "faces": len(t), "images": len(imgs), "colours": int(st[3]),
             "call_ms": {k: float(np.median(x)) for k, x in ms.items()},
             "E_start": float(ph[4][0]), "E_icm": float(ph[4][1]), "E_bp_kept": float(bp[4][2]),
             "E_final": float(bp[4][1]),
             "charts": {"texture_mesh_photo": len(ph[3]), "texture_mesh_bp": len(bp[3])},
             "seams": {"texture_mesh_photo": seams(ph[2], t), "texture_mesh_bp": seams(bp[2], t)},
             "icm_sweeps": {"texture_mesh_photo": int(ph[5][5]), "texture_mesh_bp": int(st[5])},
             "bp_sweeps": int(st[16]), "bp_kept_sweep": int(st[17]), "bp_converged": int(st[18]) == 0,
             "bp_messages_changed_last": int(st[18]), "bp_moved": int(st[19]),
             "labels_changed_vs_photo": int((ph[2] != bp[2]).sum())}
        stage = {k: dict(zip(STAGES, split[name + "/" + k])) for k in fns if name + "/" + k in split}
        if stage:
            w["stage_ms"] = stage
        sweep = []
        for s in SWEEP:
            f = calls(cs, s)["texture_mesh_bp"]
            f(imgs, Ks, Rs, ts, v, t)
            runs = [f(imgs, Ks, Rs, ts, v, t) for _ in range(3)]
            r = runs[-1]
            sweep.append({"bpSweeps": s, "call_ms": float(np.median([x[6] for x in runs])),
                          "E_bp_kept": float(r[4][2]), "E_final": float(r[4][1]), "charts": len(r[3]),
                          "seams": seams(r[2], t), "bp_sweeps": int(r[5][16]), "bp_kept_sweep": int(r[5][17]),
                          "bp_converged": int(r[5][18]) == 0})
        w["sweep"] = sweep
        res["workloads"].append(w)
        sys.stderr.write(json.dumps(w) + "\n")
    if "error" in split:
        res["split_error"] = split["error"]
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
