"""Mesh texturing with Waechter et al.'s view selection (cs_texture_mesh_photo) against cs_texture_mesh on the GPU, on
the two workloads of scripts/texture_bench.py (the chain's scene from 8 views of 640 x 480 and the simplified sphere
from 32 views of 1920 x 1080), plain and with seam_bench's per-view gain and offset (where exposure differences must
not be taken for outliers).  Per workload: both calls timed alternately in one run (event time, median of --reps
pairs after one warm-up each), the candidate stage of each from the library's CUDASIFT_MATCH_TIMING events (a child
process; for the photo call it holds the sampling and the outlier kernels), the samples, centroid fallbacks, faces
tested, candidates removed and best candidates removed of the photo call at its defaults (GMI, K = 3, sigma_min = 4),
and the sampling stage against its HBM bound at 3.35 TB/s: every sampled box's keys (8 bytes per pixel) and pixels
(4 bytes per pixel) read once, with the boxes counted as the samples (a lower bound: pixels of a box that name other
faces are left out).  The Sobel taps are assumed to hit in cache.  Also the ptxas registers, stack and spills of the
two new kernels (nvcc -Xptxas -v on texture.cu with the library's flags).  The card's name and power limit are read
in the same run.  One JSON line on stdout."""
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
from texture_bench import STAGES, workloads  # noqa: E402

KERNELS = ("texture_photo_candidate_kernel", "texture_outlier_kernel")


def cases():
    """The workloads, then each again with seam_bench's per-view gain and offset."""
    out = []
    for name, imgs, Ks, Rs, ts, v, t in workloads():
        out.append((name, imgs, Ks, Rs, ts, v, t))
        rng = np.random.default_rng(7)
        gain, off = 1 + rng.uniform(-0.2, 0.2, len(imgs)), rng.uniform(-20, 20, len(imgs))
        out.append((name + " gain+offset", [np.ascontiguousarray(im * g + o, np.float32)
                                            for im, g, o in zip(imgs, gain, off)], Ks, Rs, ts, v, t))
    return out


def calls(cs):
    return {"texture_mesh": lambda *a: cs.TextureMesh(*a), "texture_mesh_photo": lambda *a: cs.TextureMeshPhoto(*a)}


def child(reps):
    import cudasift_b200 as cs
    cs.InitCuda(0)
    for name, imgs, Ks, Rs, ts, v, t in cases():
        for call, fn in calls(cs).items():
            sys.stderr.write("workload %s/%s\n" % (name, call))
            sys.stderr.flush()
            for _ in range(reps):
                fn(imgs, Ks, Rs, ts, v, t)


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


def ptxas():
    """Registers, stack and spills of the new kernels, from nvcc -Xptxas -v on texture.cu."""
    from cudasift_b200 import build
    nvcc = build.nvcc_path()
    if nvcc is None:
        return {"error": "no nvcc"}
    import tempfile
    src = os.path.join(ROOT, "cudasift_b200", "csrc", "texture.cu")
    flags = [f for f in build.NVCC_FLAGS if f != "-shared"] + build.UNIT_FLAGS.get("texture.cu", [])
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-I", os.path.join(ROOT, "include"), "-c", src, "-o",
                                             os.path.join(d, "t.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                           text=True, timeout=600)
    out, cur = {}, None
    for line in r.stdout.splitlines():
        if "Function properties for" in line:
            cur = next((k for k in KERNELS if re.search(r"\d%sE" % k, line)), None)
        if cur:
            m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m:
                out.setdefault(cur, {}).update(stack=int(m.group(1)), spill_stores=int(m.group(2)),
                                               spill_loads=int(m.group(3)))
            m = re.search(r"Used (\d+) registers", line)
            if m:
                out.setdefault(cur, {})["registers"] = int(m.group(1))
    return out or {"error": r.stdout[-400:]}


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
    res = {"card": card(), "hbm_bytes_per_s": HBM, "kernels": ptxas(), "workloads": []}
    env = dict(os.environ, CUDASIFT_MATCH_TIMING="1")
    ch = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reps", "3"], env=env,
                        stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=3000)
    split = parse_split(ch.stderr) if ch.returncode == 0 else {"error": ch.stderr[-400:]}
    fns = calls(cs)
    for name, imgs, Ks, Rs, ts, v, t in cases():
        out = {k: fn(imgs, Ks, Rs, ts, v, t) for k, fn in fns.items()}        # warm-up
        ms = {k: [] for k in fns}
        for _ in range(a.reps):
            for k, fn in fns.items():
                out[k] = fn(imgs, Ks, Rs, ts, v, t)
                ms[k].append(out[k][6])
        st = out["texture_mesh_photo"][5]
        base = out["texture_mesh"]
        sample_bytes = 12 * int(st[11])
        w = {"workload": name, "faces": len(t), "images": len(imgs),
             "call_ms": {k: float(np.median(x)) for k, x in ms.items()},
             "candidate_pairs": int(st[2]), "samples": int(st[11]), "fallbacks": int(st[12]),
             "faces_tested": int(st[13]), "removed": int(st[14]), "best_removed": int(st[15]),
             "unseen": {"texture_mesh": int(base[5][1]), "texture_mesh_photo": int(st[1])},
             "labels_changed_vs_texture_mesh": int((base[2] != out["texture_mesh_photo"][2]).sum()),
             "sampling_bound_bytes": sample_bytes, "sampling_bound_ms": sample_bytes / HBM * 1e3}
        w["call_ratio"] = w["call_ms"]["texture_mesh_photo"] / w["call_ms"]["texture_mesh"]
        stage = {k: dict(zip(STAGES, split[name + "/" + k])) for k in fns if name + "/" + k in split}
        if stage:
            w["stage_ms"] = stage
            cand = stage.get("texture_mesh_photo", {}).get("candidates")
            if cand:
                w["sampling_bound_share"] = w["sampling_bound_ms"] / cand
        res["workloads"].append(w)
        sys.stderr.write(json.dumps(w) + "\n")
    if "error" in split:
        res["split_error"] = split["error"]
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
