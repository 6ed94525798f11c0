"""Rotation averaging (cs_rotation_averaging) at 1DSfM's size: about 5 000 images and 300 000 edges.

Prints the card's name and power limit, then one JSON line: the device time per IRLS iteration and per CG iteration
(from two runs whose CG always runs to maxLinearIterations, 10 and 40: the difference over 30 iterations per IRLS
iteration), the host spanning tree's time, and a host arm, the same IRLS on the CPU with scipy.sparse.linalg.cg, per
iteration.  Then global positioning (cs_global_positioning) at triangulate_cases.collection's scale, 1 000 images and
about 1 M observations, split the same way into ms per LM iteration and per CG iteration.  Usage: python scripts/global_bench.py [--images 5000] [--neighbours 60] [--iters 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cudasift_b200 as cs  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import triangulate_cases as tc  # noqa: E402


def graph(seed, N, neighbours):
    """Random absolute rotations, each image joined to `neighbours` random others, relative rotations with 0.5 degree
    noise, 10 % of them random, weights 50..300 (15..60 for the random ones)."""
    rng = np.random.default_rng(seed)
    Rs = Rotation.random(N, random_state=seed).as_matrix()
    i = np.repeat(np.arange(N), neighbours)
    j = (i + rng.integers(1, N, len(i))) % N
    e = np.unique(np.stack([np.minimum(i, j), np.maximum(i, j)], 1), axis=0)
    noise = Rotation.from_rotvec(np.radians(0.5) * rng.normal(size=(len(e), 3))).as_matrix()
    Q = np.einsum("eab,ecb,ecd->ead", Rs[e[:, 1]], Rs[e[:, 0]], noise)
    bad = rng.random(len(e)) < 0.1
    Q[bad] = Rotation.random(int(bad.sum()), random_state=seed + 1).as_matrix()
    w = np.where(bad, rng.integers(15, 60, len(e)), rng.integers(50, 300, len(e))).astype(np.float64)
    return e.astype(np.int32), Q, w


def host_irls(N, e, Q, w0, R, iters, sigma, maxLinear, tol):
    """The same IRLS on the host: vectorised residuals, the Laplacian in CSR, scipy's CG per component block."""
    free = np.ones(N, bool)
    free[0] = False
    times = []
    for _ in range(iters):
        t0 = time.perf_counter()
        D = np.einsum("eba,ebc,ecd->ead", R[e[:, 1]], Q, R[e[:, 0]])
        rho = Rotation.from_matrix(D).as_rotvec()
        t2 = np.sum(rho * rho, 1)
        q = sigma * sigma / (t2 + sigma * sigma)
        w = w0 * q * q
        A = sp.coo_matrix((np.concatenate([w, w]), (np.concatenate([e[:, 0], e[:, 1]]),
                                                      np.concatenate([e[:, 1], e[:, 0]]))), shape=(N, N)).tocsr()
        L = (sp.diags(np.asarray(A.sum(1)).ravel()) - A).tocsr()[free][:, free]
        b = np.zeros((N, 3))
        np.add.at(b, e[:, 0], -w[:, None] * rho)
        np.add.at(b, e[:, 1], w[:, None] * rho)
        M = sp.diags(1.0 / L.diagonal())
        x = np.zeros((N, 3))
        for k in range(3):
            x[free, k], _ = spl.cg(L, b[free, k], rtol=tol, maxiter=maxLinear, M=M)
        R = np.einsum("nab,nbc->nac", R, Rotation.from_rotvec(x).as_matrix())
        times.append(time.perf_counter() - t0)
    return float(np.median(times)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--neighbours", type=int, default=60)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip())
    cs.InitCuda(0)
    e, Q, w = graph(1, a.images, a.neighbours)
    run = lambda lin: cs.RotationAveraging(a.images, e, Q, w, maxIterations=a.iters, maxLinearIterations=lin,
                                           linearTol=1e-15)
    dev = {}
    for lin in (10, 40):
        run(lin)                                                   # warm-up: module load, buffers
        ms = [run(lin) for _ in range(a.repeat)]
        dev[lin] = (float(np.median([m[6][1] for m in ms])), float(np.median([m[6][0] for m in ms])),
                    int(ms[0][5][3]), int(ms[0][5][4]))
    (t10, tree, it10, cg10), (t40, _, it40, cg40) = dev[10], dev[40]
    perCg = (t40 - t10) / (cg40 - cg10)
    perIt = t10 / it10
    R0 = run(10)[0]
    gm = cs.RotationAveraging(a.images, e, Q, w, maxIterations=0)[0]
    host = host_irls(a.images, e, Q, w, gm.copy(), 3, np.radians(5.0), 40, 1e-8)
    xy, Ks, Rs, ts, off, mem, _ = tc.collection(1, 143000)
    datas = []
    for p in xy:
        rec = np.zeros(len(p), cs.SIFT_DTYPE)
        rec["xpos"], rec["ypos"] = p[:, 0], p[:, 1]
        b = cs.DeviceBuffer(max(rec.nbytes, 8))
        b.upload(rec)
        datas.append(type("D", (), dict(d_data=b.ptr, numPts=len(p), buf=b))())
    gp = {}
    for lin in (10, 40):
        g = lambda: cs.GlobalPositioning(datas, Ks, Rs, off, mem, maxIterations=5, maxLinearIterations=lin,
                                         linearTol=1e-15)
        g()
        runs = [g() for _ in range(3)]
        gp[lin] = (float(np.median([r[5] for r in runs])), int(runs[0][4][6]), int(runs[0][4][7]), int(runs[0][4][3]))
    gpCg = (gp[40][0] - gp[10][0]) / (gp[40][2] - gp[10][2])
    print(json.dumps(dict(positioning_images=len(xy), positioning_observations=gp[10][3], positioning_ms_10cg=gp[10][0],
                          positioning_ms_40cg=gp[40][0], positioning_lm_iterations=gp[10][1],
                          positioning_ms_per_lm_iteration_10cg=gp[10][0] / gp[10][1],
                          positioning_ms_per_cg_iteration=gpCg)))
    print(json.dumps(dict(images=a.images, edges=len(e), device_ms_10cg=t10, device_ms_40cg=t40, irls_iterations=it10,
                          ms_per_irls_iteration_10cg=perIt, ms_per_cg_iteration=perCg, host_tree_ms=tree,
                          host_scipy_ms_per_irls_iteration_40cg=host, finite=bool(np.isfinite(R0).all()))))


if __name__ == "__main__":
    main()
