#!/usr/bin/env python
"""Bundle adjustment (cs_bundle_adjust) on the GPU: call time, LM and CG iterations and costs on BAL-like synthetic
scenes and on the extracted six-view chain, with the default gauge.

  (a) the six-view chain of tests/bundle_cases.py chain(): extraction, matching, verification, tracks, then
      TriangulateTracks under about two pixels of pose error on views 2 to 5; adjusted over its inliers (use)
  (b) 50 cameras x 8 000 points x 32 000 observations (Ladybug-sized), tests/bundle_cases.py large(): cameras on a
      circle, each point seen by consecutive cameras of the path, 0.5 px noise, perturbed poses and points
  (c) 500 cameras x 200 000 points x 1 000 000 observations

The median of the call's event time over `--reps` calls after warm-up; the card's name and power limit are read in the
same run.  Phases inside the cooperative kernel are invisible to a profiler, so the time is split by differences of
calls: maxIterations = 0 (setup and evaluation), 1 LM iteration with 1 CG iteration, and 1 LM iteration with
--cg CG iterations (linearTol 1e-30 so that all of them run).  --host adds scipy.optimize.least_squares (TRF, LSMR,
jac_sparsity) on (a) and (b) over the same observations, parameters and gauge.  --refine MASK and --loss NAME add, for
every workload in the same run, the same measurements of BundleAdjustIntrinsics (cs_bundle_adjust_intrinsics) with that
refine mask (bit 0 focal, 1 k1, 2 k2), loss and --loss-scale, from the same start and k = 0, under the key
"<workload>_intrinsics".  Writes one JSON line (and --out FILE)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

WORKLOADS = {"b": (50, 8000, 4), "c": (500, 200000, 5)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception as e:
        return "unknown (%s)" % str(e)[:40]


class Data:
    def __init__(self, cs, xy):
        from cudasift_b200 import SIFT_DTYPE
        rec = np.zeros(max(len(xy), 1), SIFT_DTYPE)
        rec["xpos"][:len(xy)], rec["ypos"][:len(xy)] = xy[:, 0], xy[:, 1]
        self.buf = cs.DeviceBuffer(rec.nbytes)
        self.buf.upload(rec)
        self.d_data, self.numPts = self.buf.ptr, len(xy)


def workload(cs, name):
    """(the record sets, the scene as bundle_cases returns it, a function that frees the sets)."""
    import bundle_cases as bc
    if name == "a":
        c = bc.chain(cs)
        pts, _, _, inl, _, _ = cs.TriangulateTracks(c["datas"], c["K"], c["Rs"], c["ts0"], c["offsets"], c["members"],
                                                    numTrials=64, maxError=4.0, minTriAngle=0.5, seed=1)
        s = dict(xy=c["xy"], K=np.broadcast_to(c["K"], (6, 3, 3)), R0=c["Rs"], t0=c["ts0"], offsets=c["offsets"],
                 members=c["members"], X0=pts, use=inl, R=np.stack([np.eye(3)] * 6))
        return c["datas"], s, lambda: [cs.FreeSiftData(d) for d in c["datas"]]
    C, P, L = WORKLOADS[name]
    s = bc.large(200 + ord(name), C, P, perPoint=L)
    return [Data(cs, xy) for xy in s["xy"]], s, lambda: None


def run_gpu(name, reps, cg, intrinsics=None):
    """intrinsics None: BundleAdjust; else (refine, loss, lossScale) of BundleAdjustIntrinsics."""
    import cudasift_b200 as cs
    cs.InitCuda(0)
    datas, s, free = workload(cs, name)
    args = (datas, s["K"], s["R0"], s["t0"], s["offsets"], s["members"], s["X0"])
    use = dict(use=s["use"])
    if intrinsics:
        use.update(refine=intrinsics[0], loss=intrinsics[1], lossScale=intrinsics[2])

    def call(**kw):
        if intrinsics:
            return cs.BundleAdjustIntrinsics(*args, **kw)[2:]       # from R on: BundleAdjust's tuple
        return cs.BundleAdjust(*args, **kw)

    def timed(**kw):
        kw.update(use)
        for _ in range(2):
            out = call(**kw)
        ms = [call(**kw)[-1] for _ in range(reps)]
        return out, float(np.median(ms))
    full, ms_full = timed(maxIterations=20, maxLinearIterations=50, linearTol=1e-2)
    _, ms_eval = timed(maxIterations=0)
    _, ms_1 = timed(maxIterations=1, maxLinearIterations=1, linearTol=1e-30)
    _, ms_k = timed(maxIterations=1, maxLinearIterations=cg, linearTol=1e-30)
    free()
    R, t, X, err, inl, cost, trace, stats, _ = full
    return s, dict(cameras=len(datas), points=len(s["offsets"]) - 1, observations=int(stats[3]),
                ms_median=round(ms_full, 3),
                lm_iterations=int(stats[6]), cg_iterations=int(stats[7]), accepted=int((trace[:, 3] == 1).sum()),
                cost_initial=cost[0], cost_final=cost[1], ms_setup_eval=round(ms_eval, 3),
                ms_per_cg_iteration=round((ms_k - ms_1) / (cg - 1), 4), ms_lm_iteration_1cg=round(ms_1 - ms_eval, 3),
                rot_err_vs_truth_max=float(np.abs(R[2:] - s["R"][2:]).max()))


def host_arm(s):
    """scipy's TRF with LSMR and the Jacobian's sparsity on the same observations, residuals, parameters and gauge."""
    from scipy.optimize import least_squares
    from scipy.sparse import lil_matrix
    import bundle_cases as bc
    import bundle_oracle as bo
    pr = bo.Problem(s["xy"], s["K"], s["R0"], s["t0"], s["offsets"], s["members"], s["X0"], use=s["use"],
                    fixed=bc.gauge(s["t0"]))
    free = pr.mask
    nc = int(free.sum())
    col = -np.ones((pr.S, 6), np.int64)
    col[free] = np.arange(nc)
    pidx = np.zeros(pr.T, np.int64)
    pidx[pr.parts] = np.arange(len(pr.parts))                          # the adjusted points' variables
    A = lil_matrix((2 * pr.N, nc + 3 * len(pr.parts)), dtype=int)
    for o in range(pr.N):
        cs_ = col[pr.a[o]][col[pr.a[o]] >= 0]
        j = nc + 3 * pidx[pr.k[o]]
        for q in range(2):
            A[2 * o + q, cs_] = 1
            A[2 * o + q, j:j + 3] = 1

    def fun(v):
        dc = np.zeros((pr.S, 6))
        dc[free] = v[:nc]
        Rr, tt = pr.apply(pr.R0, pr.t0, free, dc)
        XX = pr.X0.copy()
        XX[pr.parts] += v[nc:].reshape(-1, 3)
        return pr.residuals(Rr, tt, XX)[0].reshape(-1)
    t0 = time.perf_counter()
    sol = least_squares(fun, np.zeros(nc + 3 * len(pr.parts)), jac_sparsity=A, method="trf", tr_solver="lsmr", x_scale="jac")
    return dict(host_s=round(time.perf_counter() - t0, 2), host_cost_final=float(sol.fun @ sol.fun),
                host_nfev=int(sol.nfev))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--workloads", default="abc")
    ap.add_argument("--cg", type=int, default=21)
    ap.add_argument("--host", action="store_true")
    ap.add_argument("--refine", type=int, default=None)
    ap.add_argument("--loss", default=None, choices=["trivial", "soft_l1", "cauchy"])
    ap.add_argument("--loss-scale", type=float, default=2.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(card=card())
    for w in a.workloads:
        s, res[w] = run_gpu(w, a.reps, a.cg)
        if a.host and w in "ab":
            res[w].update(host_arm(s))
        if a.refine is not None or a.loss is not None:
            mode = (3 if a.refine is None else a.refine, a.loss or "trivial", a.loss_scale)
            _, res[w + "_intrinsics"] = run_gpu(w, a.reps, a.cg, mode)
            res[w + "_intrinsics"].update(refine=mode[0], loss=mode[1], loss_scale=mode[2])
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
