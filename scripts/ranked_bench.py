#!/usr/bin/env python
"""ranked_bench.py -- cost of ranked batch extraction (cs_extractor_create_ranked) against the plain extractor.

  python scripts/ranked_bench.py --steps K --warmup W [--repeats R]

Same protocol as bench.py: synthetic 1920x1080 float images resident in HBM, 2 extractors x batch 16, a step = the
rounds of bench.py's rule, device time from CUDA events on the extractors' streams.  The arms -- plain (maxPts 32768)
and ranked with N = 256, 1000, 32768 out of maxCandidates = 32768 -- are timed alternately in one process, R times
each.  Reported per arm: images/s (median and spread over the repeats), the e2e rate with host submits (H2D of the
images, D2H of the counts and of the records each slot returns), and for the ranked arms the ranking stage's device
time per image (events around it in one batch of 16).  The card's name and power limit are read in the same run.
One JSON line on stdout.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (W, H, synthetic images, step rule)

MAXC = 32768
STREAMS, BATCH = 2, 16


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:
        return {"error": str(e)[:80]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    args.batch, args.rounds = STREAMS * BATCH, 0
    import cudasift_b200 as cs
    cs.InitCuda(0)
    L = cs.lib()
    W, H = bench.W, bench.H
    pitch = cs.iAlignUp(W, 128)
    imgs = bench.make_images(0, 8)
    dbufs = []
    for i in range(args.batch):
        im = cs.CudaImage().Allocate(W, H, pitch, False, None, imgs[i % len(imgs)])
        im.Download()
        dbufs.append(im)
    ptrs = [d.d_data for d in dbufs]
    R = bench.rounds_per_step(args)

    arms = {"plain": None, "ranked_256": 256, "ranked_1000": 1000, "ranked_%d" % MAXC: MAXC}
    exs = {}
    for name, n in arms.items():
        exs[name] = [cs.Extractor(W, H, bench.OCTAVES, MAXC if n is None else n, False, batch=BATCH,
                                  maxCandidates=None if n is None else MAXC) for _ in range(STREAMS)]
        for s, ex in enumerate(exs[name]):                      # host images for the e2e leg
            for i in range(BATCH):
                hp = L.cs_extractor_host_image_at(ex.handle, i)
                ctypes.memmove(hp, imgs[(s * BATCH + i) % len(imgs)].ctypes.data, W * H * 4)
    ev0 = [L.cs_event_create() for _ in range(STREAMS)]
    ev1 = [L.cs_event_create() for _ in range(STREAMS)]

    def step(e):
        for _ in range(R):
            for s in range(STREAMS):
                e[s].submit_device_batch(ptrs[s * BATCH:(s + 1) * BATCH], pitch, bench.INIT_BLUR, bench.THRESH, 0.0)

    def timed(e):
        for _ in range(args.warmup):
            step(e)
        for x in e:
            x.wait_batch(BATCH)
        L.cs_device_sync()
        for s in range(STREAMS):
            L.cs_event_record(ev0[s], e[s].handle)
        for _ in range(args.steps):
            step(e)
        for s in range(STREAMS):
            L.cs_event_record(ev1[s], e[s].handle)
        counts = sum((x.wait_batch(BATCH) for x in e), [])
        ms = max(L.cs_event_elapsed_ms(ev0[0], ev1[s]) for s in range(STREAMS))
        return args.steps * R * args.batch / (ms / 1e3), counts

    def e2e(e, rounds):
        hp = [[L.cs_extractor_host_image_at(x.handle, i) for i in range(BATCH)] for x in e]
        d2h, busy = 0, [False] * STREAMS
        t0 = time.perf_counter()
        for _ in range(rounds):
            for s in range(STREAMS):
                if busy[s]:
                    d2h += sum(e[s].wait_batch(BATCH)) * bench.REC + 16 * BATCH
                e[s].submit_host_batch(hp[s], bench.INIT_BLUR, bench.THRESH, 0.0)
                busy[s] = True
        for s in range(STREAMS):
            d2h += sum(e[s].wait_batch(BATCH)) * bench.REC + 16 * BATCH
        dt = time.perf_counter() - t0
        return rounds * args.batch / dt, d2h / (rounds * args.batch)

    rates = {k: [] for k in arms}
    e2es = {k: [] for k in arms}
    counts, cands = {}, {}
    e2e_rounds = max(16, min(args.steps, 200) // 12)
    for rep in range(args.repeats):                              # arms alternate within every repeat
        for name in arms:
            v, c = timed(exs[name])
            rates[name].append(v)
            counts[name] = float(np.mean(c))
            cands[name] = float(np.mean([x.candidates(i) for x in exs[name] for i in range(BATCH)]))
            e2e(exs[name], 1)
            e2es[name].append(e2e(exs[name], e2e_rounds))

    rank_us = {}
    for name, n in arms.items():
        if n is None:
            continue
        per = []
        for i in range(10):
            _, ms = exs[name][0].profile_batch(ptrs[:BATCH], pitch, bench.INIT_BLUR, bench.THRESH, 0.0)
            if i >= 2:
                per.append((ms[4] - sum(ms[:4])) / BATCH * 1e3)
        rank_us[name] = round(float(np.median(per)), 3)
    pipe = []
    for i in range(10):
        _, ms = exs["plain"][0].profile_batch(ptrs[:BATCH], pitch, bench.INIT_BLUR, bench.THRESH, 0.0)
        if i >= 2:
            pipe.append(ms[4] / BATCH * 1e3)
    pipe_us = float(np.median(pipe))

    out = {"metric": "ranked vs plain batched extraction, 1920x1080, %d extractors x batch %d" % (STREAMS, BATCH),
           "card": card(), "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "rounds_per_step": R,
           "maxCandidates": MAXC, "plain_pipeline_us_per_image": round(pipe_us, 3), "arms": {}}
    for name, n in arms.items():
        r = rates[name]
        a = {"images_per_s_median": round(float(np.median(r)), 1), "images_per_s_min": round(min(r), 1),
             "images_per_s_max": round(max(r), 1), "records_per_image": round(counts[name], 1),
             "candidates_per_image": round(cands[name], 1),
             "e2e_images_per_s_median": round(float(np.median([x[0] for x in e2es[name]])), 1),
             "e2e_d2h_bytes_per_image": int(np.median([x[1] for x in e2es[name]]))}
        if n is not None:
            a["rank_stage_us_per_image"] = rank_us[name]
            a["rank_stage_share_of_plain_pipeline"] = round(rank_us[name] / pipe_us, 4)
        out["arms"][name] = a
    print(json.dumps(out), flush=True)
    for v in exs.values():
        for x in v:
            x.close()


if __name__ == "__main__":
    main()
