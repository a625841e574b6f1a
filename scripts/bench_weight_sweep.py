#!/usr/bin/env python
"""Throughput of a cost-weight sweep: one synthetic clip (120 frames, 2 feet by default) under a grid of weight
settings, solved as one `PhysQueue` with per-clip weights (what scripts/weight_sweep.py runs) against one single-clip
`PhysBatch` per setting, one after the other.  The arms alternate `--reps` times in one process after a warm-up of each;
wall time covers creation and solve (host clock around synchronised work).  Prints one JSON line with frames/s of
both arms, the card and its power limit, and each setting's stage statuses and iterations in both arms."""
import argparse
import itertools
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--n_ee", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--slots", type=int, default=64)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    import chd
    p = chd.synth.make_problem(args.seed, n_frames=args.frames, n_ee=args.n_ee)
    # 4 x 4 x 4 = 64 settings around the defaults (0.4, 1.7, 0.3, 0.1, 0.1)
    grid = [(0.4, wa, we, 0.1, wd) for wa, we, wd in itertools.product((0.5, 1.0, 1.7, 3.0), (0.1, 0.3, 1.0, 3.0),
                                                                        (0.01, 0.1, 0.3, 1.0))]
    n = len(grid)

    def queue():
        q = chd.phys.PhysQueue([p] * n, args.slots, weights=grid)
        out = q.solve(cost_terms=True)
        q.close()
        return out

    def singles():
        st, it = np.zeros((6, n), np.int32), np.zeros((6, n), np.int32)
        for k, w in enumerate(grid):
            b = chd.phys.PhysBatch([p], weights=w)
            r = b.solve()
            b.close()
            st[:, k], it[:, k] = r["stage_status"][:, 0], r["stage_iters"][:, 0]
        return dict(stage_status=st, stage_iters=it)

    arms = dict(queue=queue, singles=singles)
    queue()                                                           # warm-up of both arms
    chd.phys.PhysBatch([p], weights=grid[0]).solve()
    times = {k: [] for k in arms}
    res = {}
    for _ in range(args.reps):
        for k, f in arms.items():
            t0 = time.perf_counter()
            res[k] = f()
            times[k].append(time.perf_counter() - t0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    frames = n * args.frames
    q, s = res["queue"], res["singles"]
    out = dict(gpu=gpu, settings=n, frames_per_setting=args.frames, n_ee=args.n_ee, slots=args.slots,
               queue_fps=[frames / t for t in times["queue"]], singles_fps=[frames / t for t in times["singles"]],
               queue_s=times["queue"], singles_s=times["singles"],
               same_status_1_to_22=int((q["stage_status"][:4] == s["stage_status"][:4]).all(axis=0).sum()),
               same_iters_1_to_22=int((q["stage_iters"][:4] == s["stage_iters"][:4]).all(axis=0).sum()),
               same_status_all=int((q["stage_status"] == s["stage_status"]).all(axis=0).sum()),
               per_setting=[dict(weights=w, queue_status=q["stage_status"][:, k].tolist(),
                                 queue_iters=q["stage_iters"][:, k].tolist(),
                                 singles_status=s["stage_status"][:, k].tolist(),
                                 singles_iters=s["stage_iters"][:, k].tolist(),
                                 cost_terms=q["cost_terms"][k].tolist()) for k, w in enumerate(grid)])
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
