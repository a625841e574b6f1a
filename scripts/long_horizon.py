#!/usr/bin/env python
"""Long-horizon configuration of BASELINE.json (600-frame sequences, 4 end-effectors, dense contact switches):
solve a batch on cuda:0 and report per-stage status / iterations / residuals, the wall time, the evaluation and
line-search kernel time per launch and the card's name and power limit.  Clips of any length run: past about 14 200
variables per sequence (e.g. --frames 1200 --sparse, or --frames 900) the evaluation and line-search kernels keep the
iterate in global memory instead of shared memory.

--stage3-long runs stage 3 on these sequences too (switch times as band unknowns, `PhysBatch(stage3_band_above=96)`);
--stage-times N then solves the stages once more, one by one for the whole batch with at most N iterations each, and
reports the KKT kernel time per launch of every stage."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_card():
    """name and power limit [W] of cuda:0 (nvidia-smi), None where it cannot be read"""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception:
        return {"gpu": None, "power_limit_w": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--frames", type=int, default=600)
    ap.add_argument("--n_ee", type=int, default=4)
    ap.add_argument("--sparse", action="store_true", help="walking gait instead of dense switches")
    ap.add_argument("--stage3-long", action="store_true", help="banded switch times: stage 3 beyond 96 phase durations")
    ap.add_argument("--stage-times", type=int, default=0, metavar="N",
                    help="extra pass: KKT kernel time per launch of every stage over its first N iterations")
    args = ap.parse_args()
    import chd
    problems = [chd.synth.make_problem(s, n_frames=args.frames, n_ee=args.n_ee, dense=not args.sparse) for s in range(args.batch)]
    band = 96 if args.stage3_long else None
    t0 = time.time()
    batch = chd.phys.PhysBatch(problems, stage3_band_above=band)
    batch.set_timing(True)
    t1 = time.time()
    out = batch.solve()
    t2 = time.time()
    d = batch.dims
    st, it = out["stage_status"], out["stage_iters"]
    per_stage = {}
    for name, s in chd.phys.STAGES.items():
        ran = st[s] != -9
        vals, cnts = np.unique(st[s], return_counts=True)
        per_stage[name] = {"status": {int(v): int(c) for v, c in zip(vals, cnts)},
                           "iters_min_median_max": [int(it[s][ran].min()), float(np.median(it[s][ran])), int(it[s][ran].max())]
                           if ran.any() else None}
    kt = batch.kernel_times()
    res = {
        "config": "%d x %d frames, %d ee, %s" % (args.batch, args.frames, args.n_ee, "walk" if args.sparse else "dense switches"),
        "stage3_band_above": band,
        "dims": {k: int(d[k]) for k in ("n_max", "m_max", "na_max", "nb_max", "w_max")},
        "sizes_fixed_nb_w_ndur": batch.sizes_fixed().tolist(),
        "create_s": t1 - t0, "solve_s": t2 - t1, "frames_per_s": args.batch * args.frames / (t2 - t1),
        "stage_status": st.tolist(), "stage_iters": it.tolist(), "per_stage": per_stage,
        "stage3_converged": float((st[4] == 0).mean()),
        "success": out["success"].tolist(), "launches": int(batch.launch_count()),
        "kernels": {k: list(v) for k, v in kt.items()},
        "eval_ms_per_launch": kt["eval"][0] / max(kt["eval"][1], 1),
        "linesearch_ms_per_launch": kt["linesearch"][0] / max(kt["linesearch"][1], 1),
        **gpu_card(),
    }
    if args.stage_times:
        batch.reset()
        batch.set_timing(True)
        kkt = {}
        for name in ("1.1", "1.2", "2.1", "2.2", "3"):
            batch.kernel_times(reset=True)
            r = batch.solve_stage(name, max_iter=args.stage_times)
            ms, n = batch.kernel_times()["kkt"]
            kkt[name] = {"kkt_ms_per_launch": ms / max(n, 1), "launches": n, "status": r["status"].tolist(),
                         "iters": r["iters"].tolist()}
        res["stage_by_stage"] = kkt
    print(json.dumps(res))


if __name__ == "__main__":
    main()
