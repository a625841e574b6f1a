#!/usr/bin/env python
"""Cost-weight sweep of the physics solve: one or more clip directories (phys_optim's four input files each) x the
Cartesian grid of the comma separated `--w_*` values, every (clip, setting) pair solved as one clip of a single
`chd.phys.PhysQueue` with its own weights.  For every pair it writes one row (JSON or CSV, by the extension of
`--results`): the clip, the setting, the stage statuses and iterations, the success flags, the ten unweighted cost terms
(`chd.phys.COST_TERMS`) of the final iterate and its scaled NLP error and unscaled constraint violation.  With
`--out_dir` it also writes phys_optim's four output files of every pair to <out_dir>/<clip name>/setting_<k>/.  `--tol`
and `--last_stage` (`chd.phys.SolverOptions`) apply to every pair: a looser tolerance, or a sweep that stops after
stage 2.2 (`--last_stage dynamics`, which writes only the solution files of the snapshots taken), is a cheaper preview.

    python scripts/weight_sweep.py --in_dir clip --nframes 120 --n_ee 2 --w_ee 0.1,0.3,1 --w_dur 0.1,1 \\
        --results sweep.csv --slots 64
"""
import argparse
import csv
import itertools
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from phys_optim import WEIGHT_DEFAULTS, WEIGHT_FLAGS  # noqa: E402


def weight_grid(args):
    """Every setting of the sweep: the Cartesian product of the `--w_*` value lists, in flag order (the last flag
    varies fastest)."""
    return list(itertools.product(*[[float(x) for x in str(getattr(args, k)).split(",")] for k in WEIGHT_FLAGS]))


def sweep_options(args):
    """The `SolverOptions` of every setting, None when neither `--tol` nor `--last_stage` is set (the defaults)."""
    import chd
    kw = {k: getattr(args, k) for k in ("tol", "last_stage") if getattr(args, k, None) is not None}
    return chd.phys.SolverOptions(**kw) if kw else None


def final_stage(stage_status):
    """Stage id whose iterate is the final one: the last stage that ran (stage 4 when it ran after stage 3, or the
    clip's last_stage)."""
    return max(s for s in range(6) if stage_status[s] != -9)


def sweep_rows(out, clips, grid):
    """One dict per (clip, setting) pair of a `PhysQueue.solve(cost_terms=True)` result over `len(clips) * len(grid)`
    problems, clip major."""
    import chd
    names = {v: k for k, v in chd.phys.STAGES.items()}
    rows = []
    for c, clip in enumerate(clips):
        for k, w in enumerate(grid):
            i = c * len(grid) + k
            st = out["stage_status"][:, i]
            fin = final_stage(st)
            row = dict(clip=clip, setting=k, **{f: w[j] for j, f in enumerate(WEIGHT_FLAGS)})
            for s in range(6):
                row["status_" + names[s]] = int(st[s])
                row["iters_" + names[s]] = int(out["stage_iters"][s, i])
            row["dynamics_succeed"], row["durations_succeed"] = (int(v) for v in out["success"][i])
            row.update({t: float(out["cost_terms"][i, j]) for j, t in enumerate(chd.phys.COST_TERMS)})
            row["final_stage"] = names[fin]
            row["final_error"] = float(out["stage_stats"][fin, i, 1])
            row["final_constr_viol"] = float(out["stage_stats"][fin, i, 2])
            rows.append(row)
    return rows


def write_rows(path, rows):
    if path.endswith(".csv"):
        with open(path, "w", newline="") as f:
            w = csv.DictWriter(f, fieldnames=list(rows[0]))
            w.writeheader()
            w.writerows(rows)
    else:
        with open(path, "w") as f:
            json.dump(rows, f, indent=1)


def main(argv=None):
    ap = argparse.ArgumentParser(allow_abbrev=False)
    ap.add_argument("--in_dir", required=True, help="clip directories, comma separated")
    ap.add_argument("--nframes", default="100", help="one value, or one per clip")
    ap.add_argument("--n_ee", type=int, default=4)
    for k, v in zip(WEIGHT_FLAGS, WEIGHT_DEFAULTS):
        ap.add_argument("--" + k, default=v, help="values of the grid (comma separated)")
    ap.add_argument("--slots", type=int, default=64, help="device slots of the queue")
    ap.add_argument("--results", default="sweep.json", help="rows of the sweep: .json or .csv")
    ap.add_argument("--out_dir", default=None, help="also write phys_optim's four files of every (clip, setting)")
    ap.add_argument("--stage3_long", action="store_true",
                    help="run stage 3 on sequences with more than 96 phase durations too (switch times as band unknowns)")
    ap.add_argument("--tol", type=float, default=None, help="IPOPT's tol of every setting (default 1e-3)")
    ap.add_argument("--last_stage", default=None, help="no_dynamics, dynamics or durations (the default) for every setting")
    args = ap.parse_args(argv)
    import chd
    in_dirs = args.in_dir.split(",")
    nframes = [int(x) for x in str(args.nframes).split(",")]
    if len(nframes) == 1:
        nframes = nframes * len(in_dirs)
    if len(nframes) != len(in_dirs):
        raise ValueError("--nframes: %d values for %d clips" % (len(nframes), len(in_dirs)))
    grid = weight_grid(args)
    clips = [chd.io_formats.read_phys_inputs(d, f, n_ee=args.n_ee) for d, f in zip(in_dirs, nframes)]
    problems = [p for p in clips for _ in grid]
    weights = [w for _ in clips for w in grid]
    t0 = time.perf_counter()
    options = sweep_options(args)
    q = chd.phys.PhysQueue(problems, args.slots, weights=weights, stage3_band_above=96 if args.stage3_long else None,
                           options=options)
    out = q.solve(cost_terms=True)
    q.close()
    wall = time.perf_counter() - t0
    rows = sweep_rows(out, in_dirs, grid)
    write_rows(args.results, rows)
    if args.out_dir:
        ne_max = max(p.n_ee for p in clips)
        for i, (r, p) in enumerate(zip(rows, problems)):
            d = os.path.join(args.out_dir, os.path.basename(os.path.normpath(r["clip"])), "setting_%d" % r["setting"])
            os.makedirs(d, exist_ok=True)
            chd.phys.write_outputs(out, i, p, d, ne_max)
    frames = sum(p.n_frames for p in problems)
    print("%d clips x %d settings through %d slots: %.2f s, %.0f frames/s -> %s"
          % (len(clips), len(grid), q.slots, wall, frames / wall, args.results))


if __name__ == "__main__":
    main()
