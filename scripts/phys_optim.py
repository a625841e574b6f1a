#!/usr/bin/env python
"""Drop-in for the reference's `./phys_optim` executable (towr_phys_optim/phys_optim.cpp), same flags
(gflags syntax `--flag value` or `--flag=value`, phys_optim.cpp:23-31), same four input files and the same four
output files, solved on the GPU.  `scripts/run_phys_mocap.py:159-174` can point its `--towr-phys-optim-path` here.

Extension: `--in_dir` / `--out_dir` / `--nframes` accept comma separated lists so that many clips are solved as one
batch (that is where the GPU pays off); `--n_ee 2` selects the toes-only parameterisation; `--slots S` solves the list
through a queue of S device slots (`chd.phys.PhysQueue`: memory for S clips, each slot refilled as its clip finishes).
Under torchrun, `--slots S` runs such a queue on every rank's GPU, the ranks claiming their next clips from one shared
counter (`chd.parallel.ShardedSolver(slots=S)`), and rank 0 writes the four files of every clip.  Every `--w_*` flag takes
one value for all clips or a comma separated list aligned with `--in_dir`, one value per clip.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def write_results(out, problems, out_dirs, n_ee_max):
    """The four output files of every clip (`chd.phys.write_outputs`) and its status line, from a `solve()` result with
    all three snapshots: the one-GPU run and rank 0 of a `--slots` run under torchrun write through here."""
    import chd
    for i, (p, od) in enumerate(zip(problems, out_dirs)):
        chd.phys.write_outputs(out, i, p, od, n_ee_max)
        print("[%d] stages status %s iterations %s -> %s" % (i, out["stage_status"][:, i].tolist(), out["stage_iters"][:, i].tolist(), od))


WEIGHT_FLAGS = ("w_com_lin", "w_com_ang", "w_ee", "w_smooth", "w_dur")
WEIGHT_DEFAULTS = ("0.4", "1.7", "0.3", "0.1", "0.1")   # phys_optim.cpp:27-31


def parse_weights(args, n):
    """The `--w_*` flags as the solvers take them: one 5-tuple when every flag holds a single value, else one 5-tuple
    per clip, a single value standing for every clip.  A list whose length is not n raises ValueError."""
    cols = []
    for k in WEIGHT_FLAGS:
        v = [float(x) for x in str(getattr(args, k)).split(",")]
        if len(v) not in (1, n):
            raise ValueError("--%s: %d values for %d clips" % (k, len(v), n))
        cols.append(v)
    if all(len(v) == 1 for v in cols):
        return tuple(v[0] for v in cols)
    return [tuple(v[i] if len(v) > 1 else v[0] for v in cols) for i in range(n)]


def main(argv=None):
    ap = argparse.ArgumentParser(allow_abbrev=False)
    ap.add_argument("--out_dir", default="sol_out")
    ap.add_argument("--in_dir", default="./")
    ap.add_argument("--nframes", default="100")
    for k, v in zip(WEIGHT_FLAGS, WEIGHT_DEFAULTS):
        ap.add_argument("--" + k, default=v, help="one value, or one per clip (comma separated)")
    ap.add_argument("--n_ee", type=int, default=4)
    ap.add_argument("--stage3_long", action="store_true",
                    help="run stage 3 on sequences with more than 96 phase durations too (switch times as band unknowns)")
    ap.add_argument("--slots", type=int, default=0,
                    help="solve the clips through a queue of this many device slots instead of one batch")
    args = ap.parse_args(argv)
    import chd
    in_dirs = args.in_dir.split(",")
    out_dirs = args.out_dir.split(",")
    nframes = [int(x) for x in str(args.nframes).split(",")]
    if len(nframes) == 1:
        nframes = nframes * len(in_dirs)
    assert len(in_dirs) == len(out_dirs) == len(nframes)
    print("Out Dir: %s\nInput Directory: %s\nnum frames: %s" % (args.out_dir, args.in_dir, args.nframes))
    weights = parse_weights(args, len(in_dirs))
    if isinstance(weights, tuple):
        print("Optim weights (%g, %g, %g, %g)\nDuration cost weight %g" % weights)
    else:
        print("Optim weights (%s, %s, %s, %s)\nDuration cost weight %s" % tuple(getattr(args, k) for k in WEIGHT_FLAGS))
    problems = [chd.io_formats.read_phys_inputs(d, f, n_ee=args.n_ee) for d, f in zip(in_dirs, nframes)]
    band = 96 if args.stage3_long else None
    world, rank, local = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    if world > 1 and args.slots:
        # torchrun with a queue on every GPU: each rank claims its next clips from one counter in the process group's
        # store, and the results of every clip, all three snapshots included, are merged by clip index on every rank
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        out = chd.parallel.solve_sharded(problems, weights=weights, device=local, rank=rank, world=world,
                                         stage3_band_above=band, slots=args.slots)
        dist.destroy_process_group()
        if rank == 0:
            write_results(out, problems, out_dirs, max(p.n_ee for p in problems))
        return
    if world > 1:
        # torchrun: one process per GPU, sequences sharded by predicted work, one gather of the final trajectories;
        # only the durations snapshot travels, so the sharded mode writes sol_out_durations.txt + success_log.txt
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        out = chd.parallel.solve_sharded(problems, weights=weights, device=local, rank=rank, world=world,
                                         stage3_band_above=band)
        dist.destroy_process_group()
        if rank == 0:
            ne_max = max(p.n_ee for p in problems)
            for i, (p, od) in enumerate(zip(problems, out_dirs)):
                nf, n_ee = int(out["frames"][i]), p.n_ee
                cols = np.concatenate(chd.phys.sample_columns(n_ee, ne_max))
                chd.io_formats.write_solution(os.path.join(od, "sol_out_durations.txt"), p.dt, out["samples"][i, :nf][:, cols], n_ee)
                chd.io_formats.write_success_log(os.path.join(od, "success_log.txt"), out["success"][i, 0], out["success"][i, 1])
        return
    if args.slots:
        batch = chd.phys.PhysQueue(problems, args.slots, weights=weights, stage3_band_above=band)
    else:
        batch = chd.phys.PhysBatch(problems, weights=weights, stage3_band_above=band)
    out = batch.solve()
    write_results(out, problems, out_dirs, batch.n_ee_max)


if __name__ == "__main__":
    main()
