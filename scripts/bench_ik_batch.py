"""Batched full-body IK on cuda:0 (`chd.results.apply_results_batch` / `retarget_batch`, kernel `chd_ik_solve`) against
the per-clip loops of `apply_results(device="cuda:0")` / `retarget(device="cuda:0")`, i.e. one batch-of-one kernel call
per clip (per result file for apply), on the 69-joint ybot-like character of scripts/bench_skeletons.py (67 joints in
the files, the two heels added by apply_results).  Prints one JSON line:
  per workload K x F (clips x frames), for `apply` (3 result files per clip x 30 iterations, 61 targets) and `retarget`
  (200 iterations): host-clock seconds of both arms over `--runs` alternating runs after one warm-up call of each arm,
  peak device memory of each arm, max |difference| between the arms' outputs (rotation entries, local translations in
  cm), and the CUDA-event time per iteration of one chd_ik_solve call on the same clips with the counted fp64 flop rate
  (ik_flop below) next to the card's measured DFMA and DMMA rates;
  gpu: card name and power limit, read in the same run.
Needs a GPU; writes only under a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import chd  # noqa: E402
from bench_skeletons import ybot_like  # noqa: E402

TAGS = ("no_dynamics", "dynamics", "durations")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1]), "max_sm_mhz": float(out[2])}
    except Exception as e:                 # the numbers are still reported, without the card's settings
        return {"gpu": None, "error": str(e)}


def ik_flop(parents, tj, translate=True):
    """fp64 operations of one frame and iteration of chd_k_ik_iter, counted from the ancestor table: per target pair and
    strict common ancestor 114 (two arms, per axis two cross products and the 3 x 3 outer product), per common ancestor 9
    (translation block); Cholesky n^3 / 3 and the two triangular solves 2 n^2 (n = 3T); J^T y 54 per (joint, target below)
    for the rotation and 18 per (joint, target at or below) for the translation columns.  Forward kinematics, the Euler
    angles and the update are left out (O(J))."""
    J = len(parents)
    anc = []
    for j in range(J):
        a, k = [], int(parents[j])
        while k >= 0:
            a.append(k)
            k = int(parents[k])
        anc.append(set(a))
    total = 0.0
    for i1, t1 in enumerate(tj):
        for t2 in tj[:i1 + 1]:
            common = anc[t1] & anc[t2]
            strict = len(common)
            both = (anc[t1] | {t1}) & (anc[t2] | {t2})
            total += 114 * strict + (9 * len(both) if translate else 0)
    n = 3 * len(tj)
    total += n ** 3 / 3.0 + 2 * n * n
    for t in tj:
        total += 54 * len(anc[t]) + (18 * (len(anc[t]) + 1) if translate else 0)
    return total


def write_character(d):
    """The 67-joint character skeleton (one frame, rotations zeroed) for re-targeting and apply_results."""
    names, parents, off = ybot_like()
    names, parents, off = names[:67], np.array(parents[:67]), np.asarray(off[:67], float)
    a = chd.results.SkelAnim(names, parents, off, np.tile(np.eye(3), (1, 67, 1, 1)), off[None].copy())
    path = os.path.join(d, "ybot_skel.bvh")
    chd.results.save_bvh(path, a, names)
    return names, parents, off, path


def write_clip(d, k, F, rng, names, parents, off):
    """A character clip (smooth random angles) and the three result files' contents it is applied with."""
    J = len(names)
    e = np.cumsum(rng.normal(0, 0.01, (F, J, 3)), axis=0)
    P = np.tile(off[None], (F, 1, 1))
    P[:, 0] = np.cumsum(rng.normal(0, 0.5, (F, 3)), axis=0) + [0, 90, 0]
    a = chd.results.SkelAnim(names, parents, off, chd.results.rot_zyx(e), P)
    path = os.path.join(d, "clip%d_%d.bvh" % (F, k))
    chd.results.save_bvh(path, a, names)
    info = chd.prepare.ybot_info()
    gp = a.global_positions()
    feet = gp[:, [info.toes[0], info.toes[1], info.ankles[0], info.ankles[1]]]
    res = []
    for _ in TAGS:
        base_rot = chd.prepare.euler_zyx_from_matrix(a.rotations[:, 0]) + rng.normal(0, 0.02, (F, 3))
        res.append(chd.results.TowrResults(4, 1.0 / 30, (gp[:, 0] + rng.normal(0, 1.0, (F, 3))) / 100.0, base_rot, chd.results.rot_zyx(base_rot),
                                           (feet + rng.normal(0, 1.0, feet.shape)) / 100.0, np.zeros((F, 4, 3)), np.ones((F, 4), np.int64)))
    return path, res


def write_source(d, k, F, rng):
    """A 28-joint `combined` source clip for re-targeting."""
    pr = chd.prepare
    off = np.asarray(pr.COMBINED_OFFSETS, float)
    e = np.cumsum(rng.normal(0, 0.01, (F, 28, 3)), axis=0)
    P = np.tile(off[None], (F, 1, 1))
    P[:, 0] = np.cumsum(rng.normal(0, 0.5, (F, 3)), axis=0) + [0, -90, 300]
    a = chd.results.SkelAnim(list(pr.COMBINED_NAMES), np.array(pr.COMBINED_PARENTS), off, chd.results.rot_zyx(e), P)
    path = os.path.join(d, "src%d_%d.bvh" % (F, k))
    chd.results.save_bvh(path, a, a.names)
    return path


def max_diff(xs, ys):
    return (float(max(np.abs(x.rotations - y.rotations).max() for x, y in zip(xs, ys))),
            float(max(np.abs(x.positions - y.positions).max() for x, y in zip(xs, ys))))


def kernel_time(anims, targets, iterations, smoothness, translate, reps):
    """CUDA-event ms per iteration of one chd_ik_solve call on the stacked clips."""
    import torch
    dev = torch.device("cuda:0")
    tj = list(targets[0])
    frames = [a.rotations.shape[0] for a in anims]
    R0 = torch.as_tensor(np.concatenate([a.rotations for a in anims]), device=dev)
    P0 = torch.as_tensor(np.concatenate([a.positions for a in anims]), device=dev)
    goal = torch.as_tensor(np.concatenate([np.stack([tg[j] for j in tj], 1) for tg in targets]), device=dev).contiguous()
    R, P = R0.clone(), P0.clone()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for r in range(reps + 1):
        R.copy_(R0)
        P.copy_(P0)
        e0.record()
        chd.results._ik_kernel(anims[0].parents, tj, frames, R, P, goal, iterations, 7.0, smoothness, translate)
        e1.record()
        torch.cuda.synchronize()
        if r:                                # the first call is a warm-up
            ms.append(e0.elapsed_time(e1) / iterations)
    return float(np.median(ms)), sum(frames), anims[0].parents, tj


def timed(fn):
    import torch
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base


def compare(arms, runs, warm):
    """Warm up each arm, then alternate them `runs` times; returns per-arm seconds, peak bytes and the last outputs."""
    for fn in warm.values():
        fn()
    rec = {k: dict(s=[], peak_bytes=0) for k in arms}
    outs = {}
    for _ in range(runs):
        for k, fn in arms.items():
            o, s, peak = timed(fn)
            rec[k]["s"].append(s)
            rec[k]["peak_bytes"] = max(rec[k]["peak_bytes"], peak)
            outs[k] = o
    return rec, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="1x120,8x120,64x120,8x600", help="KxF: clips x frames")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5, help="chd_ik_solve calls per kernel timing")
    ap.add_argument("--only", default="apply,retarget")
    a = ap.parse_args()
    import torch
    dev = "cuda:0"
    out = {"gpu": gpu_info()}
    dfma, dmma = chd.phys.measure_fp64_peak()
    out["dfma_gflops_measured"], out["dmma_gflops_measured"] = dfma, dmma
    rs = chd.results
    info = chd.prepare.ybot_info()
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as tmp:
        names, parents, off, skel = write_character(tmp)
        for spec in a.workloads.split(","):
            K, F = (int(v) for v in spec.split("x"))
            w = {}
            if "apply" in a.only:
                clips = [write_clip(tmp, k, F, rng, names, parents, off) for k in range(K)]
                jobs = [(r, path, 0, F) for path, res in clips for r in res]
                arms = {"batch": lambda: rs.apply_results_batch(jobs, info, device=dev, iterations=30),
                        "loop": lambda: [rs.apply_results(*j, info, device=dev, iterations=30) for j in jobs]}
                warm = {"batch": lambda: rs.apply_results_batch(jobs[:1], info, device=dev, iterations=30),
                        "loop": lambda: rs.apply_results(*jobs[0], info, device=dev, iterations=30)}
                rec, outs = compare(arms, a.runs, warm)
                dr, dp = max_diff([o[0] for o in outs["batch"]], [o[0] for o in outs["loop"]])
                setups = [rs._apply_setup(*j, info, True, dev) for j in jobs]
                ms, Ft, par, tj = kernel_time([s[0] for s in setups], [s[3] for s in setups], 30, 0.001, True, a.reps)
                fl = ik_flop(par, tj) * Ft
                w["apply"] = dict(jobs=len(jobs), J=len(par), T=len(tj), batch=rec["batch"], loop=rec["loop"],
                                  speedup=float(np.median(rec["loop"]["s"]) / np.median(rec["batch"]["s"])),
                                  max_abs_diff_rot=dr, max_abs_diff_pos_cm=dp, kernel_ms_per_iter=ms,
                                  gflop_per_iter=fl / 1e9, gflops=fl / (ms * 1e6), frac_of_dfma=fl / (ms * 1e6) / dfma, frac_of_dmma=fl / (ms * 1e6) / dmma)
                print("apply %s" % spec, json.dumps(w["apply"]), file=sys.stderr, flush=True)
            if "retarget" in a.only:
                srcs = [write_source(tmp, k, F, rng) for k in range(K)]
                arms = {"batch": lambda: rs.retarget_batch(srcs, skel, info, device=dev),
                        "loop": lambda: [rs.retarget(s, skel, info, device=dev) for s in srcs]}
                warm = {"batch": lambda: rs.retarget_batch(srcs[:1], skel, info, device=dev),
                        "loop": lambda: rs.retarget(srcs[0], skel, info, device=dev)}
                rec, outs = compare(arms, a.runs, warm)
                dr, dp = max_diff(outs["batch"], outs["loop"])
                sk, h = rs._retarget_skeleton(skel, info)
                setups = [rs._retarget_setup(s, sk, h, info) for s in srcs]
                ms, Ft, par, tj = kernel_time([s[0] for s in setups], [s[1] for s in setups], 200, 0.0, True, a.reps)
                fl = ik_flop(par, tj) * Ft
                w["retarget"] = dict(J=len(par), T=len(tj), batch=rec["batch"], loop=rec["loop"],
                                     speedup=float(np.median(rec["loop"]["s"]) / np.median(rec["batch"]["s"])),
                                     max_abs_diff_rot=dr, max_abs_diff_pos_cm=dp, kernel_ms_per_iter=ms,
                                     gflop_per_iter=fl / 1e9, gflops=fl / (ms * 1e6), frac_of_dfma=fl / (ms * 1e6) / dfma, frac_of_dmma=fl / (ms * 1e6) / dmma)
                print("retarget %s" % spec, json.dumps(w["retarget"]), file=sys.stderr, flush=True)
            out[spec] = w
            torch.cuda.empty_cache()
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
