#!/usr/bin/env python
"""Physics solve queue (`chd.phys.PhysQueue`) against consecutive `PhysBatch` solves of the same clips (DESIGN §7).

Two configurations:
  short: 256 clips of 120 frames, 2 feet (chd.synth.make_problem seeds 0..255, bench.py's inputs): the queue at 64 and
         128 slots against four consecutive 64-clip batches;
  long:  64 clips of 600 frames, 4 feet, densely switching: the queue at 16 slots against four 16-clip batches.
A third, `--config claim`, times the short configuration's 64-slot queue in its own order against the same queue fed by a
`chd.parallel.StoreClaim` over a FileStore (one process: the cost of the claim callback and the store round trips that
the multi-GPU queue of `ShardedSolver(slots=...)` adds).
Every arm is warmed up, then the arms alternate in one process; each timed repetition is creation + solve (what a user
of either pays).  A second pass with kernel timing on gives `chd_k_kkt` ms per launch and the admission time.  Per clip
the outputs of every arm are compared with the batches' (statuses, iteration counts, trajectories).  Prints the card's
name and power limit and one JSON line per configuration.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         check=True, capture_output=True, text=True).stdout.strip().split(", ")
    return {"gpu": out[0], "power_limit": out[1], "max_sm_clock": out[2]}


class PoolMeter:
    """Bytes currently allocated from device 0's default memory pool (libchd allocates with cudaMallocAsync from it)."""

    def __init__(self):
        self.cu = C.CDLL("libcuda.so.1")
        assert self.cu.cuInit(0) == 0
        dev = C.c_int()
        assert self.cu.cuDeviceGet(C.byref(dev), 0) == 0
        self.pool = C.c_void_p()
        assert self.cu.cuDeviceGetDefaultMemPool(C.byref(self.pool), dev) == 0

    def used(self):
        v = C.c_uint64()
        assert self.cu.cuMemPoolGetAttribute(self.pool, 7, C.byref(v)) == 0   # CU_MEMPOOL_ATTR_USED_MEM_CURRENT
        return v.value


def solve_batches(chd, ps, per, timing=False):
    """Consecutive batches of `per` clips; results concatenated in clip order, plus the instrumentation of all."""
    parts, kkt_ms, kkt_n = [], 0.0, 0
    for a in range(0, len(ps), per):
        b = chd.phys.PhysBatch(ps[a:a + per])
        b.set_timing(timing)
        out = b.solve()
        kt = b.kernel_times()
        kkt_ms, kkt_n = kkt_ms + kt["kkt"][0], kkt_n + kt["kkt"][1]
        b.close()
        parts.append(out)
    return chd.phys.concat_results(parts), {"kkt_ms": kkt_ms, "kkt_launches": kkt_n}


def solve_queue(chd, ps, slots, timing=False, meter=None, claim=None):
    u0 = meter.used() if meter else 0
    if claim is not None:
        claim.restart()                                 # a fresh counter: the queue starts over
    q = chd.phys.PhysQueue(ps, slots, claim=claim)
    dev_bytes = (meter.used() - u0) if meter else None
    h0 = q.h2d_bytes()
    q.set_timing(timing)
    out = q.solve()
    kt = q.kernel_times()
    info = {"kkt_ms": kt["kkt"][0], "kkt_launches": kt["kkt"][1], "admit_ms": kt["admit"][0], "admit_rounds": kt["admit"][1],
            "admit_bytes": q.h2d_bytes() - h0, "device_bytes": dev_bytes, "slots": q.slots}
    q.close()
    return out, info


def compare(ref, got):
    """Per clip: equal statuses, equal stage 1.1-2.2 iteration counts, largest trajectory difference (snapshot 1 = after
    stage 2.2, snapshot 2 = final)."""
    n = ref["frames"].shape[0]
    fo = min(ref["samples"].shape[2], got["samples"].shape[2])
    d1 = np.abs(ref["samples"][1, :, :fo] - got["samples"][1, :, :fo]).max()
    d2 = np.abs(ref["samples"][2, :, :fo] - got["samples"][2, :, :fo]).max()
    return {"status_equal": int((ref["stage_status"] == got["stage_status"]).all(axis=0).sum()),
            "iters_1_to_22_equal": int((ref["stage_iters"][:4] == got["stage_iters"][:4]).all(axis=0).sum()),
            "frames_equal": bool((ref["frames"] == got["frames"]).all()), "clips": n,
            "max_abs_diff_snap1": float(d1), "max_abs_diff_final": float(d2)}


def run(chd, name, ps, per, slot_list, reps, meter):
    frames = int(sum(p.n_frames for p in ps))
    arms = [("batches%d" % per, lambda t=False: solve_batches(chd, ps, per, t))]
    arms += [("queue%d" % s, (lambda s: lambda t=False: solve_queue(chd, ps, s, t, meter))(s)) for s in slot_list]
    for _, f in arms:                                  # warm-up: module load, pool growth
        f()
    times = {a: [] for a, _ in arms}
    outs, infos = {}, {}
    for r in range(reps):
        for a, f in arms:
            t0 = time.perf_counter()
            outs[a], infos[a] = f()
            times[a].append(time.perf_counter() - t0)
    res = {"config": name, "clips": len(ps), "frames": frames, "arms": {}}
    ref = outs[arms[0][0]]
    sum_iters = int(ref["stage_iters"].sum())
    for a, f in arms:
        _, tinfo = f(True)                              # kernel timing on: per-launch times (slower; not the wall time)
        med = float(np.median(times[a]))
        info = dict(infos[a])
        loop = tinfo["kkt_launches"]
        arm = {"wall_s": [round(t, 4) for t in times[a]], "frames_per_s": round(frames / med, 1),
               "kkt_ms_per_launch": round(tinfo["kkt_ms"] / max(loop, 1), 4), "loop_iterations": loop,
               "live_clips_per_launch": round(sum_iters / max(loop, 1), 2)}
        if "admit_ms" in tinfo:
            arm.update(slots=info["slots"], admit_rounds=tinfo["admit_rounds"], admit_ms=round(tinfo["admit_ms"], 3),
                       admit_upload_bytes=info["admit_bytes"],
                       device_bytes_per_slot=None if info["device_bytes"] is None else int(info["device_bytes"] / info["slots"]))
        arm["vs_batches"] = compare(ref, outs[a])
        res["arms"][a] = arm
    return res


class CountingClaim:
    """A claim source that counts its calls (store round trips) on the way to another, and the host time they take."""

    def __init__(self, inner):
        self.inner, self.calls, self.seconds = inner, 0, 0.0

    def restart(self):
        self.calls, self.seconds = 0, 0.0
        self.inner.restart()

    def __call__(self, want):
        t0 = time.perf_counter()
        r = self.inner(want)
        self.calls += 1
        self.seconds += time.perf_counter() - t0
        return r


def run_claim(chd, ps, slots, reps):
    """The queue in its own order against the same queue claiming from a FileStore counter, alternated."""
    import tempfile
    import torch.distributed as dist
    frames = int(sum(p.n_frames for p in ps))
    with tempfile.TemporaryDirectory() as tmp:
        claim = CountingClaim(chd.parallel.StoreClaim(dist.FileStore(os.path.join(tmp, "claims"), 1), "bench", len(ps)))
        arms = [("queue%d" % slots, lambda: solve_queue(chd, ps, slots)),
                ("queue%d_store_claim" % slots, lambda: solve_queue(chd, ps, slots, claim=claim))]
        for _, f in arms:                              # warm-up
            f()
        times = {a: [] for a, _ in arms}
        outs = {}
        for r in range(reps):
            for a, f in arms:
                t0 = time.perf_counter()
                outs[a] = f()[0]
                times[a].append(time.perf_counter() - t0)
        res = {"config": "%d x 120 frames, 2 feet: own order vs StoreClaim over a FileStore" % len(ps), "clips": len(ps),
               "frames": frames, "arms": {}}
        for a, _ in arms:
            med = float(np.median(times[a]))
            res["arms"][a] = {"wall_s": [round(t, 4) for t in times[a]], "frames_per_s": round(frames / med, 1),
                              "vs_own_order": compare(outs[arms[0][0]], outs[a])}
        res["arms"][arms[1][0]]["claim_calls"] = claim.calls
        res["arms"][arms[1][0]]["claim_ms"] = round(1e3 * claim.seconds, 3)       # in the callback, last solve
        res["arms"][arms[1][0]]["all_solved"] = bool(outs[arms[1][0]]["solved"].all())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=["short", "long", "both", "claim"], default="both")
    ap.add_argument("--reps", type=int, default=3, help="timed repetitions of every arm (short configuration)")
    ap.add_argument("--reps-long", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import chd
    info = card()
    print("card: %(gpu)s, power limit %(power_limit)s, max SM clock %(max_sm_clock)s" % info, flush=True)
    meter = PoolMeter()
    lines = []
    if args.config in ("short", "both"):
        ps = [chd.synth.make_problem(s, 120, 2) for s in range(256)]
        lines.append(run(chd, "256 x 120 frames, 2 feet", ps, 64, [64, 128], args.reps, meter))
        print(json.dumps(dict(lines[-1], card=info)), flush=True)
    if args.config == "claim":
        ps = [chd.synth.make_problem(s, 120, 2) for s in range(256)]
        lines.append(run_claim(chd, ps, 64, args.reps))
        print(json.dumps(dict(lines[-1], card=info)), flush=True)
    if args.config in ("long", "both"):
        ps = [chd.synth.make_problem(s, 600, 4, dense=True) for s in range(64)]
        lines.append(run(chd, "64 x 600 frames, 4 feet, dense", ps, 16, [16], args.reps_long, meter))
        print(json.dumps(dict(lines[-1], card=info)), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for l in lines:
                f.write(json.dumps(dict(l, card=info)) + "\n")


if __name__ == "__main__":
    main()
