"""Batched kinematic initialisation on cuda:0 (`chd.kinopt.optimize_trajectory_batch`, kernel `chd_kin_solve`).  Prints one
JSON line:
  solve:      CUDA-event time per chd_kin_solve launch on normal equations of seeded synthetic clips, and the per-frame
              torch sweep (`_banded_cholesky_solve`, the CPU solver) on the same 600-frame system; achieved fp64 rate
              from the counted flop (kin_flop below) against the measured DMMA rate of the card.
  end_to_end: optimize_trajectory_batch against the per-clip loop of optimize_trajectory(device="cuda:0"), after one
              untimed call, with the per-clip final costs of both arms.
  gpu:        card name and power limit, read in the same run.
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
import chd  # noqa: E402

N = 87


def kin_flop(F):
    """fp64 operations of one clip's factorisation and substitutions (n = 87 unknowns per frame): per frame the Schur
    updates with L1 L1^T and L2 L2^T (n^3 each), the Cholesky (n^3 / 3), A1 = B1 - L2 L1^T (2 n^3), the two triangular
    solves for L1 and L2 (n^3 each) and the forward and backward substitutions (2 n^2 per block product, n^2 per
    triangular solve)."""
    n3, n2 = N ** 3, N ** 2
    total = 0.0
    for f in range(F):
        h1, h2 = f + 1 < F, f + 2 < F
        total += n3 * ((f >= 1) + (f >= 2)) + n3 / 3.0 + 2 * n3 * (h1 and f >= 1) + n3 * (h1 + h2)
        total += 2 * (n2 + 2 * n2 * ((f >= 1) + (f >= 2)))
    return total


def clip_inputs(d, F, seed):
    ko = chd.kinopt
    chd.synth.write_mocap_clip(d, F, seed=seed)
    kp = chd.contact.load_keypoint_dir(os.path.join(d, "openpose_result"))
    p3, rp, ang = ko.combined_inputs(ko.load_totalcap_results(os.path.join(d, "tracked_results.json")))
    b = chd.prepare.load_bvh(os.path.join(d, "skeleton.bvh"))
    return dict(poses2D=np.concatenate([kp[:, :, :2], np.zeros((F, 3, 2))], 1), conf=np.concatenate([kp[:, :, 2], np.zeros((F, 3))], 1),
                poses3D=p3, root_pos=rp, ang=ang, parents=b.parents, offsets=b.offsets, ppx=960.0, ppy=540.0, focal=np.array(ko.MTC_FOCAL),
                vel=ko.contacts_to_constraints(np.load(os.path.join(d, "foot_contacts.npy"))))


ARGS = ("poses2D", "conf", "poses3D", "root_pos", "ang", "parents", "offsets", "ppx", "ppy", "focal", "vel")


def normal_equations(clips, dev):
    """Batch model and its normal equations at the IK-free start (root translation, zero angles) of every clip."""
    import torch
    ko = chd.kinopt
    probs, xs = [], []
    for c in clips:
        j2n, pw, dw = ko.make_weights(c["poses2D"], c["conf"], (c["ppx"], c["ppy"]), c["focal"])
        off = ko.update_skeleton(c["parents"], c["offsets"], c["poses3D"][:, ko.FORWARD] + c["root_pos"][:, None])
        probs.append(ko.Problem(c["parents"], off, c["poses3D"], c["root_pos"], j2n, pw, dw, c["vel"], np.zeros(3), np.zeros(3)))
        x = np.zeros((c["poses3D"].shape[0], ko.NV))
        x[:, :3] = c["root_pos"]
        xs.append(x)
    m = ko._Model(probs, dev)
    _, H, g = m.normal_equations(torch.as_tensor(np.concatenate(xs), device=dev), ko.StageWeights())
    return m, H, g


def time_events(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1]), "max_sm_mhz": float(out[2])}
    except Exception as e:                 # the numbers are still reported, without the card's settings
        return {"gpu": None, "error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--batches", default="1x120,8x120,64x120,8x600", help="end-to-end batches, KxF")
    ap.add_argument("--max-nfev", type=int, default=50)
    a = ap.parse_args()
    import torch
    ko = chd.kinopt
    dev = torch.device("cuda:0")
    out = {"gpu": gpu_info()}
    _, dmma = chd.phys.measure_fp64_peak()
    out["dmma_gflops_measured"] = dmma
    with tempfile.TemporaryDirectory() as tmp:
        cache = {}

        def clips(K, F):
            for k in range(K):
                if (F, k) not in cache:
                    cache[(F, k)] = clip_inputs(os.path.join(tmp, "c%d_%d" % (F, k)), F, seed=1000 * F + k)
            return [cache[(F, k)] for k in range(K)]

        # ---- (a) solve only ----
        solve = {}
        for K, F in ((1, 120), (64, 120), (1, 600), (8, 600)):
            m, H, g = normal_equations(clips(K, F), dev)
            sv = ko._KinSolver(m)
            lam = np.full(K, 1e-3)
            live = np.arange(K)
            ms = time_events(lambda: sv(H, g, lam, live), a.reps)
            st = sv.status.cpu().numpy()
            fl = K * kin_flop(F)
            solve["%dx%d" % (K, F)] = dict(ms_per_launch=ms, status_ok=bool((st == 0).all()), gflop=fl / 1e9,
                                           gflops=fl / (ms * 1e6), frac_of_dmma=fl / (ms * 1e6) / dmma)
            if K == 1 and F == 600:
                solve["sweep_1x600_ms"] = time_events(lambda: ko._banded_cholesky_solve(torch, H, g, 1e-3), 2)
                ref = ko._banded_cholesky_solve(torch, H, g, 1e-3)
                solve["sweep_1x600_max_abs_diff"] = float((ref - sv.s).abs().max())
            print("solve %dx%d done" % (K, F), json.dumps(solve), file=sys.stderr, flush=True)
            del m, H, g, sv
            torch.cuda.empty_cache()
        out["solve"] = solve
        # ---- (b) end to end ----
        e2e = {}
        # one untimed call first, so that the first configuration does not carry the one-off start-up cost
        F0 = int(a.batches.split(",")[0].split("x")[1])
        ko.optimize_trajectory(*[clips(1, F0)[0][k] for k in ARGS], device="cuda:0", max_nfev=a.max_nfev)
        for spec in a.batches.split(","):
            K, F = (int(v) for v in spec.split("x"))
            cs = clips(K, F)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rb = ko.optimize_trajectory_batch(*[[c[k] for c in cs] for k in ARGS], device="cuda:0", max_nfev=a.max_nfev)
            torch.cuda.synchronize()
            tb = time.perf_counter() - t0
            t0 = time.perf_counter()
            rl = [ko.optimize_trajectory(*[c[k] for k in ARGS], device="cuda:0", max_nfev=a.max_nfev) for c in cs]
            torch.cuda.synchronize()
            tl = time.perf_counter() - t0
            e2e[spec] = dict(batch_s=tb, loop_s=tl, speedup=tl / tb,
                             batch_cost=[r[6]["stage2"]["cost"] for r in rb], loop_cost=[r[6]["stage2"]["cost"] for r in rl],
                             batch_nfev=[[r[6]["stage1"]["nfev"], r[6]["stage2"]["nfev"]] for r in rb],
                             loop_nfev=[[r[6]["stage1"]["nfev"], r[6]["stage2"]["nfev"]] for r in rl],
                             max_pos_diff_cm=float(max(np.linalg.norm(x[1] - y[1], axis=-1).max() for x, y in zip(rb, rl))))
            print("end to end %s done" % spec, json.dumps(e2e[spec]), file=sys.stderr, flush=True)
            torch.cuda.empty_cache()
        out["end_to_end"] = e2e
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
