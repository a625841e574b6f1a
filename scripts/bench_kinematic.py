"""Timing of the two kinematic steps around the hot path (not part of bench.py's contract): the kinematic optimiser
(`chd.kinopt.optimize_trajectory`, 2 x 50 evaluations like the reference's two least_squares stages) and the IK of
`apply_results` (30 iterations, 69-joint character), on cuda:0 (`chd_kin_solve` / `chd_ik_solve`) and on the host
cores (torch).  One JSON line.
The reference's own optimize_trajectory needed 7.5 s for the 14-frame golden clip in the build container
(tests/golden/kinopt/run.npz `seconds`); its dense Jacobian is 4 GB at 120 frames."""
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np


def main():
    import torch
    import chd
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 120
    d = tempfile.mkdtemp()
    vd = os.path.join(d, "w")
    chd.synth.write_mocap_clip(vd, F, seed=0)
    out = {"frames": F}
    for dev in (["cuda:0"] if torch.cuda.is_available() else []) + [None]:
        tag = dev or "cpu"
        # warm-up on the first 12 frames (cuSOLVER / cuBLAS handles), then the timed run
        chd.kinopt.optimize_2d_3d(os.path.join(vd, "w.mp4"), os.path.join(vd, "skeleton.bvh"), os.path.join(d, "kw" + tag), 0, 12, device=dev)
        t0 = time.perf_counter()
        res = chd.kinopt.optimize_2d_3d(os.path.join(vd, "w.mp4"), os.path.join(vd, "skeleton.bvh"), os.path.join(d, "k" + tag), 0, F, device=dev)
        if dev:
            torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        out["kinopt_s_" + tag] = dt
        out["kinopt_cost_" + tag] = res[-1]["stage2"]["cost"]
    # IK of apply_results on a 69-joint skeleton
    from bench_skeletons import ybot_like
    names, parents, off = ybot_like()
    rng = np.random.default_rng(0)
    J = len(names)
    e = np.cumsum(rng.normal(0, 0.01, (F, J, 3)), axis=0)
    R = chd.results.rot_zyx(e)
    P = np.tile(np.asarray(off, float)[None], (F, 1, 1))
    anim = chd.results.SkelAnim(names, np.array(parents), np.asarray(off, float), R, P)
    gp = anim.global_positions()
    tj = list(range(0, 57)) + [60, 65, 67, 68]
    targets = {j: gp[:, j] + rng.normal(0, 1.0, (F, 3)) for j in tj}
    for dev in (["cuda:0"] if torch.cuda.is_available() else []) + [None]:
        tag = dev or "cpu"
        for rep in range(2):
            t0 = time.perf_counter()
            if dev:          # returns host arrays, so the time includes the kernel
                chd.results.ik_solve_batch([anim], [targets], iterations=30, damping=7.0, smoothness=0.001, device=dev)
            else:
                chd.results.ik_solve(anim, targets, iterations=30, damping=7.0, smoothness=0.001)
            dt = time.perf_counter() - t0
        out["ik_s_" + tag] = dt
    print(json.dumps(out))


if __name__ == "__main__":
    main()
