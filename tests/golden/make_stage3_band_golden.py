"""Oracle reference for tests/test_stage3_band_gpu.py::test_banded_above_limit_matches_oracle: the CPU oracle's staged
schedule (oracle/phys.py, chd-ipm with the phase durations in its own dense border) on a 200-frame, 4-end-effector,
densely switching synthetic clip (`chd.synth.make_problem(0, n_frames=200, n_ee=4, dense=True)`, 113 phase
durations), with stage 3 run although the clip has more than the product's 96 border durations.  The oracle needs
691 s of one CPU core for it (stage 3 runs into its 2000-iteration cap, stage 4 then converges), too long for the GPU
suite, so its result is kept here:

    python tests/golden/make_stage3_band_golden.py

Writes tests/golden/stage3_band/oracle_dense200.npz: the three SaveSolution snapshots, per solved stage its id, status,
iterations and objective, the success flags and the oracle's wall time.
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "stage3_band", "oracle_dense200.npz")


def main():
    import chd
    from oracle.phys import OracleProblem
    t0 = time.time()
    o = OracleProblem(chd.synth.make_problem(0, n_frames=200, n_ee=4, dense=True))
    res, ids, snaps = [], [], {}
    for st in ("1.1", "1.2"):
        res.append(o.solve_stage(st)), ids.append(st)
    snaps["no_dynamics"] = o.sample()
    for st in ("2.1", "2.2"):
        res.append(o.solve_stage(st)), ids.append(st)
    snaps["dynamics"] = o.sample()
    dyn_ok = res[3]["status"] == 0
    res.append(o.solve_stage("3")), ids.append("3")        # whatever the number of phase durations
    dur_ok = res[-1]["status"] == 0
    if not dur_ok:                                         # phys_optim.cpp:713-749
        res.append(o.solve_stage("4")), ids.append("4")
        dur_ok = res[-1]["status"] == 0
    snaps["durations"] = o.sample()
    seconds = time.time() - t0
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, stage_ids=np.array(ids), status=np.array([r["status"] for r in res]),
                        iters=np.array([r["iters"] for r in res]), f=np.array([r["f"] for r in res]),
                        success=np.array([dyn_ok, dur_ok]), seconds=seconds, **snaps)
    print("stages", ids, [r["status"] for r in res], [r["iters"] for r in res], "%.0f s" % seconds)


if __name__ == "__main__":
    main()
