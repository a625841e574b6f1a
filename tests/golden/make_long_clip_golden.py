"""Oracle reference for tests/test_long_clip_gpu.py: the CPU oracle's staged schedule (oracle/phys.py, chd-ipm) on a
1100-frame, 4-end-effector walking clip (`chd.synth.make_problem(0, n_frames=1100, n_ee=4)`), whose iterate is larger
than the evaluation and line-search kernels can hold in shared memory.  The clip has more phase durations than the
product's 96 border durations, so, as in the product, stage 3 is not attempted: the schedule is 1.1, 1.2, 2.1, 2.2, 4.
Too slow for the GPU suite, so its result is kept here:

    python tests/golden/make_long_clip_golden.py

Writes tests/golden/long_clip/oracle_walk1100.npz: the three SaveSolution snapshots, per solved stage its id, status,
iterations and objective, the success flags and the oracle's wall time.
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "long_clip", "oracle_walk1100.npz")
FRAMES, N_EE = 1100, 4


def main():
    import chd
    from oracle.phys import OracleProblem
    t0 = time.time()
    o = OracleProblem(chd.synth.make_problem(0, n_frames=FRAMES, n_ee=N_EE))
    assert o.n_dur > 96
    ref = o.solve()                                        # 1.1, 1.2, 2.1, 2.2, 4 (phys_optim.cpp:554-749)
    seconds = time.time() - t0
    res, ids = ref["stages"], ref["stage_ids"]
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, stage_ids=np.array(ids), status=np.array([r["status"] for r in res]),
                        iters=np.array([r["iters"] for r in res]), f=np.array([r["f"] for r in res]),
                        success=np.array(ref["success"]), seconds=seconds, no_dynamics=ref["no_dynamics"],
                        dynamics=ref["dynamics"], durations=ref["durations"])
    print("stages", ids, [r["status"] for r in res], [r["iters"] for r in res], "%.0f s" % seconds)


if __name__ == "__main__":
    main()
