"""GPU vs CPU-oracle iteration counts / final objective per stage for a few sequences (diagnostic)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import chd
from oracle.phys import OracleProblem
n_ee = int(sys.argv[1]); seeds = [int(s) for s in sys.argv[2].split(",")]
F = int(sys.argv[3]) if len(sys.argv) > 3 else 120
dense = len(sys.argv) > 4 and sys.argv[4] == "dense"
ps = [chd.synth.make_problem(s, n_frames=F, n_ee=n_ee, dense=dense) for s in seeds]
b = chd.phys.PhysBatch(ps)
out = b.solve()
st = b.stage_stats()
ids = chd.phys.STAGES
base, pos, frc, _ = chd.phys.sample_columns(n_ee, n_ee)
for i, p in enumerate(ps):
    ref = OracleProblem(p).solve()
    print("seed", seeds[i], "gpu iters", out["stage_iters"][:, i].tolist(), "status", out["stage_status"][:, i].tolist())
    print("   oracle", [(k, s["iters"], s["status"], "%.6f" % s["f"]) for k, s in zip(ref["stage_ids"], ref["stages"])])
    print("   gpu f", ["%.6f" % st[ids[k], i, 0] for k in ref["stage_ids"]], "viol", ["%.1e" % st[ids[k], i, 2] for k in ref["stage_ids"]])
    nf = out["frames"][i]
    d = np.abs(out["samples"][2, i, :nf] - ref["durations"])
    print("   max |diff| pos %.2e force %.2e" % (d[:, np.r_[base, pos]].max(), d[:, frc].max()))
