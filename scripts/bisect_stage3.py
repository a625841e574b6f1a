"""Diagnostic: where do the CUDA solver and the CPU oracle part ways in stage 3?  Runs stages 1.1-2.2, then stage 3 capped
at k iterations on both sides and prints the iterate summaries."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import chd
from oracle.phys import OracleProblem
n_ee, seed, F = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
dense = len(sys.argv) > 5 and sys.argv[5] == "dense"
ks = [int(k) for k in sys.argv[4].split(",")]
p = chd.synth.make_problem(seed, n_frames=F, n_ee=n_ee, dense=dense)
for k in ks:
    b = chd.phys.PhysBatch([p])
    o = OracleProblem(p)
    for st in ("1.1", "1.2", "2.1", "2.2"):
        b.solve_stage(st), o.solve_stage(st)
    g = b.solve_stage("3", max_iter=k)
    r = o.solve_stage("3", max_iter=k, verbose=2 if k <= 2 else 0)
    xg = b.get_x()[0, :b.sizes[0, 0]]
    o.set_stage("3")
    xo = o.get_x()
    print("k=%d gpu: it %d st %d f %.9f E0 %.3e viol %.3e mu %.2e dw %.3e | oracle: it %d st %d f %.9f E0 %.3e viol %.3e mu %.2e dw %.3e | max|dx| %.2e" % (
        k, g["iters"][0], g["status"][0], g["f"][0], g["E0"][0], g["viol"][0], g["mu"][0], g["delta_w"][0],
        r["iters"], r["status"], r["f"], r["E0"], r["viol"], r["mu"], r["delta_w"], np.abs(xg - xo).max()))
    sizes = o.var_set_sizes()
    names = ["lin", "ang"] + ["mot%d" % e for e in range(n_ee)] + ["frc%d" % e for e in range(n_ee)] + ["dur%d" % e for e in range(n_ee)]
    offs = np.concatenate([[0], np.cumsum(sizes)])
    d = np.abs(xg - xo)
    top = np.argsort(-d)[:6]
    print("     largest |x_gpu - x_oracle|:", [(int(i), names[int(np.searchsorted(offs, i, side="right") - 1)], "%.3e" % d[i], "%.6g" % xg[i], "%.6g" % xo[i]) for i in top])
    b.close()
