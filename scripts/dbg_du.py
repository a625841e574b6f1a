import os, sys; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, ctypes as C, chd
from oracle.phys import OracleProblem
p = chd.synth.make_problem(1, n_ee=2)
b = chd.phys.PhysBatch([p])
o = OracleProblem(p)
g = b.solve_stage("1.1"); r = o.solve_stage("1.1")
g = b.solve_stage("1.2"); r = o.solve_stage("1.2")
print("1.2 gpu", g["iters"], g["f"], "oracle", r["iters"], r["f"])
dbg = np.zeros(16); b.L.chd_phys_debug_ipm.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]; b.L.chd_phys_debug_ipm(b.h, 0, dbg.ctypes.data)
print("DU additions counted:", dbg[14])
H = o.cost_hessian().diagonal(); sizes = o.var_set_sizes(); lo = sizes[0]+sizes[1]; hi = lo + sizes[2]+sizes[3]
print("oracle unobserved motion vars:", int((H[lo:hi] == 0).sum()), "of", hi-lo)
