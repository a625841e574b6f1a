// TEST INFRASTRUCTURE ONLY -- host build of the product's work-item evaluators (csrc/chd_eval.cuh) for the CPU test
// suite: the same source the CUDA kernels include, compiled with a one-thread shim of the CUDA built-ins, so the
// stage-3 evaluation logic (run-time polynomial location, switch-time columns, table rebuilds) can be checked
// against the oracle without a GPU, and of the KKT plan (csrc/chd_kkt_plan.h).  Never loaded by the product.
#include <cmath>
#include <cstring>
#include <vector>

#define __device__
#define __forceinline__ inline
struct EmuDim { int x = 0; };
static EmuDim threadIdx;
static struct { int x = 1; } blockDim;
static inline void __syncthreads() {}
static inline double atomicAdd(double* p, double v) { double o = *p; *p += v; return o; }

#include "../../contact-human-dynamics_b200/csrc/chd_eval.cuh"

extern "C" int chd_emu_eval(const chd_phys_problem* prob, const chd_phys_weights* w, int stage, const double* x, int dyn,
                            double* cost, double* grad, double* g, double* Jv, int* ent_col, int* dims /*n, m, nslots, n_dur*/,
                            int* ent_ptr, int* row_set, double* row_lo, double* row_hi, int* dur_xoff) {
  ChdHostBatch hb;
  chd_phys_weights wt = {0.4, 1.7, 0.3, 0.1, 0.1};
  if (w) wt = *w;
  int rc = chd_build_layout(prob, 1, wt, hb);
  if (rc) return rc;
  const ChdSeq& h = hb.seq[0];
  if (dims) dims[0] = h.n, dims[1] = h.m, dims[2] = h.nslots, dims[3] = h.n_dur;
  if (ent_ptr) std::memcpy(ent_ptr, hb.ent_ptr.data(), sizeof(int) * (h.m + 1));
  if (row_set) std::memcpy(row_set, hb.row_set.data(), sizeof(int) * h.m);
  if (row_lo) std::memcpy(row_lo, hb.row_lo.data(), sizeof(double) * h.m);
  if (row_hi) std::memcpy(row_hi, hb.row_hi.data(), sizeof(double) * h.m);
  if (dur_xoff) std::memcpy(dur_xoff, h.dur_xoff, sizeof(int) * h.n_ee);
  if (!x) return 0;
  ChdDev D;
  std::memset(&D, 0, sizeof(D));
  D.B = 1, D.S = hb.S, D.Pmax = hb.Pmax, D.n_max = hb.n_max, D.m_max = hb.m_max, D.slots_max = hb.slots_max;
  D.sets_max = hb.sets_max, D.tab_max = hb.tab_max, D.F_max = hb.F_max, D.Kd_max = hb.Kd_max, D.Kr_max = hb.Kr_max;
  D.par_stride = hb.par_stride(), D.n_ee_max = hb.n_ee_max, D.Ph_max = hb.Ph_max;
  D.seq = hb.seq.data();
  D.poly_T = hb.poly_T.data(), D.poly_tend = hb.poly_tend.data(), D.node_const = hb.node_const.data(), D.par = hb.par.data();
  D.t_dyn = hb.t_dyn.data(), D.t_rom = hb.t_rom.data(), D.t_data = hb.t_data.data(), D.dur0 = hb.dur0.data();
  D.node_var = hb.node_var.data(), D.itab = hb.itab.data(), D.ent_ptr = hb.ent_ptr.data(), D.poly_ph = hb.poly_ph.data();
  D.ent_col = hb.ent_col.data(), D.sets = hb.sets.data(), D.phase_tend = hb.phase_tend.data();
  ChdStageDev sg;
  const ChdStageCfg& c0 = hb.stage[stage];
  sg.set_mask = c0.set_mask, sg.max_iter = c0.max_iter, sg.snap_after = -1, sg.opt_dur = stage == CHD_STAGE_3;
  for (int i = 0; i < 3; ++i) sg.w_data[i] = c0.w_data[i], sg.w_vel[i] = c0.w_vel[i], sg.w_acc[i] = c0.w_acc[i];
  sg.w_dur = c0.w_dur;
  ChdCtx c;
  chd_make_ctx(D, 0, x, c);
  c.dyn = dyn, c.opt_dur = sg.opt_dur && h.n_dur > 0;
  if (dyn) chd_tables_from_x(c, x, D.poly_T, D.poly_tend, D.phase_tend);
  std::vector<double> red(4, 0.0), gs(h.n, 0.0);
  std::vector<double> gv(h.m, 0.0), jv(h.nslots, 0.0);
  double f = 0.0;
  chd_eval_all<true>(c, sg, gv.data(), jv.data(), gs.data(), &f, red.data());
  if (cost) *cost = f;
  if (grad) std::memcpy(grad, gs.data(), sizeof(double) * h.n);
  if (g) std::memcpy(g, gv.data(), sizeof(double) * h.m);
  if (Jv) std::memcpy(Jv, jv.data(), sizeof(double) * h.nslots);
  if (ent_col) std::memcpy(ent_col, hb.ent_col.data(), sizeof(int) * h.nslots);
  return 0;
}

// The KKT plan batch creation computes for these batch strides, kernel static shared-memory sizes and opt-in limit.
extern "C" int chd_emu_kkt_plan(int Na_max, int nb_max, int w_max, int w_fix_max, int n_max, long long kkt_static,
                                long long gwin_static, long long smem_optin, ChdKktPlan* out) {
  *out = chd_kkt_plan(Na_max, nb_max, w_max, w_fix_max, n_max, kkt_static, gwin_static, smem_optin);
  return (int)sizeof(ChdKktPlan);
}
