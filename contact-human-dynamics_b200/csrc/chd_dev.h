// Device-side views of a phys-optim batch (product code).
#pragma once
#include "chd_core.h"
#include "chd_kkt_plan.h"
#include "chd_layout.h"

#define CHD_FILT_MAX 24
#define CHD_THREADS 512
#define CHD_NL_GUARD 1.0    /* stage 3 line search: trial refused while theta_t - (1-alpha) theta > CHD_NL_GUARD * max(alpha theta, CHD_NL_FLOOR max(1, theta_ref)) */
#define CHD_NL_FLOOR 1e-4
#define CHD_UNOBS_EPS 1e-14 /* "sees": diagonal of the scaled cost Hessian above this (a sample sitting exactly on a node gives weights of 1e-17) */
#define CHD_DW_UNOBS 1e-4   /* fixed Levenberg-Marquardt weight of foot-motion node values no cost sample sees (zero diagonal of the cost Hessian) */
#define CHD_TERMS_THREADS 256
#define CHD_CURV_MIN 1e-8   /* multiplier threshold below which y^+ Jd^T Jd is not added (same in oracle/ipm_oracle.cpp) */

// row flags
#define CHD_ROW_ACTIVE 1
#define CHD_ROW_EQ 2
#define CHD_ROW_HASL 4
#define CHD_ROW_HASU 8
#define CHD_ROW_WARM 16   /* row keeps the interior-point state of the previous stage (stage 3 after 2.2) */

// Interior-point state of one sequence ("chd-ipm", see DESIGN.md).
#define CHD_PH_BEGIN 0
#define CHD_PH_RUN 1
#define CHD_PH_FINISHED 2
struct ChdIpm {
  int status;    // of the current stage: 1 running, 0 converged, -1 iteration cap, -2 numerical failure
  int iter, nfilt, ls_fail, max_iter, n_bounds, m_act, pad0;
  // schedule state: every sequence walks through the staged schedule at its own pace
  int stage, pos, phase, snap, step_ready;
  int last_p1;  // 1 + id of the stage this sequence completed last (0: none since the last reset); stage 3 starts from the
                // primal-dual point of stage 2.2 when that is what ran before it
  int warm;     // this stage was warm started
  int dyn;      // the durations have left their input values (stage 3 ran): spline tables and Jacobian columns are run-time data
  int band_ovf; // a coupling fell outside the band sized by the layout (stage 3 moved a polynomial too far): the stage fails
  int kw_req;   // the KKT kernel asks for Kwork <- Kbase to be refreshed by the side-stream copy before its next launch
  int st_status[6], st_iters[6];
  double mu, delta_w, sf, theta_max, theta_min, mu_filter, tau;
  double f, E0, viol_u, dual_u, compl_u;          // error measures at the current iterate
  double phi0, theta0, dphi, a_pr, a_du;          // line-search inputs produced by the KKT kernel
  double dw_floor;                                // current floor of delta_w (adaptive: CHD_AF_N)
  int af_cnt, af_off;                             // consecutive full steps taken at the floor; 1: the lowered floor was taken back for this stage
  int af_it, af_pad;                              // iteration of the first drop of the floor
  double af_E;                                    // scaled error at that iteration
  double theta_ref;                               // theta at the first iteration of the stage (nonlinearity guard of stage 3)
  double filt[2 * CHD_FILT_MAX];
  double st_stat[6][4];                           // per stage at its end: f, E0 (scaled NLP error), unscaled constraint violation, unscaled dual infeasibility
  double prof[8];   // clock64 cycles per phase of chd_k_kkt (0 errors, 1 assembly, 2 factor, 3 border, 4 back-subst, 5 step recovery; inside 2: 6 warp 0's next diagonal tile, 7 the trailing updates)
};

struct ChdStageDev {
  unsigned set_mask;
  int max_iter;
  int snap_after;   // SaveSolution snapshot written when the stage ends (-1: none)
  int opt_dur;      // stage 3: the phase durations are unknowns (as switch times), warm start from the previous stage
  double w_data[3], w_vel[3], w_acc[3], w_dur;
};

struct ChdDev {
  int B, S, Pmax, n_max, m_max, slots_max, sets_max, tab_max, F_max, Kd_max, Kr_max, Na_max, nb_max, w_max, par_stride,
      n_ee_max, fo_max, Ph_max, win_smem, nbc_max, Q, Qfix, nbt, win_tiles, pan_doubles;
  size_t kstride;                             // doubles per sequence of a tile-format KKT buffer (band | bord | corn)
                                              // (win_smem .. pan_doubles, kstride, scratch_stride: ChdKktPlan)
  // ---- static layout ----
  const ChdSeq* seq;
  // poly_T / poly_tend / phase_tend / ent_col are rewritten on the device once stage 3 moves the durations
  double *poly_T, *poly_tend;
  const double *node_const, *par, *t_dyn, *t_rom, *t_data, *row_lo, *row_hi, *dur0;
  const int *node_var, *itab, *ent_ptr, *var_kkt, *row_kkt, *row_set, *poly_ph;
  int* ent_col;
  double *poly_Tt, *poly_tendt;                // tables of the line search's trial durations (stage 3)
  double* jty;                                // B x n_max  J^T y accumulator of sequences with run-time columns
  const int *ent_row, *col_ptr, *col_ent;      // row of every slot; slots by column
  const ChdSet* sets;
  double* phase_tend;                         // B x n_ee_max x Ph_max cumulative phase end times
  // ---- iterate ----
  double *x, *xt, *dx, *grad;                 // B x n_max
  double *g, *gt;                             // B x m_max   (unscaled constraint values at x / trial x)
  double* Jv;                                 // B x slots_max
  int* rflag;                                 // B x m_max
  unsigned char* unobs;                       // B x n_max  foot-motion node values without cost curvature (chd_hess_build)
  double *sc, *dL, *dU, *s, *y, *zL, *zU, *ds, *dy, *dzL, *dzU;  // B x m_max
  double* cost;                               // B x 2 (current, trial)
  // ---- KKT ----
  double* Kwork;                              // B x kstride  KKT matrix of the current iteration, overwritten by its factors
  double* Kbase;                              // B x kstride  per-stage constant part (Gauss-Newton cost Hessian)
  double* sol;                                // B x (Na_max + nb_max)
  double* scratch;                            // per-sequence vectors + elimination window when they do not fit in shared memory
  double *rhs0, *rhs1;                        // right-hand side of the KKT system as rhs0 + mu * rhs1 (chd_k_asm), [B][Na_max + nb_max]
  size_t scratch_stride;                      // doubles per sequence in `scratch`
  ChdIpm* ipm;                                // B
  const ChdStageDev* stages;                  // B x 6 stage configurations, [b * 6 + stage id] (chd_stage)
  int sched[8], nsched;                       // stage ids of the running schedule
  double* snapshots;                          // 3 x B x fo_max x (6 + 7 n_ee_max)
};

// Admission of queued clips into freed slots (chd_k_admit, chd_queue.cu).  A segment is one per-sequence row of a
// device array: the admitted slot's row is copied from the clip's staged record, or zeroed (src < 0).
#define CHD_ADMIT_SEGS 64
struct ChdAdmitSeg {
  char* dst;             // row of slot 0
  size_t slot_bytes;     // distance between the rows of two slots
  size_t bytes;          // bytes of one row
  long long src;         // offset of the row in a clip record; -1: zero fill
};
struct ChdAdmit {
  const char* rec;       // staged records, rec_bytes apart: record j goes to slot slot[j]
  size_t rec_bytes;
  const int* slot;
  int nseg;
  ChdAdmitSeg seg[CHD_ADMIT_SEGS];
};

// IPM constants (Opts of oracle/ipm_oracle.cpp; IPOPT defaults unless noted)
#define CHD_TOL 1e-3            /* phys_optim.cpp:578 */
#define CHD_CONSTR_VIOL_TOL 1e-4
#define CHD_DUAL_INF_TOL 1.0
#define CHD_COMPL_INF_TOL 1e-4
#define CHD_MU_INIT 0.1
#define CHD_KAPPA_EPS 10.0
#define CHD_KAPPA_MU 0.2
#define CHD_THETA_MU 1.5
#define CHD_TAU_MIN 0.99
#define CHD_KAPPA1 1e-2
#define CHD_KAPPA2 1e-2
#define CHD_KAPPA_SIGMA 1e10
#define CHD_S_MAX 100.0
#define CHD_SCAL_MAX_GRAD 100.0
#define CHD_BOUND_RELAX 1e-8
#define CHD_DELTA_W0 1e-4
#define CHD_DELTA_C 1e-8
#define CHD_DW_POLISH 1.0   /* Levenberg-Marquardt weight of a feasibility-polish step (every test but the unscaled violation passes) */
#define CHD_DW_MIN 1e-8
#define CHD_AF_N 10          /* after this many consecutive full steps taken at the floor of delta_w the floor drops by 10x ... */
#define CHD_AF_MIN 1e-10     /* ... down to this; a backtrack, or an error that has not halved after 30 iterations, restores CHD_DW_MIN for the stage */
#define CHD_DW_MAX 1e4
#define CHD_DW_INC 4.0
#define CHD_DW_DEC 3.0
#define CHD_MAX_BACKTRACK 25
#define CHD_GAMMA_THETA 1e-5
#define CHD_GAMMA_PHI 1e-5
#define CHD_S_PHI 2.3
#define CHD_S_THETA 1.1
#define CHD_ETA_PHI 1e-8
#define CHD_INF 1e19

#if defined(__CUDACC__) || defined(CHD_HOST_EMU)
// Interior-point terms of one constraint row with flags f, defined once for the assembly, the KKT kernel's error
// measures and step recovery, and the line search: theta and phi at the current iterate and at a trial point are the
// same functions.  Bounds and multipliers are taken by reference so that a row without the bound never reads them.
struct ChdGaps { double L, U; };   // s - dL and dU - s; 1.0 for a bound the row does not have
__device__ __forceinline__ ChdGaps chd_row_gaps(int f, double s, const double& dL, const double& dU) {
  return {(f & CHD_ROW_HASL) ? s - dL : 1.0, (f & CHD_ROW_HASU) ? dU - s : 1.0};
}
struct ChdSigma {   // zL / gapL and zU / gapU (0.0 for a bound the row does not have); their sum is the barrier weight
  double L, U;
  __device__ __forceinline__ double sum() const { return L + U; }
};
__device__ __forceinline__ ChdSigma chd_row_sigma(int f, ChdGaps gap, const double& zL, const double& zU) {
  return {(f & CHD_ROW_HASL) ? zL / gap.L : 0.0, (f & CHD_ROW_HASU) ? zU / gap.U : 0.0};
}
// coefficient of the barrier parameter in the row's right-hand side
__device__ __forceinline__ double chd_row_mu_coef(int f, ChdGaps gap) {
  return ((f & CHD_ROW_HASL) ? 1.0 / gap.L : 0.0) - ((f & CHD_ROW_HASU) ? 1.0 / gap.U : 0.0);
}
// primal residual of the scaled constraint value d (theta sums its magnitude, the constraint violation takes the largest)
__device__ __forceinline__ double chd_row_res(int f, double d, const double& dL, const double& s) {
  return (f & CHD_ROW_EQ) ? d - dL : d - s;
}
// barrier term: acc - mu log gapL - mu log gapU, over the bounds the row has
__device__ __forceinline__ void chd_row_barrier(int f, double mu, ChdGaps gap, double& acc) {
  if (f & CHD_ROW_HASL) acc -= mu * log(gap.L);
  if (f & CHD_ROW_HASU) acc -= mu * log(gap.U);
}

// configuration of `stage` for sequence b: every sequence has its own six rows (its cost weights)
__device__ __forceinline__ const ChdStageDev& chd_stage(const ChdDev& D, int b, int stage) { return D.stages[(size_t)b * 6 + stage]; }

// puts one sequence at the start of the schedule D.sched (chd_k_sched_reset, chd_k_admit)
__device__ __forceinline__ void chd_sched_begin(const ChdDev& D, ChdIpm& I) {
  I.pos = 0, I.stage = D.sched[0], I.phase = CHD_PH_BEGIN, I.snap = -1, I.step_ready = 0, I.kw_req = 0, I.status = 1;
  for (int q = 0; q < 6; ++q) I.st_status[q] = -9, I.st_iters[q] = 0;
}

// a stage ended for this sequence: record its outcome, request the snapshot, move on in the schedule
// (phys_optim.cpp:709-749: stage 4 only runs when stage 3 did not succeed)
__device__ __forceinline__ void chd_stage_advance(const ChdDev& D, ChdIpm& I, int status, int snap_after) {
  I.st_status[I.stage] = status;
  I.st_iters[I.stage] = I.iter;
  I.st_stat[I.stage][0] = I.f, I.st_stat[I.stage][1] = I.E0, I.st_stat[I.stage][2] = I.viol_u, I.st_stat[I.stage][3] = I.dual_u;
  I.last_p1 = I.stage + 1;
  I.step_ready = 0;
  I.kw_req = 0;
  I.pos += 1;
  if (I.stage == CHD_STAGE_3 && status == 0 && I.pos < D.nsched && D.sched[I.pos] == CHD_STAGE_4) I.pos += 1;
  else if (I.stage == CHD_STAGE_3 && status != 0 && I.pos < D.nsched && D.sched[I.pos] == CHD_STAGE_4) snap_after = -1;  // SaveSolution comes after stage 4 (:758)
  I.snap = snap_after;
  if (I.pos < D.nsched) I.stage = D.sched[I.pos], I.phase = CHD_PH_BEGIN;
  else I.phase = CHD_PH_FINISHED;
}
#endif
