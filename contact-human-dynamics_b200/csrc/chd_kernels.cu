// sm_90a kernels of the batched interior-point trajectory optimiser (product code).
// One CTA owns one sequence in every kernel; sequences are independent NLPs (SURVEY.md 8(e)).
//
//   chd_k_stage_begin : row activity flags + IPM state reset for a stage
//   chd_k_eval        : f, grad f, g, Jacobian slot values at the current x       (HBM/L2 streaming)
//   chd_k_init        : gradient-based scaling, relaxed bounds, slack / multiplier initialisation
//   chd_k_kkt         : error measures + barrier update, condensed KKT assembly (band + border),
//                       unpivoted band LDL^T with dense border, triangular solves, step recovery
//   chd_k_linesearch  : filter backtracking line search (trial point in shared memory, or in global memory when the
//                       iterate is too long for it), update
//   chd_k_sample      : SaveSolution sampling (phys_optim.cpp:63-143)
//   chd_k_cost_terms  : the unweighted cost terms at the current x
#include <cuda_runtime.h>

#include "chd_block.cuh"
#include "chd_eval.cuh"

// ------------------------------------------------------------------ stage begin -------------------
__global__ void chd_k_stage_begin(ChdDev D) {
  const int b = blockIdx.x;
  if (D.ipm[b].phase != CHD_PH_BEGIN) return;
  const ChdStageDev sg = chd_stage(D, b, D.ipm[b].stage);
  const int max_iter = sg.max_iter;
  const ChdSeq* h = D.seq + b;
  if (sg.opt_dur && h->n_dur == 0) {
    // more phase durations than the dense border holds (CHD_MAX_DUR) and no banded switch times: stage 3 is not
    // attempted; like the reference
    // after a failed stage 3 the schedule continues with the fixed-duration stage 4 (phys_optim.cpp:713-749)
    __syncthreads();
    if (threadIdx.x == 0) {
      D.ipm[b].iter = 0;
      chd_stage_advance(D, b, D.ipm[b], -3);
    }
    return;
  }
  // stage 3 continues from the primal-dual point stage 2.2 left behind (same rows + the duration rows)
  const bool warm = sg.opt_dur && D.ipm[b].last_p1 == CHD_STAGE_22 + 1;
  int* rf = D.rflag + (size_t)b * D.m_max;
  const double* lo = D.row_lo + (size_t)b * D.m_max;
  const double* hi = D.row_hi + (size_t)b * D.m_max;
  const int* rset = D.row_set + (size_t)b * D.m_max;
  for (int r = threadIdx.x; r < D.m_max; r += blockDim.x) {
    int f = 0;
    if (r < h->m && (sg.set_mask & CHD_MASK(rset[r]))) {
      f = CHD_ROW_ACTIVE;
      if (lo[r] == hi[r]) f |= CHD_ROW_EQ;
      else {
        if (lo[r] > -CHD_INF) f |= CHD_ROW_HASL;
        if (hi[r] < CHD_INF) f |= CHD_ROW_HASU;
      }
      if (warm && (rf[r] & CHD_ROW_ACTIVE)) f |= CHD_ROW_WARM;   // keeps scaling, slack and multipliers (chd_k_init)
    }
    rf[r] = f;
    D.g[(size_t)b * D.m_max + r] = 0.0;
  }
  if (sg.opt_dur) {
    // from here on the spline tables follow the durations held in x (PhaseDurations::SetVariables)
    ChdCtx c;
    chd_make_ctx(D, b, D.x + (size_t)b * D.n_max, c);
    chd_tables_from_x(c, c.x, D.poly_T + (size_t)b * D.S * D.Pmax, D.poly_tend + (size_t)b * D.S * D.Pmax,
                      D.phase_tend + (size_t)b * D.n_ee_max * D.Ph_max);
  }
  if (threadIdx.x == 0) {
    ChdIpm& I = D.ipm[b];
    I.status = 1;
    I.iter = 0;
    I.nfilt = 0;
    I.ls_fail = 0;
    I.max_iter = max_iter;
    I.warm = warm;
    if (sg.opt_dur) I.dyn = 1;
    I.band_ovf = 0;
    if (!warm) I.mu = CHD_MU_INIT, I.sf = 1.0, I.delta_w = CHD_DELTA_W0;
    else I.delta_w = fmax(I.delta_w, CHD_DELTA_W0);
    I.mu_filter = -1.0;
    I.dw_floor = CHD_DW_MIN, I.af_cnt = 0, I.af_off = 0, I.af_it = 0, I.af_E = 0.0;
    for (int q = 0; q < 8; ++q) I.prof[q] = 0.0;
    for (int q = 40; q < 48; ++q) I.filt[q] = 0.0;
  }
}

// ------------------------------------------------------------------ evaluation --------------------
// dynamic shared memory: x[n_max] | grad[n_max] | red[CHD_THREADS]
// GLOBAL (iterates too long for shared memory, chd_iter_form in chd_api.cu): red[CHD_THREADS] only; x is read from
// D.x and the gradient accumulates in the sequence's row of D.grad (fp64 global atomics: this CTA is the row's only
// writer, and the barrier after the zeroing orders it before every addition)
template <bool GLOBAL>
__global__ void __launch_bounds__(CHD_THREADS) chd_k_eval(ChdDev D) {
  extern __shared__ double sm[];
  const int b = blockIdx.x;
  if (D.ipm[b].phase != CHD_PH_BEGIN && D.ipm[b].phase != CHD_PH_RUN) return;
  const ChdStageDev sg = chd_stage(D, b, D.ipm[b].stage);
  const ChdSeq* h = D.seq + b;
  const double* xs;
  double *gs, *red;
  if (GLOBAL) {
    xs = D.x + (size_t)b * D.n_max;
    gs = D.grad + (size_t)b * D.n_max;
    red = sm;
    for (int i = threadIdx.x; i < h->n; i += blockDim.x) gs[i] = 0.0;
  } else {
    double* xsm = sm;
    gs = sm + D.n_max;
    red = sm + 2 * D.n_max;
    const double* x = D.x + (size_t)b * D.n_max;
    for (int i = threadIdx.x; i < h->n; i += blockDim.x) xsm[i] = x[i], gs[i] = 0.0;
    xs = xsm;
  }
  __syncthreads();
  ChdCtx c;
  chd_make_ctx(D, b, xs, c);
  c.dyn = D.ipm[b].dyn;
  c.opt_dur = sg.opt_dur;
  chd_eval_all<true>(c, sg, D.g + (size_t)b * D.m_max, D.Jv + (size_t)b * D.slots_max, gs, D.cost + 2 * b, red);
  if (!GLOBAL) {
    double* grad = D.grad + (size_t)b * D.n_max;
    for (int i = threadIdx.x; i < h->n; i += blockDim.x) grad[i] = gs[i];
  }
}
template __global__ void chd_k_eval<false>(ChdDev D);
template __global__ void chd_k_eval<true>(ChdDev D);

// ------------------------------------------------------------------ init --------------------------
// IPOPT gradient-based scaling (nlp_scaling_max_gradient 100), relaxed bounds, slack push, z = 1, y = 0.
__global__ void __launch_bounds__(CHD_THREADS) chd_k_init(ChdDev D) {
  __shared__ double red[CHD_THREADS];
  const int b = blockIdx.x;
  if (D.ipm[b].phase != CHD_PH_BEGIN) return;
  const ChdSeq* h = D.seq + b;
  const size_t ro = (size_t)b * D.m_max;
  const int* vk = D.var_kkt + (size_t)b * D.n_max;
  const double* grad = D.grad + (size_t)b * D.n_max;
  double gm = 0.0;
  for (int i = threadIdx.x; i < h->n; i += blockDim.x)
    if (vk[i] >= 0) gm = fmax(gm, fabs(grad[i]));
  gm = chd_block_max(gm, red);
  const bool warm = D.ipm[b].warm;
  const double mu0 = D.ipm[b].mu;
  const double sf = warm ? D.ipm[b].sf : (gm > CHD_SCAL_MAX_GRAD ? CHD_SCAL_MAX_GRAD / gm : 1.0);
  const int* ep = D.ent_ptr + (size_t)b * (D.m_max + 1);
  const int* ec = D.ent_col + (size_t)b * D.slots_max;
  const double* Jv = D.Jv + (size_t)b * D.slots_max;
  int nb_l = 0;
  for (int r = threadIdx.x; r < h->m; r += blockDim.x) {
    const int f = D.rflag[ro + r];
    if (!(f & CHD_ROW_ACTIVE)) continue;
    if (f & CHD_ROW_WARM) {   // inherited from stage 2.2: scaling, bounds, slack and multipliers stay
      if (!(f & CHD_ROW_EQ)) nb_l += ((f & CHD_ROW_HASL) ? 1 : 0) + ((f & CHD_ROW_HASU) ? 1 : 0);
      continue;
    }
    double rm = 0.0;
    for (int e = ep[r]; e < ep[r + 1]; ++e) {
      const int col = ec[e];
      if (col >= 0 && vk[col] >= 0) rm = fmax(rm, fabs(Jv[e]));
    }
    double sc = rm > CHD_SCAL_MAX_GRAD ? CHD_SCAL_MAX_GRAD / rm : 1.0;
    sc = fmax(sc, 1e-8);
    D.sc[ro + r] = sc;
    const double lo = D.row_lo[ro + r] * sc, hi = D.row_hi[ro + r] * sc;
    const double d = sc * D.g[ro + r];
    D.y[ro + r] = 0.0;
    if (f & CHD_ROW_EQ) {
      D.dL[ro + r] = lo, D.dU[ro + r] = hi, D.s[ro + r] = d, D.zL[ro + r] = 0.0, D.zU[ro + r] = 0.0;
      continue;
    }
    const bool hl = f & CHD_ROW_HASL, hu = f & CHD_ROW_HASU;
    const double dL = hl ? lo - CHD_BOUND_RELAX * fmax(1.0, fabs(lo)) : -INFINITY;
    const double dU = hu ? hi + CHD_BOUND_RELAX * fmax(1.0, fabs(hi)) : INFINITY;
    double s = d;
    if (hl) {
      double pL = CHD_KAPPA1 * fmax(1.0, fabs(dL));
      if (hu) pL = fmin(pL, CHD_KAPPA2 * (dU - dL));
      s = fmax(s, dL + pL);
    }
    if (hu) {
      double pU = CHD_KAPPA1 * fmax(1.0, fabs(dU));
      if (hl) pU = fmin(pU, CHD_KAPPA2 * (dU - dL));
      s = fmin(s, dU - pU);
    }
    D.dL[ro + r] = dL, D.dU[ro + r] = dU, D.s[ro + r] = s;
    // new rows of a warm-started stage start on the central path of the inherited barrier parameter
    D.zL[ro + r] = hl ? (warm ? mu0 / (s - dL) : 1.0) : 0.0;
    D.zU[ro + r] = hu ? (warm ? mu0 / (dU - s) : 1.0) : 0.0;
    nb_l += (hl ? 1 : 0) + (hu ? 1 : 0);
  }
  const double nbnd = chd_block_sum((double)nb_l, red);
  int act = 0;
  for (int r = threadIdx.x; r < h->m; r += blockDim.x) act += (D.rflag[ro + r] & CHD_ROW_ACTIVE) ? 1 : 0;
  const double nact = chd_block_sum((double)act, red);
  if (threadIdx.x == 0) {
    D.ipm[b].sf = sf;
    D.ipm[b].n_bounds = (int)nbnd;
    D.ipm[b].m_act = (int)nact;
  }
}

// ------------------------------------------------------------------ line search -------------------
// dynamic shared memory: xt[n_max] | red[CHD_THREADS]
// GLOBAL (iterates too long for shared memory, chd_iter_form in chd_api.cu): red[CHD_THREADS] only; the trial point is
// built in the sequence's row of D.xt
template <bool GLOBAL>
__global__ void __launch_bounds__(CHD_THREADS) chd_k_linesearch(ChdDev D) {
  extern __shared__ double sm[];
  __shared__ int s_ok, s_ftype, s_trust;
  __shared__ double s_cost;
  const int b = blockIdx.x;
  ChdIpm& I = D.ipm[b];
  if (I.phase != CHD_PH_RUN || !I.step_ready) return;
  const ChdStageDev& sg = chd_stage(D, b, I.stage);
  const ChdSeq* h = D.seq + b;
  const int n = h->n, m = h->m, tid = threadIdx.x, nt = blockDim.x;
  const size_t ro = (size_t)b * D.m_max, vo = (size_t)b * D.n_max;
  const int* rf = D.rflag + ro;
  double* xt = GLOBAL ? D.xt + vo : sm;
  double* red = GLOBAL ? sm : sm + D.n_max;
  const double* x = D.x + vo;
  const double* dx = D.dx + vo;
  double* gt = D.gt + ro;
  const double mu = I.mu, sf = I.sf, theta = I.theta0, phi0 = I.phi0, dphi = I.dphi, a_pr = I.a_pr, a_du = I.a_du;
  if (a_pr == 0.0 && dphi == 0.0) {  // failed factorisation: nothing to do this iteration
    if (tid == 0) I.iter += 1, I.step_ready = 0;
    return;
  }
  ChdCtx c;
  chd_make_ctx(D, b, xt, c);
  c.dyn = I.dyn;
  c.opt_dur = sg.opt_dur;
  if (sg.opt_dur) {   // the trial durations get their own spline tables
    c.poly_T = D.poly_Tt + (size_t)b * D.S * D.Pmax;
    c.poly_tend = D.poly_tendt + (size_t)b * D.S * D.Pmax;
    const size_t cnt = (size_t)D.S * D.Pmax;
    for (size_t i = tid; i < cnt; i += nt) {   // base splines and padding: fixed
      D.poly_Tt[(size_t)b * cnt + i] = D.poly_T[(size_t)b * cnt + i];
      D.poly_tendt[(size_t)b * cnt + i] = D.poly_tend[(size_t)b * cnt + i];
    }
    __syncthreads();
  }
  const double theta_ref = I.theta_ref;
  double alpha = a_pr;
  int ls = 0;
  bool accepted = false, ftype = false;
  for (ls = 0; ls < CHD_MAX_BACKTRACK; ++ls) {
    for (int i = tid; i < n; i += nt) xt[i] = x[i] + alpha * dx[i];
    __syncthreads();
    if (sg.opt_dur) {
      // trust region of stage 3: every switch time stays within CHD_TAU_TRUST of its input value (the band of the KKT
      // matrix is sized for the polynomials that can reach a sample time within that distance)
      if (tid == 0) s_trust = 0;
      __syncthreads();
      if (tid < h->n_ee) {
        double t = 0.0, t0 = 0.0;
        int bad = 0;
        for (int k = 0; k < h->n_phases[tid] - 1; ++k) {
          t += xt[h->dur_xoff[tid] + k];
          t0 += c.dur0[(size_t)tid * c.Ph_max + k];
          if (fabs(t - t0) > CHD_TAU_TRUST) bad = 1;
        }
        if (bad) s_trust = 1;
      }
      chd_tables_from_x(c, xt, D.poly_Tt + (size_t)b * D.S * D.Pmax, D.poly_tendt + (size_t)b * D.S * D.Pmax, nullptr);
      __syncthreads();
    }
    chd_eval_all<false>(c, sg, gt, nullptr, nullptr, &s_cost, red);
    double a_th = 0.0, a_bar = 0.0;
    for (int r = tid; r < m; r += nt) {
      const int f = rf[r];
      if (!(f & CHD_ROW_ACTIVE)) continue;
      const bool eq = f & CHD_ROW_EQ;
      const double st = eq ? 0.0 : D.s[ro + r] + alpha * D.ds[ro + r];   // trial slack (an equality row has none)
      a_th += fabs(chd_row_res(f, D.sc[ro + r] * gt[r], D.dL[ro + r], st));
      if (!eq) chd_row_barrier(f, mu, chd_row_gaps(f, st, D.dL[ro + r], D.dU[ro + r]), a_bar);
    }
    const double theta_t = chd_block_sum(a_th, red);
    const double bar_t = chd_block_sum(a_bar, red);
    if (tid == 0) {
      const double phit = sf * s_cost + bar_t;
      bool ok = isfinite(phit) && isfinite(theta_t) && theta_t <= I.theta_max;
      // nonlinearity guard of stage 3: the linearised constraints predict theta(alpha) = (1 - alpha) theta; the trial
      // point is refused while the second-order error exceeds the predicted decrease (or a small absolute level)
      if (sg.opt_dur && s_trust) ok = false;
      if (sg.opt_dur && ok && theta_t - (1.0 - alpha) * theta > CHD_NL_GUARD * fmax(alpha * theta, CHD_NL_FLOOR * fmax(1.0, theta_ref))) ok = false;
      for (int q = 0; ok && q < I.nfilt; ++q)
        if (theta_t >= I.filt[2 * q] && phit >= I.filt[2 * q + 1]) ok = false;
      bool acc = false, ft = false;
      if (ok) {
        const bool switching = dphi < 0 && alpha * pow(-dphi, CHD_S_PHI) > pow(theta, CHD_S_THETA);
        const bool armijo = phit <= phi0 + CHD_ETA_PHI * alpha * dphi;
        if (theta <= I.theta_min && switching) {
          if (armijo) acc = true, ft = true;
        } else if (theta_t <= (1 - CHD_GAMMA_THETA) * theta || phit <= phi0 - CHD_GAMMA_PHI * theta) {
          acc = true;
          ft = switching && armijo;
        }
      }
      s_ok = acc, s_ftype = ft;
    }
    __syncthreads();
    accepted = s_ok, ftype = s_ftype;
    __syncthreads();
    if (accepted) break;
    alpha *= 0.5;
  }
  if (!accepted) {
    alpha *= 2.0;  // the last (smallest) trial step is taken, as in the filter line search of oracle/ipm_oracle.cpp
    ls = CHD_MAX_BACKTRACK;
  }
  // x was left at the accepted trial point in xt
  double* xg = D.x + vo;
  for (int i = tid; i < n; i += nt) xg[i] = xt[i];
  if (sg.opt_dur) {
    __syncthreads();
    chd_tables_from_x(c, xt, D.poly_T + (size_t)b * D.S * D.Pmax, D.poly_tend + (size_t)b * D.S * D.Pmax,
                      D.phase_tend + (size_t)b * D.n_ee_max * D.Ph_max);
  }
  for (int r = tid; r < m; r += nt) {
    const int f = rf[r];
    if (!(f & CHD_ROW_ACTIVE)) continue;
    D.y[ro + r] += alpha * D.dy[ro + r];
    if (f & CHD_ROW_EQ) continue;
    const double s = D.s[ro + r] + alpha * D.ds[ro + r];
    D.s[ro + r] = s;
    const ChdGaps gap = chd_row_gaps(f, s, D.dL[ro + r], D.dU[ro + r]);
    if (f & CHD_ROW_HASL) {
      double z = D.zL[ro + r] + a_du * D.dzL[ro + r];
      z = fmin(fmax(z, mu / (CHD_KAPPA_SIGMA * gap.L)), CHD_KAPPA_SIGMA * mu / gap.L);
      D.zL[ro + r] = z;
    }
    if (f & CHD_ROW_HASU) {
      double z = D.zU[ro + r] + a_du * D.dzU[ro + r];
      z = fmin(fmax(z, mu / (CHD_KAPPA_SIGMA * gap.U)), CHD_KAPPA_SIGMA * mu / gap.U);
      D.zU[ro + r] = z;
    }
  }
  if (tid == 0) {
    if (accepted && !ftype && I.nfilt < CHD_FILT_MAX) {
      I.filt[2 * I.nfilt] = (1 - CHD_GAMMA_THETA) * theta;
      I.filt[2 * I.nfilt + 1] = phi0 - CHD_GAMMA_PHI * theta;
      I.nfilt += 1;
    }
    if (!accepted) I.ls_fail += 1;
    // Levenberg-Marquardt style adaptation of the primal regularisation
    // Adaptive floor of the Levenberg-Marquardt weight.  Sequences that take full steps at the floor converge linearly at
    // a rate set by the floor (the reduced Hessian along force directions is ~1e-10): after CHD_AF_N such steps in a row
    // the floor drops by 10x (not below CHD_AF_MIN).  The lower floor is a gamble (the Gauss-Newton model misses
    // constraint curvature: some sequences start to oscillate or crawl), so it is taken back for the rest of the stage
    // at the first backtrack, or when the scaled error has not halved 30 iterations after the first drop.
    if (!I.af_off) {
      const bool at_floor = ls == 0 && I.delta_w <= I.dw_floor * 1.0000001;
      if (I.dw_floor < CHD_DW_MIN) {
        if (ls > 0 || (I.iter - I.af_it >= 30 && I.E0 > 0.5 * I.af_E)) I.dw_floor = CHD_DW_MIN, I.af_off = 1;
        else if (at_floor && ++I.af_cnt >= CHD_AF_N) I.dw_floor = fmax(I.dw_floor * 0.1, CHD_AF_MIN), I.af_cnt = 0;
      } else if (at_floor) {
        if (++I.af_cnt >= CHD_AF_N) I.dw_floor = fmax(I.dw_floor * 0.1, CHD_AF_MIN), I.af_cnt = 0, I.af_E = I.E0, I.af_it = I.iter;
      } else if (ls > 0) {
        I.af_cnt = 0;
      }
    }
    if (ls == 0) I.delta_w = fmax(I.delta_w / CHD_DW_DEC, I.dw_floor);
    else I.delta_w = fmin(I.delta_w * pow(CHD_DW_INC, (double)min(ls, 3)), CHD_DW_MAX);
    I.iter += 1;
    I.step_ready = 0;
  }
}
template __global__ void chd_k_linesearch<false>(ChdDev D);
template __global__ void chd_k_linesearch<true>(ChdDev D);

// ------------------------------------------------------------------ cost terms --------------------
// The CHD_PHYS_N_TERMS unweighted cost terms of a sequence at the current x (chd_phys_cost_terms): data fit of the base
// position, the base orientation and the feet; velocity smoothing (same order); acceleration smoothing (same order);
// duration change.  The cost items of chd_eval_all with weight 1, all of them whatever the stage, on the spline tables
// of the current durations.  Per-thread accumulators and a fixed-order tree reduction, no atomics: a sequence's terms
// are bitwise the same run to run and in any batch with the same strides.  finished_only: only the sequences whose
// schedule is over (the slots a queue harvests at a check point).  out: B x CHD_PHYS_N_TERMS.
__global__ void __launch_bounds__(CHD_TERMS_THREADS) chd_k_cost_terms(ChdDev D, int finished_only, double* out) {
  __shared__ double red[CHD_PHYS_N_TERMS][CHD_TERMS_THREADS];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (finished_only && D.ipm[b].phase != CHD_PH_FINISHED) return;
  ChdCtx c;
  chd_make_ctx(D, b, D.x + (size_t)b * D.n_max, c);
  const ChdSeq* h = c.h;
  double acc[CHD_PHYS_N_TERMS];
#pragma unroll
  for (int q = 0; q < CHD_PHYS_N_TERMS; ++q) acc[q] = 0.0;
  const int nsp = 2 + h->n_ee, F = h->F, ns = h->n_smooth;
  for (int it = tid; it < nsp * F; it += blockDim.x) {
    const int s = it / F, i = it % F, cls = s < 2 ? s : 2;
    const double d = chd_item_data<false>(c, s, i, 1.0, nullptr);
    const double v = i < ns ? chd_item_smooth<false>(c, s, i, 0, 1.0, nullptr) : 0.0;
    const double a = i < ns ? chd_item_smooth<false>(c, s, i, 1, 1.0, nullptr) : 0.0;
#pragma unroll
    for (int q = 0; q < 3; ++q)
      if (q == cls) acc[q] += d, acc[3 + q] += v, acc[6 + q] += a;
  }
  if (h->n_dur)
    for (int ee = 0; ee < h->n_ee; ++ee)
      for (int k = tid; k < h->n_phases[ee] - 1; k += blockDim.x) acc[9] += chd_item_durcost<false>(c, ee, k, 1.0, nullptr);
#pragma unroll
  for (int q = 0; q < CHD_PHYS_N_TERMS; ++q) red[q][tid] = acc[q];
  __syncthreads();
  for (int off = blockDim.x / 2; off > 0; off >>= 1) {
    if (tid < off) {
#pragma unroll
      for (int q = 0; q < CHD_PHYS_N_TERMS; ++q) red[q][tid] += red[q][tid + off];
    }
    __syncthreads();
  }
  if (tid < CHD_PHYS_N_TERMS) out[(size_t)b * CHD_PHYS_N_TERMS + tid] = red[tid][0];
}

// ------------------------------------------------------------------ sampling ----------------------
// SaveSolution (phys_optim.cpp:63-143): t accumulates dt while t <= T + 1e-5.
// out: B x fo_max x (6 + 7 n_ee_max)
__device__ void chd_sample_seq(const ChdDev& D, int b, double* out, int* frames_out) {
  const ChdSeq* h = D.seq + b;
  ChdCtx c;
  chd_make_ctx(D, b, D.x + (size_t)b * D.n_max, c);
  const int n_ee = h->n_ee, stride = 6 + 7 * D.n_ee_max;
  double tot = 0.0;
  for (int k = 0; k < h->sp_npoly[0]; ++k) tot += c.poly_T[k];  // Spline::GetTotalTime of base_linear
  const int nf = (int)((tot + 1e-5) / h->dt) + 1;
  if (threadIdx.x == 0 && frames_out) frames_out[b] = nf;
  // sample times: the reference accumulates t += dt; thread j reproduces the same rounding for its frames by
  // continuing its own accumulation (frames i, i + blockDim, ...) from a prefix it sums once
  double t = 0.0;
  int at = 0;
  for (int i = threadIdx.x; i < nf; i += blockDim.x) {
    for (; at < i; ++at) t += h->dt;
    if (!(t <= tot + 1e-5)) continue;
    double* o = out + ((size_t)b * D.fo_max + i) * stride;
    ChdSpl P;
    double v[3];
    chd_spl_at(c, 0, t, P);
    chd_spl_val(c, P, 0, v);
    o[0] = v[0], o[1] = v[1], o[2] = v[2];
    chd_spl_at(c, 1, t, P);
    chd_spl_val(c, P, 0, v);
    for (int d = 0; d < 3; ++d) o[3 + d] = v[d] / M_PI * 180;
    for (int ee = 0; ee < n_ee; ++ee) {
      chd_spl_at(c, chd_sp_motion(ee), t, P);
      chd_spl_val(c, P, 0, v);
      for (int d = 0; d < 3; ++d) o[6 + 3 * ee + d] = v[d];
      chd_spl_at(c, chd_sp_force(n_ee, ee), t, P);
      chd_spl_val(c, P, 0, v);
      for (int d = 0; d < 3; ++d) o[6 + 3 * D.n_ee_max + 3 * ee + d] = v[d];
      // PhaseDurations::IsContactPhase (phys_optim.cpp:135): phase id parity against the start flag
      {
        const double* pt = D.phase_tend + ((size_t)b * D.n_ee_max + ee) * D.Ph_max;
        double tl;
        const int ph = chd_locate(pt, h->n_phases[ee], t, &tl);
        o[6 + 6 * D.n_ee_max + ee] = ((ph % 2 == 0) ? h->start_contact[ee] : !h->start_contact[ee]) ? 1.0 : 0.0;
      }
    }
  }
}

__global__ void chd_k_sample(ChdDev D, double* out, int* frames_out) { chd_sample_seq(D, blockIdx.x, out, frames_out); }

// writes the SaveSolution snapshot of the sequences whose stage just ended (phys_optim.cpp:603,661,758)
__global__ void chd_k_snapshot(ChdDev D, int* frames_out) {
  const int b = blockIdx.x;
  const int snap = D.ipm[b].snap;
  if (snap < 0) return;
  const size_t stride = 6 + 7 * (size_t)D.n_ee_max;
  chd_sample_seq(D, b, D.snapshots + (size_t)snap * D.B * D.fo_max * stride, frames_out);
  __syncthreads();
  if (threadIdx.x == 0) D.ipm[b].snap = -1;
}

// spline tables from the durations in x for every sequence whose durations differ from the input ones
// (chd_phys_set_x with foreign durations); marks those sequences as run-time patterned
__global__ void chd_k_tables(ChdDev D) {
  const int b = blockIdx.x;
  const ChdSeq* h = D.seq + b;
  __shared__ int s_diff;
  if (threadIdx.x == 0) s_diff = 0;
  __syncthreads();
  const double* x = D.x + (size_t)b * D.n_max;
  for (int ee = 0; ee < h->n_ee && h->n_dur; ++ee)
    for (int k = threadIdx.x; k < h->n_phases[ee] - 1; k += blockDim.x)
      if (x[h->dur_xoff[ee] + k] != D.dur0[((size_t)b * D.n_ee_max + ee) * D.Ph_max + k]) s_diff = 1;
  __syncthreads();
  if (!s_diff && !D.ipm[b].dyn) return;
  ChdCtx c;
  chd_make_ctx(D, b, x, c);
  chd_tables_from_x(c, x, D.poly_T + (size_t)b * D.S * D.Pmax, D.poly_tend + (size_t)b * D.S * D.Pmax,
                    D.phase_tend + (size_t)b * D.n_ee_max * D.Ph_max);
  if (threadIdx.x == 0) D.ipm[b].dyn = 1;
}
// back to the input durations (chd_phys_reset): the host-built tables and columns are restored by the caller
__global__ void chd_k_clear_dyn(ChdDev D) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= D.B) return;
  D.ipm[b].dyn = 0, D.ipm[b].last_p1 = 0;
}

// puts every sequence at the start of the schedule D.sched
__global__ void chd_k_sched_reset(ChdDev D) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= D.B) return;
  chd_sched_begin(D, D.ipm[b]);
}
