// KKT kernels of the batched interior-point solver (product code, sm_90a).
//
//   chd_k_hess_base : once per stage -- Gauss-Newton Hessian of the (quadratic, fixed-duration) cost terms
//                     of data_cost.cpp / vel_smooth_cost.cpp, scaled by the objective scaling, in tile format (Kbase);
//                     with chd_k_hess_zero it also prepares Kwork of the stage's first iteration
//   chd_k_kcopy     : per iteration, side stream -- Kwork <- Kbase for the sequences that continue in their stage
//   chd_k_curv      : per iteration, side stream, after the line search -- y+ Jd^T Jd of the squared-distance rows
//   chd_k_asm       : per iteration, right before chd_k_kkt -- Jacobian dependent matrix entries and the right-hand
//                     side as rhs0 + mu * rhs1 (several CTAs per sequence: the cost is the L2 reductions)
//   chd_k_kkt       : per iteration, one CTA per sequence -- IPOPT error measures + barrier update, tiled band LDL^T
//                     with dense border (shared-memory window or, for wide bands, in place on Kwork; panel, trailing
//                     and corner updates on the FP64 tensor core), triangular solves, step recovery and
//                     fraction-to-the-boundary rule
//   chd_k_fp64_peak : DFMA / DMMA throughput probe for the roofline denominators of bench.py
// Replaces IPOPT's per-iteration MA57 factorisation (phys_optim.cpp:573) for the block-banded systems this NLP
// produces.
#include <cuda_runtime.h>

#include "chd_block.cuh"
#include "chd_eval.cuh"
#include "chd_kkt_tiles.cuh"

// Gauss-Newton Hessian of a least-squares cost sample by one warp: H += wgt * J^T J, where the sample residual (3 rows)
// is a signed sum over (up to two) located polynomials of B(deriv) node values.  Every Jacobian column is a 3-vector:
// wgt_q e_dim for a node slot, and -- stage 3, foot splines, positions -- the switch-time columns of chd_spl_tau.
// Entry e = polynomial * 14 + slot (12 node slots, 2 switch-time slots); ws: 28 x 4 doubles of per-warp scratch
// (kkt index or -1, column vector); the 28 x 28 pair loop is spread over the lanes.
__device__ __forceinline__ void chd_hess_sample(const ChdCtx& c, const ChdKT& K, const int* vk, int s, const ChdSpl* P, const double* sign, int np,
                                                int deriv, double wgt, int lane, double* ws) {
  const bool tau = c.opt_dur && s >= 2 && deriv == 0;
  if (lane < 28) {
    const int pa = lane / 14, q = lane % 14;
    double v0 = 0.0, v1 = 0.0, v2 = 0.0;
    int ia = -1;
    if (pa < np) {
      if (q < 12) {
        const int va = P[pa].var[q];
        const double wa = sign[pa] * chd_slot_w(P[pa], deriv, q);
        if (va >= 0 && wa != 0.0) {
          ia = vk[va];
          v0 = q % 3 == 0 ? wa : 0.0, v1 = q % 3 == 1 ? wa : 0.0, v2 = q % 3 == 2 ? wa : 0.0;
        }
      } else if (tau) {
        ChdTau u;
        chd_spl_tau(c, s, s - 2, P[pa], u);
        const int var = q == 12 ? u.va : u.vb;
        const double* dv = q == 12 ? u.da : u.db;
        if (var >= 0) ia = vk[var], v0 = sign[pa] * dv[0], v1 = sign[pa] * dv[1], v2 = sign[pa] * dv[2];
      }
    }
    ws[lane * 4 + 0] = (double)ia, ws[lane * 4 + 1] = v0, ws[lane * 4 + 2] = v1, ws[lane * 4 + 3] = v2;
  }
  __syncwarp();
  const int ne = np * 14;
  for (int idx = lane; idx < ne * ne; idx += 32) {
    const int a = idx / ne, bq = idx - a * ne;
    const int ia = (int)ws[a * 4], ib = (int)ws[bq * 4];
    if (ia < 0 || ib < 0 || ia < ib) continue;
    const double v = ws[a * 4 + 1] * ws[bq * 4 + 1] + ws[a * 4 + 2] * ws[bq * 4 + 2] + ws[a * 4 + 3] * ws[bq * 4 + 3];
    if (v != 0.0) chd_kadd(K, ia, ib, wgt * v);
  }
  __syncwarp();
}

// Cost part of the KKT matrix of sequence b: Gauss-Newton Hessian of the cost terms of data_cost.cpp /
// vel_smooth_cost.cpp / duration_cost.cpp at the current x, scaled by the objective scaling, added into `base` (zeroed
// before).  Constant during a fixed-duration stage (the costs are quadratic in the node values: Kbase, built when the
// stage begins); in stage 3 the basis weights move with the durations and it is rebuilt into Kwork every iteration.
// The samples are dealt to `nparts` CTAs (the reductions into L2 are the cost).
__device__ void chd_hess_build(const ChdDev& D, int b, const ChdStageDev& sg, double* base, int part, int nparts) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const ChdSeq* h = D.seq + b;
  ChdKT K;
  chd_kt_init(D, h, base, K);
  K.ovf = &D.ipm[b].band_ovf;
  const double sf = D.ipm[b].sf;
  const int* vk = D.var_kkt + (size_t)b * D.n_max;
  ChdCtx c;
  chd_make_ctx(D, b, D.x + (size_t)b * D.n_max, c);
  c.dyn = D.ipm[b].dyn;
  c.opt_dur = sg.opt_dur;
  const int n_ee = h->n_ee, nsp = 2 + n_ee, F = h->F, ns = h->n_smooth;
  // one warp per cost sample (the 28 x 28 pair loop of a sample is spread over its lanes)
  __shared__ double s_hws[CHD_THREADS / 32][28 * 4];
  const int lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
  for (int it = part * nwarp + warp; it < nsp * F; it += nparts * nwarp) {
    const int s = it / F, i = it % F, cls = s < 2 ? s : 2;
    ChdSpl P[2];
    double sgn[2] = {1.0, -1.0};
    chd_spl_at(c, s, c.t_data[i], P[1]);
    if (sg.w_data[cls] != 0.0) chd_hess_sample(c, K, vk, s, P + 1, sgn, 1, 0, sf * sg.w_data[cls], lane, s_hws[warp]);
    if (i < ns && (sg.w_vel[cls] != 0.0 || sg.w_acc[cls] != 0.0)) {
      chd_spl_at(c, s, c.t_data[i] + h->dt, P[0]);
      if (sg.w_vel[cls] != 0.0) chd_hess_sample(c, K, vk, s, P, sgn, 2, 0, sf * sg.w_vel[cls], lane, s_hws[warp]);
      if (sg.w_acc[cls] != 0.0) chd_hess_sample(c, K, vk, s, P, sgn, 2, 1, sf * sg.w_acc[cls], lane, s_hws[warp]);
    }
  }
  if (part == 0)
    for (int i = K.Na + tid; i < K.Np; i += nt) *chd_kdiag(K, i, true) = 1.0;  // identity padding of the band
  if (part == 0 && !sg.opt_dur && h->dur_band)   // banded switch times outside stage 3: decoupled unknowns, unit diagonal
    for (int i = tid; i < h->n_dur; i += nt) *chd_kdiag(K, vk[h->dur_xoff[0] + i], true) = 1.0;   // the duration variables of all feet are contiguous in x
  if (part == 0 && sg.opt_dur && sg.w_dur != 0.0) {   // duration_cost.cpp: w I in the durations = w D^T D in the switch times
    for (int ee = 0; ee < n_ee; ++ee)
      for (int k = tid; k < h->n_phases[ee] - 1; k += nt) {
        const int i = vk[h->dur_xoff[ee] + k];
        chd_kadd(K, i, i, sf * sg.w_dur);
        if (k > 0) {
          const int j = vk[h->dur_xoff[ee] + k - 1];
          chd_kadd(K, j, j, sf * sg.w_dur);
          chd_kadd(K, i, j, -sf * sg.w_dur);
        }
      }
  }
}
// zero fill of one tile-format matrix, slice `part` of `nparts` (the identity padding of the band is written by
// chd_hess_build, i.e. by a later kernel: the padding entries lie in some other CTA's slice)
__device__ void chd_hess_clear(const ChdDev& D, int b, double* base, int part, int nparts) {
  const size_t cnt2 = D.kstride / 2, per = (cnt2 + nparts - 1) / nparts;
  const size_t lo = (size_t)part * per, hi = lo + per < cnt2 ? lo + per : cnt2;
  double2* dst = reinterpret_cast<double2*>(base);
  for (size_t i = lo + threadIdx.x; i < hi; i += blockDim.x) dst[i] = make_double2(0.0, 0.0);
}
// zero fill of the right-hand-side accumulators of chd_k_asm of sequence b, by one CTA
__device__ void chd_rhs_clear(const ChdDev& D, int b) {
  const size_t go = (size_t)b * (D.Na_max + D.nb_max);
  for (int i = threadIdx.x; i < D.Na_max + D.nb_max; i += blockDim.x) D.rhs0[go + i] = 0.0, D.rhs1[go + i] = 0.0;
}

// stage 3, every iteration after the line search (side stream, grid (G, B)): the cost Hessian at the accepted iterate
// goes straight into Kwork, which chd_k_kcopy has zeroed for the sequences of that stage
__global__ void __launch_bounds__(CHD_THREADS) chd_k_hess_dur(ChdDev D) {
  const int b = blockIdx.y;
  const ChdIpm& I = D.ipm[b];
  if (I.phase != CHD_PH_RUN || !I.kw_req) return;
  const ChdStageDev sg = chd_stage(D, b, I.stage);
  if (!sg.opt_dur) return;
  chd_hess_build(D, b, sg, D.Kwork + (size_t)b * D.kstride, blockIdx.x, gridDim.x);
}
// after the cost Hessian is complete: foot-motion node values that no cost sample sees (zero diagonal) are flagged for
// chd_assemble's fixed regularisation.  mode 0 (main stream): sequences at the beginning of a stage (Kbase), which then
// start running; mode 1 (side stream): sequences iterating in stage 3 (Kwork, before the curvature terms are added)
__global__ void __launch_bounds__(128) chd_k_hess_fin(ChdDev D, int mode) {
  const int b = blockIdx.x;
  ChdIpm& I = D.ipm[b];
  double* base;
  if (mode == 0) {
    if (I.phase != CHD_PH_BEGIN) return;
    base = D.Kbase + (size_t)b * D.kstride;
  } else {
    if (I.phase != CHD_PH_RUN || !I.kw_req || !chd_stage(D, b, I.stage).opt_dur) return;
    base = D.Kwork + (size_t)b * D.kstride;
  }
  const ChdSeq* h = D.seq + b;
  const int* vk = D.var_kkt + (size_t)b * D.n_max;
  ChdKT K;
  chd_kt_init(D, h, base, K);
  unsigned char* un = D.unobs + (size_t)b * D.n_max;
  const int mot_lo = h->sp_xoff[2], mot_hi = h->sp_xoff[2 + h->n_ee];
  for (int i = mot_lo + threadIdx.x; i < mot_hi; i += blockDim.x) {
    const int k = vk[i];
    un[i] = k >= 0 && *chd_kdiag(K, k) <= CHD_UNOBS_EPS;
  }
  __syncthreads();
  if (mode == 0 && threadIdx.x == 0) I.phase = CHD_PH_RUN;
}

// y^+ * Jd^T Jd of the squared-distance rows (leg length, toe-heel distance) of sequence b added into K: one warp
// per active row, rows dealt round-robin to `nw` warps of which this is number `wid`.  ws: 192 doubles of per-warp
// scratch, slot -> (kkt index, weight, 3-vector column of Jd).  Called from chd_k_hess_base (first iteration of a
// stage) and from chd_k_curv (all later iterations, side stream).
__device__ __forceinline__ void chd_curv_rows(const ChdDev& D, int b, const ChdKT& K, const ChdStageDev& sg, int wid, int nw, int lane,
                                              double* ws) {
  const ChdSeq* h = D.seq + b;
  const size_t ro = (size_t)b * D.m_max, vo = (size_t)b * D.n_max;
  const int* vk = D.var_kkt + vo;
  ChdCtx c;
  chd_make_ctx(D, b, D.x + vo, c);
  c.dyn = D.ipm[b].dyn;
  c.opt_dur = sg.opt_dur;
  for (int si = 0; si < h->nsets; ++si) {
    const ChdSet st = c.sets[si];
    if (!(sg.set_mask & CHD_MASK(st.type))) continue;
    if (st.type != CHD_SET_ROM && st.type != CHD_SET_HEEL) continue;
    const int nslot = st.type == CHD_SET_ROM ? 38 : 28;   // node slots + the switch-time slots (stage 3)
    for (int k = wid; k < st.nitems; k += nw) {
      const int R = st.row0 + k;
      const double yc = D.sc[ro + R] * D.y[ro + R];
      if (!(yc > CHD_CURV_MIN)) continue;
      const double t = c.t_rom[k];
      ChdSpl P0, P1, P2;
      double dRh[3][3];
      if (st.type == CHD_SET_ROM) {
        // d = p_ee - R(e) h - c : blocks lin (-B e_dim), ang (-B dR_dim h), ee (+B e_dim)
        chd_spl_at(c, 0, t, P0);
        chd_spl_at(c, 1, t, P1);
        chd_spl_at(c, chd_sp_motion(st.a), t, P2);
        double e[3];
        chd_spl_val(c, P1, 0, e);
        ChdTrig tr;
        chd_trig(e, tr);
        const double* hip = chd_hip(c, st.a, t);
        for (int j = 0; j < 3; ++j) {
          double Dj[9];
          chd_dR(tr, j, Dj);
          chd_mv(Dj, hip, dRh[j]);
        }
      } else {
        chd_spl_at(c, chd_sp_motion(st.a), t, P0);   // d = p_a - p_b
        chd_spl_at(c, chd_sp_motion(st.b), t, P1);
      }
      ChdTau ua, ub;
      ua.va = ua.vb = ub.va = ub.vb = -1;
      if (c.opt_dur) {
        if (st.type == CHD_SET_ROM) chd_spl_tau(c, chd_sp_motion(st.a), st.a, P2, ua);
        else chd_spl_tau(c, chd_sp_motion(st.a), st.a, P0, ua), chd_spl_tau(c, chd_sp_motion(st.b), st.b, P1, ub);
      }
      const int nnode = st.type == CHD_SET_ROM ? 36 : 24;
      for (int a = lane; a < nslot; a += 32) {
        if (a >= nnode) {   // switch-time columns: d(d)/d(tau) is the 3-vector da / db of the foot spline (second foot: minus)
          const int t4 = a - nnode;
          const ChdTau& u = t4 < 2 ? ua : ub;
          const int var = (t4 & 1) ? u.vb : u.va;
          const double* dv = (t4 & 1) ? u.db : u.da;
          const int ia = var >= 0 ? vk[var] : -1;
          ws[a * 5 + 0] = (double)ia;
          ws[a * 5 + 1] = ia >= 0 ? (t4 < 2 ? 1.0 : -1.0) : 0.0;
          ws[a * 5 + 2] = ia >= 0 ? dv[0] : 0.0, ws[a * 5 + 3] = ia >= 0 ? dv[1] : 0.0, ws[a * 5 + 4] = ia >= 0 ? dv[2] : 0.0;
          continue;
        }
        const int ba = a / 12, qa = a % 12, da = qa % 3;
        const ChdSpl& Pa = ba == 0 ? P0 : (ba == 1 ? P1 : P2);
        const int va = Pa.var[qa];
        const int ia = va >= 0 ? vk[va] : -1;
        double sgn, v3[3] = {da == 0 ? 1.0 : 0.0, da == 1 ? 1.0 : 0.0, da == 2 ? 1.0 : 0.0};
        if (st.type == CHD_SET_ROM) {
          sgn = ba == 2 ? 1.0 : -1.0;
          if (ba == 1) v3[0] = dRh[da][0], v3[1] = dRh[da][1], v3[2] = dRh[da][2];
        } else {
          sgn = ba == 0 ? 1.0 : -1.0;
        }
        ws[a * 5 + 0] = (double)ia;
        ws[a * 5 + 1] = ia >= 0 ? sgn * chd_slot_w(Pa, 0, qa) : 0.0;
        ws[a * 5 + 2] = v3[0], ws[a * 5 + 3] = v3[1], ws[a * 5 + 4] = v3[2];
      }
      __syncwarp();
      for (int idx = lane; idx < nslot * nslot; idx += 32) {
        const int a = idx / nslot, bq = idx - a * nslot;
        const double wa = ws[a * 5 + 1], wb = ws[bq * 5 + 1];
        if (wa == 0.0 || wb == 0.0) continue;
        const int ia = (int)ws[a * 5], ib = (int)ws[bq * 5];
        if (ia < ib) continue;
        const double dotv = ws[a * 5 + 2] * ws[bq * 5 + 2] + ws[a * 5 + 3] * ws[bq * 5 + 3] + ws[a * 5 + 4] * ws[bq * 5 + 4];
        if (dotv != 0.0) chd_kadd(K, ia, ib, yc * wa * wb * dotv);
      }
      __syncwarp();
    }
  }
}

// Stage begin, grid (G, B), sequences in CHD_PH_BEGIN: what chd_k_kcopy, chd_k_hess_dur and chd_k_curv prepare for
// every later iteration, so that chd_k_asm and chd_k_kkt see the first iteration of a stage like any other --
// Kbase, Kwork, rhs0, rhs1 <- 0 (chd_k_hess_zero); the distance-row curvature at the initial point (x, y, scaling
// are final after chd_k_init; y != 0 in a warm-started stage 3) into Kwork, then the cost Hessian into Kbase and
// Kwork (chd_k_hess_base; this order spills less); the flags and BEGIN -> RUN (chd_k_hess_fin, mode 0).
// kw_req stays 0 here: the side-stream kernels of the previous iteration may still be running, and they leave the
// Kwork / rhs0 / rhs1 of a sequence whose stage just ended alone only because chd_stage_advance cleared its kw_req
// before they were launched.
__global__ void __launch_bounds__(256) chd_k_hess_zero(ChdDev D) {
  const int b = blockIdx.y;
  if (D.ipm[b].phase != CHD_PH_BEGIN) return;
  chd_hess_clear(D, b, D.Kbase + (size_t)b * D.kstride, blockIdx.x, gridDim.x);
  chd_hess_clear(D, b, D.Kwork + (size_t)b * D.kstride, blockIdx.x, gridDim.x);
  if (blockIdx.x == 0) chd_rhs_clear(D, b);
}
// (256 threads, two CTAs per SM, grid (16, B): launched every iteration, its CTAs exit at once for the sequences that
// do not begin a stage, but each needs its registers free before it starts -- with 512 threads at 128 registers that
// is a whole SM, so they would wait for the side-stream kernels of the previous iteration to drain)
__global__ void __launch_bounds__(256, 2) chd_k_hess_base(ChdDev D) {
  __shared__ double s_ws[8][192];
  const int b = blockIdx.y;
  if (D.ipm[b].phase != CHD_PH_BEGIN) return;
  const ChdStageDev sg = chd_stage(D, b, D.ipm[b].stage);
  ChdKT K;
  chd_kt_init(D, D.seq + b, D.Kwork + (size_t)b * D.kstride, K);
  K.ovf = &D.ipm[b].band_ovf;
  const int warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  chd_curv_rows(D, b, K, sg, blockIdx.x * nwarp + warp, gridDim.x * nwarp, threadIdx.x & 31, s_ws[warp]);
  chd_hess_build(D, b, sg, D.Kbase + (size_t)b * D.kstride, blockIdx.x, gridDim.x);
  chd_hess_build(D, b, sg, D.Kwork + (size_t)b * D.kstride, blockIdx.x, gridDim.x);
}

// Jacobian-dependent part of the condensed KKT system of sequence b by threads t0, t0 + tstep, ...: matrix entries
// (global reductions into K) and the right-hand side split as rhs = g0 + mu * g1 -- every term is affine in the
// barrier parameter, which is only decided inside chd_k_kkt -- accumulated with global reductions.  Narrow inequality
// rows (<= 12 slots: terrain, friction pyramid, height) are condensed into the primal block (J^T Sigma J); wide ones
// (leg length) keep their multiplier as an unknown with diagonal -1/Sigma, which needs 36 instead of 666 matrix
// updates per row.
__device__ __forceinline__ void chd_assemble(const ChdDev& D, int b, const ChdKT& K, double delta_w, double sf, int t0, int tstep,
                                             double* g0, double* g1) {
  const ChdSeq* h = D.seq + b;
  const int n = chd_stage(D, b, D.ipm[b].stage).opt_dur ? h->n : h->n - h->n_dur;   // the durations are unknowns in stage 3 only
  const int m = h->m, Na = K.Na;
  const size_t ro = (size_t)b * D.m_max, vo = (size_t)b * D.n_max;
  const int* rf = D.rflag + ro;
  const int* vk = D.var_kkt + vo;
  const int* rk = D.row_kkt + ro;
  const int* ep = D.ent_ptr + (size_t)b * (D.m_max + 1);
  const int* ec = D.ent_col + (size_t)b * D.slots_max;
  const double* Jv = D.Jv + (size_t)b * D.slots_max;
  const double* grad = D.grad + vo;
  auto gidx = [&](int kk) { return kk < Na ? kk : D.Na_max + (kk - Na); };
  auto g_add = [&](int kk, double v0, double v1) {
    atomicAdd(g0 + gidx(kk), v0);
    if (v1 != 0.0) atomicAdd(g1 + gidx(kk), v1);
  };
  // foot-motion node values that no cost sample sees (polynomials shorter than a frame): without curvature of their own
  // the Newton step uses them as free slack and they drift by orders of magnitude, which stage 3 (where the sample
  // times sweep over those polynomials) cannot digest.  They get a fixed Levenberg-Marquardt weight on top of the
  // adaptive one -- what the initial scaling of IPOPT's L-BFGS matrix does for the reference.
  const unsigned char* unobs = D.unobs + vo;
  for (int i = t0; i < n; i += tstep) {
    const int k = vk[i];
    if (k < 0) continue;
    if (unobs[i]) chd_kadd(K, k, k, CHD_DW_UNOBS);
    chd_kadd(K, k, k, delta_w);
    g_add(k, -sf * grad[i], 0.0);
  }
  for (int r = t0; r < m; r += tstep) {
    const int f = rf[r];
    const int k = rk[r];
    if (!(f & CHD_ROW_ACTIVE)) {
      if (k >= 0) chd_kadd(K, k, k, -1.0);   // row of an inactive set: decoupled dummy unknown
      continue;
    }
    const double sc = D.sc[ro + r];
    const int e0 = ep[r], e1 = ep[r + 1];
    if (k >= 0) {
      // explicit row: equality, or wide inequality with its slack eliminated
      double diag = -CHD_DELTA_C, rr0 = -chd_row_res(f, sc * D.g[ro + r], D.dL[ro + r], D.s[ro + r]), rr1 = 0.0;
      if (!(f & CHD_ROW_EQ)) {
        const ChdGaps gap = chd_row_gaps(f, D.s[ro + r], D.dL[ro + r], D.dU[ro + r]);
        const double Sig = chd_row_sigma(f, gap, D.zL[ro + r], D.zU[ro + r]).sum();
        diag -= 1.0 / Sig;
        rr0 += D.y[ro + r] / Sig;
        rr1 = chd_row_mu_coef(f, gap) / Sig;
      }
      chd_kadd(K, k, k, diag);
      g_add(k, rr0, rr1);
      const double ys = sc * D.y[ro + r];
      for (int e = e0; e < e1; ++e) {
        const int col = ec[e];
        if (col < 0) continue;
        const int kc = vk[col];
        if (kc < 0) continue;
        const double jv = Jv[e];
        if (jv == 0.0) continue;
        chd_kadd(K, k, kc, sc * jv);
        g_add(kc, -ys * jv, 0.0);
      }
    } else {
      // condensed narrow inequality row
      const double s = D.s[ro + r];
      const ChdGaps gap = chd_row_gaps(f, s, D.dL[ro + r], D.dU[ro + r]);
      const double Sig = chd_row_sigma(f, gap, D.zL[ro + r], D.zU[ro + r]).sum();
      const double coef0 = Sig * chd_row_res(f, sc * D.g[ro + r], D.dL[ro + r], s);
      const double beta = chd_row_mu_coef(f, gap);
      for (int ea = e0; ea < e1; ++ea) {
        const int ca = ec[ea];
        if (ca < 0) continue;
        const int ka = vk[ca];
        if (ka < 0) continue;
        const double va = sc * Jv[ea];
        if (va == 0.0) continue;
        g_add(ka, -va * coef0, va * beta);
        for (int eb = e0; eb < e1; ++eb) {
          const int cb = ec[eb];
          if (cb < 0) continue;
          const int kb = vk[cb];
          if (kb < 0 || ka < kb) continue;
          const double vb = sc * Jv[eb];
          if (vb != 0.0) chd_kadd(K, ka, kb, Sig * va * vb);
        }
      }
    }
  }
}

// What every phase of chd_k_kkt sees of its sequence: the thread's place in the CTA, the sequence's arrays and KKT
// storage, the sizes of the current stage, the carve-up of the dynamic shared memory (doubles)
//   red[CHD_KKT_THREADS] | cc[nbp8*nbp8] | ypan[(Q+nbt)*64] | xpan[(Q+nbt)*64] ... (pan_doubles from ypan) | dinv[16]
//   | win[win_tiles * 64] | bwin[Q*nbt*64]            (the last two in global scratch when they do not fit)
// and the barrier parameter / step rules decided by the error measures.  (The solution vector D.sol is addressed by
// each phase that uses it: a pointer held across the factorisation costs spills.)
struct ChdKktCtx {
  int b, tid, nt, lane, warp, nwarp;
  ChdIpm* I;
  ChdStageDev sg;
  const ChdSeq* h;
  int n, m, n_act, Qs, Q, nbt, nbp8, nbl, nbc, NBR, nbt_s;
  size_t ro, vo, n_even, xs_len, win_region;
  const int *rf, *vk, *rk, *ep, *ec;
  const double *Jv, *grad;
  ChdKT K;
  double *red, *cc, *ypan, *xpan, *dinv, *win, *bwin, *vecn, *xs, *xs2;
  double sf, mu, tau, delta_w;
  bool polish;
};

template <bool WS>
__device__ __forceinline__ void chd_kkt_ctx_init(const ChdDev& D, ChdIpm& I, ChdKktCtx& c) {
  extern __shared__ double sm[];
  const int b = blockIdx.x;
  c.b = b, c.I = &I;
  c.sg = chd_stage(D, b, I.stage);
  const ChdSeq* h = c.h = D.seq + b;
  c.n = h->n, c.m = h->m, c.tid = threadIdx.x, c.nt = blockDim.x;
  c.lane = c.tid & 31, c.warp = c.tid >> 5, c.nwarp = c.nt >> 5;
  c.ro = (size_t)b * D.m_max, c.vo = (size_t)b * D.n_max;
  c.rf = D.rflag + c.ro;
  c.vk = D.var_kkt + c.vo;
  c.rk = D.row_kkt + c.ro;
  c.ep = D.ent_ptr + (size_t)b * (D.m_max + 1);
  c.ec = D.ent_col + (size_t)b * D.slots_max;
  c.Jv = D.Jv + (size_t)b * D.slots_max;
  c.grad = D.grad + c.vo;
  ChdKT& K = c.K;
  chd_kt_init(D, h, D.Kwork + (size_t)b * D.kstride, K);
  K.ovf = &I.band_ovf;
  if (!c.sg.opt_dur) K.q = D.Qfix - 1;   // fixed-duration stages: the static pattern needs fewer band tiles than stage 3 may
  // (Q is the number of block rows of the elimination window of this stage, Qs the storage stride of a block column)
  c.n_act = c.sg.opt_dur ? c.n : c.n - h->n_dur;          // the durations (last n_dur entries of x) are unknowns in stage 3 only
  c.Qs = K.Q, c.Q = c.sg.opt_dur ? K.Q : D.Qfix, c.nbt = K.nbt, c.nbp8 = K.nbp8, c.nbl = c.sg.opt_dur ? h->nb : h->nb_fix, c.nbc = K.nbc;
  // the right-hand side rides along as border row NBR, directly behind the border unknowns of this stage; nbt_s = border
  // tiles in use (the switch-time columns of stage 3 are all zero in the fixed-duration stages: not even looked at)
  c.NBR = c.nbl, c.nbt_s = (c.nbl + 1 + 7) >> 3;
  // WS: everything in shared memory.  !WS (long horizons / very wide bands): only the reduction buffer, the
  // corner and the panel buffers stay in shared memory; the per-unknown vectors and the window live in a global
  // (L2 resident) scratch area  vecn | xs | xs2 | win | bwin.
  c.n_even = (size_t)((D.n_max + 1) & ~1), c.xs_len = (size_t)(8 * D.nbc_max + c.nbp8);
  double* gs = WS ? nullptr : D.scratch + (size_t)b * D.scratch_stride;
  c.red = sm;
  c.cc = c.red + CHD_KKT_THREADS;
  c.ypan = c.cc + c.nbp8 * c.nbp8;
  c.xpan = c.ypan + (c.Q + c.nbt) * 64;
  c.dinv = c.ypan + D.pan_doubles;
  // WS: the per-unknown vectors vecn (step recovery) and xs (solution after the factorisation) alias the tail of the
  // window region, which is dead whenever they are live (the back-substitution stages its tiles in the front part only)
  c.win_region = (size_t)D.win_tiles * 64 + (size_t)c.Qs * c.nbt * 64;
  c.win = WS ? c.dinv + 16 : gs + c.n_even + c.xs_len + 8 * (size_t)D.nbc_max;
  c.bwin = c.win + (size_t)D.win_tiles * 64;
  c.vecn = WS ? c.win + c.win_region - c.n_even : gs;
  c.xs = WS ? c.vecn - c.xs_len : c.vecn + c.n_even;
  c.xs2 = WS ? c.ypan : c.xs + c.xs_len;      // back-substitution accumulator (WS: aliases the then idle panel buffers)
  c.sf = I.sf;
}

// A. error measures, convergence test, barrier update.  Returns true when the sequence has finished its stage (it has
// moved on in the schedule); otherwise decides mu, tau and delta_w of this iteration.
__device__ __forceinline__ bool chd_kkt_errors(const ChdDev& D, ChdKktCtx& c, int& s_fail) {
  ChdIpm& I = *c.I;
  const int b = c.b, tid = c.tid, nt = c.nt, n = c.n, m = c.m, n_act = c.n_act;
  const size_t ro = c.ro, vo = c.vo;
  const int *rf = c.rf, *vk = c.vk, *ep = c.ep, *ec = c.ec;
  const double *Jv = c.Jv, *grad = c.grad, sf = c.sf;
  double* red = c.red;
  double mu = I.mu;
  // J^T y is gathered per variable from a column-oriented index of the Jacobian slots (no shared-memory fp64
  // atomics, which are compare-and-swap loops): per-row multipliers first, into the (idle) dy array
  const int* erow = D.ent_row + (size_t)b * D.slots_max;
  const int* cptr = D.col_ptr + (size_t)b * (D.n_max + 1);
  const int* cent = D.col_ent + (size_t)b * D.slots_max;
  double* rowv = D.dy + ro;
  double a_ysum = 0, a_zsum = 0, a_cviol = 0, a_theta = 0, a_rs = 0, a_cmax = -INFINITY, a_cmin = INFINITY, a_violu = 0;
  for (int r = tid; r < m; r += nt) {
    const int f = rf[r];
    if (!(f & CHD_ROW_ACTIVE)) {
      rowv[r] = 0.0;
      continue;
    }
    const double sc = D.sc[ro + r], gval = D.g[ro + r], d = sc * gval, y = D.y[ro + r];
    a_ysum += fabs(y);
    a_violu = fmax(a_violu, fmax(D.row_lo[ro + r] - gval, gval - D.row_hi[ro + r]));
    rowv[r] = sc * y;
    const double rp = chd_row_res(f, d, D.dL[ro + r], D.s[ro + r]);
    a_cviol = fmax(a_cviol, fabs(rp));
    a_theta += fabs(rp);
    if (!(f & CHD_ROW_EQ)) {
      const double zL = D.zL[ro + r], zU = D.zU[ro + r];
      const ChdGaps gap = chd_row_gaps(f, D.s[ro + r], D.dL[ro + r], D.dU[ro + r]);
      a_rs = fmax(a_rs, fabs(-y - zL + zU));
      a_zsum += zL + zU;
      if (f & CHD_ROW_HASL) { const double cp = gap.L * zL; a_cmax = fmax(a_cmax, cp); a_cmin = fmin(a_cmin, cp); }
      if (f & CHD_ROW_HASU) { const double cp = gap.U * zU; a_cmax = fmax(a_cmax, cp); a_cmin = fmin(a_cmin, cp); }
    }
  }
  __syncthreads();
  double a_dual = 0;
  if (!I.dyn) {
    for (int i = tid; i < n_act; i += nt) {
      double v = sf * grad[i];
      for (int t = cptr[i]; t < cptr[i + 1]; ++t) {
        const int e = cent[t];
        v += rowv[erow[e]] * Jv[e];
      }
      if (vk[i] >= 0) a_dual = fmax(a_dual, fabs(v));
    }
  } else {
    // run-time Jacobian columns (stage 3 onwards): the column index of the layout is stale, J^T y goes through
    // reductions into a per-sequence global vector
    double* jty = D.jty + vo;
    for (int i = tid; i < n; i += nt) jty[i] = 0.0;
    __syncthreads();
    for (int r = tid; r < m; r += nt) {
      const double ys = rowv[r];
      if (ys == 0.0) continue;
      for (int e = ep[r]; e < ep[r + 1]; ++e) {
        const int col = ec[e];
        if (col >= 0 && Jv[e] != 0.0) atomicAdd(jty + col, ys * Jv[e]);
      }
    }
    __syncthreads();
    for (int i = tid; i < n_act; i += nt)
      if (vk[i] >= 0) a_dual = fmax(a_dual, fabs(sf * grad[i] + jty[i]));
  }
  const double ysum = chd_block_sum(a_ysum, red), zsum = chd_block_sum(a_zsum, red);
  const double cviol = chd_block_max(a_cviol, red), theta = chd_block_sum(a_theta, red);
  const double dual_inf = fmax(chd_block_max(a_dual, red), chd_block_max(a_rs, red));
  const double cmax = chd_block_max(a_cmax, red), cmin = chd_block_min(a_cmin, red);
  const double violu = fmax(chd_block_max(a_violu, red), 0.0);
  const int nbnd = I.n_bounds;
  const double s_d = fmax(CHD_S_MAX, (ysum + zsum) / fmax((double)(I.m_act + nbnd), 1.0)) / CHD_S_MAX;
  const double s_c = fmax(CHD_S_MAX, zsum / fmax((double)nbnd, 1.0)) / CHD_S_MAX;
  auto compl_err = [&](double mm) { return nbnd > 0 ? fmax(fabs(cmax - mm), fabs(cmin - mm)) : 0.0; };
  const double E0 = fmax(fmax(dual_inf / s_d, cviol), compl_err(0.0) / s_c);
  const double dual_u = dual_inf / sf, compl_u = compl_err(0.0) / sf;
  bool done = false;
  int new_status = 1;
  if (E0 <= CHD_TOL && violu <= CHD_CONSTR_VIOL_TOL && dual_u <= CHD_DUAL_INF_TOL && compl_u <= CHD_COMPL_INF_TOL) new_status = 0, done = true;
  else if (I.iter >= I.max_iter) new_status = -1, done = true;
  if (!done) {
    const double mu_min = fmin(CHD_TOL, CHD_COMPL_INF_TOL) / (CHD_KAPPA_EPS + 1.0);
    while (true) {
      const double Emu = fmax(fmax(dual_inf / s_d, cviol), compl_err(mu) / s_c);
      if (Emu <= CHD_KAPPA_EPS * mu && mu > mu_min) mu = fmax(mu_min, fmin(CHD_KAPPA_MU * mu, pow(mu, CHD_THETA_MU)));
      else break;
    }
  }
  __syncthreads();
  if (tid == 0) {
    I.f = D.cost[2 * b];
    I.E0 = E0, I.viol_u = violu, I.dual_u = dual_u, I.compl_u = compl_u;
    I.status = new_status;
    s_fail = 0;
    if (done) chd_stage_advance(D, I, new_status, c.sg.snap_after);
    if (!done) {
      I.mu = mu;
      I.tau = fmax(CHD_TAU_MIN, 1.0 - mu);
      if (I.iter == 0) I.theta_max = 1e4 * fmax(1.0, theta), I.theta_min = 1e-4 * fmax(1.0, theta), I.theta_ref = theta;
      if (mu != I.mu_filter) I.nfilt = 0, I.mu_filter = mu;
      I.theta0 = theta;
    }
  }
  if (done) return true;
  c.mu = mu;
  c.tau = fmax(CHD_TAU_MIN, 1.0 - mu);
  // feasibility polish: every test but the unscaled constraint violation passes -> this step only restores feasibility
  // (a large Levenberg-Marquardt weight makes it the least-norm Newton correction of the constraints; the adaptive
  // weight itself is left alone)
  c.polish = E0 <= CHD_TOL && dual_u <= CHD_DUAL_INF_TOL && compl_u <= CHD_COMPL_INF_TOL && violu > CHD_CONSTR_VIOL_TOL &&
             I.delta_w < CHD_DW_POLISH;
  c.delta_w = c.polish ? CHD_DW_POLISH : I.delta_w;
  return false;
}

// B. what this iteration's barrier parameter and step rule decide of the KKT system, which chd_k_asm has assembled
// otherwise: a feasibility-polish step tops up the adaptive weight chd_k_asm put on the diagonal, and the right-hand
// side rhs0 + mu * rhs1 goes into border row NBR (band unknowns) and corner row NBR (border unknowns).
__device__ __forceinline__ void chd_kkt_assemble(const ChdDev& D, const ChdKktCtx& c) {
  const ChdIpm& I = *c.I;
  const ChdKT& K = c.K;
  const int tid = c.tid, nt = c.nt, n_act = c.n_act, nbl = c.nbl, nbt = c.nbt, nbp8 = c.nbp8, NBR = c.NBR, Na = K.Na;
  const int* vk = c.vk;
  const double mu = c.mu;
  if (c.polish) {
    const double extra = c.delta_w - I.delta_w;
    for (int i = tid; i < n_act; i += nt)
      if (vk[i] >= 0) chd_kadd(K, vk[i], vk[i], extra);
  }
  const double* r0 = D.rhs0 + (size_t)c.b * (D.Na_max + D.nb_max);
  const double* r1 = D.rhs1 + (size_t)c.b * (D.Na_max + D.nb_max);
  for (int i = tid; i < K.Np; i += nt)
    K.bord[((size_t)(i >> 3) * nbt + (NBR >> 3)) * 64 + (NBR & 7) * 8 + (i & 7)] = i < Na ? r0[i] + mu * r1[i] : 0.0;
  for (int i = tid; i < nbl; i += nt) K.corn[(size_t)NBR * nbp8 + i] = r0[D.Na_max + i] + mu * r1[D.Na_max + i];
}

// One 2 x 2 block of the trailing update C -= X Y^T: panel rows gi[0], gi[1] (X) against panel columns gj[0], gj[1] (Y)
// of the panel buffers, vi / vj = which of them take part.  The operand fragments of the block are loaded once and every
// target tile's C is loaded before the first product; one m16n8k8 per panel column (the two row tiles stacked).
// Targets that are not updated here (the upper tile of a diagonal block, a row or column that takes no part, warp 0's
// next diagonal tile) are computed from a zero C and not stored.
template <class BandTile, class BordTile>
__device__ __forceinline__ void chd_kkt_update_block(const ChdKktCtx& c, const int* gi, const int* gj, const bool* vi, const bool* vj, bool diag,
                                                     int GB, const BandTile& band_tile, const BordTile& bord_tile) {
  const int lane = c.lane;
  const double2 z = make_double2(0.0, 0.0);
  double2 xf[2], yf[2];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    xf[a] = vi[a] ? *reinterpret_cast<const double2*>(c.xpan + gi[a] * 64 + 2 * lane) : z;
    yf[a] = vj[a] ? *reinterpret_cast<const double2*>(c.ypan + gj[a] * 64 + 2 * lane) : z;
  }
  double* Cp[4];
  double2 cv[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int a = t & 1, cl = t >> 1;          // tile (row a, column cl) of the block
    bool ok = vi[a] && vj[cl] && !(diag && a == 0 && cl == 1);
    // the next diagonal tile is updated by warp 0.  With a single band tile per block column (GB = 0) group 0 is the
    // first border tile, whose corner block is updated here like every other
    ok = ok && !(GB > 0 && gi[a] == 0 && gj[cl] == 0);
    // this lane's (row g, columns 2t, 2t+1) of the target: band tile, border tile or corner block (row stride nbp8)
    Cp[t] = nullptr;
    if (ok) {
      if (gi[a] < GB) Cp[t] = band_tile(gi[a], gj[cl]) + (lane >> 2) * 8 + 2 * (lane & 3);
      else if (gj[cl] < GB) Cp[t] = bord_tile(gi[a] - GB, gj[cl]) + (lane >> 2) * 8 + 2 * (lane & 3);
      else Cp[t] = c.cc + (size_t)((gi[a] - GB) * 8 + (lane >> 2)) * c.nbp8 + (gj[cl] - GB) * 8 + 2 * (lane & 3);
    }
    cv[t] = ok ? *reinterpret_cast<const double2*>(Cp[t]) : z;
  }
  const double2 xt = make_double2(-xf[0].x, -xf[0].y), xb = make_double2(-xf[1].x, -xf[1].y);
#pragma unroll
  for (int cl = 0; cl < 2; ++cl) chd_mma_16x8x8(cv[2 * cl], cv[2 * cl + 1], xt, xb, yf[cl]);
#pragma unroll
  for (int t = 0; t < 4; ++t)
    if (Cp[t]) *reinterpret_cast<double2*>(Cp[t]) = cv[t];
}

// Trailing updates of one block column by the warps 1 .. nwarp-1, for at most 64 panel groups (every shared-memory
// window; global windows of narrower bands).  2 x 2 register blocking over the compacted list of the groups with a
// non-zero X tile: one trip loads the operand fragments of two panel rows (X) and two panel columns (Y) once and
// updates up to four target tiles with them -- the loop is shared-memory bandwidth bound, this cuts the bytes per tile
// update from 2 KB to 1.5 KB and the index work 4x.  cmp: this warp's rank -> group table.
template <class BandTile, class BordTile>
__device__ __forceinline__ void chd_kkt_update_compact(const ChdKktCtx& c, const unsigned short* s_pairs, unsigned char* cmp, const int* gnz,
                                                       int GB, int Gm, int tq, const BandTile& band_tile, const BordTile& bord_tile) {
  const int lane = c.lane, warp = c.warp;
  // compact list of the groups with a non-zero X tile (every warp builds it redundantly: no extra barrier).
  // the pair table enumerates (i >= j) row by row, so its first na(na+1)/2 entries pair the first na entries.
  int na;
  {
    // up to 64 groups, two per lane; scatter by rank through a per-warp table (__fns is slow)
    const int g1 = lane + 32;
    const bool act0 = lane < Gm && (lane >= GB || lane < tq) && gnz[lane];
    const bool act1 = g1 < Gm && (g1 >= GB || g1 < tq) && gnz[g1 < 96 ? g1 : 0];
    const unsigned m0 = __ballot_sync(0xffffffffu, act0), m1 = __ballot_sync(0xffffffffu, act1);
    const unsigned below = (1u << lane) - 1u;
    const int n0 = __popc(m0);
    na = n0 + __popc(m1);
    if (act0) cmp[__popc(m0 & below)] = (unsigned char)lane;
    if (act1) cmp[n0 + __popc(m1 & below)] = (unsigned char)g1;
    __syncwarp();
  }
  const int step = c.nwarp - 1;
  const int nb2 = (na + 1) >> 1, nblk = nb2 * (nb2 + 1) / 2;
  for (int p = warp - 1; p < nblk; p += step) {
    const int bi = s_pairs[p] >> 8, bj = s_pairs[p] & 255;
    const int i1 = 2 * bi + 1, j1 = 2 * bj + 1;
    const int gi[2] = {cmp[2 * bi], cmp[i1 & 63]}, gj[2] = {cmp[2 * bj], cmp[j1 & 63]};
    const bool vi[2] = {true, i1 < na}, vj[2] = {true, j1 < na};
    chd_kkt_update_block(c, gi, gj, vi, vj, bi == bj, GB, band_tile, bord_tile);
  }
}

// Trailing updates of one block column by the warps 1 .. nwarp-1 with more than 64 panel groups (window in global (L2)
// memory): the same 2 x 2 blocks over the groups themselves (the per-warp compacted list holds 64 groups); blocks
// without a live target are skipped.
template <class BandTile, class BordTile>
__device__ __forceinline__ void chd_kkt_update_wide(const ChdKktCtx& c, const unsigned short* s_pairs, const int* gnz, int GB, int Gm,
                                                    int tq, const BandTile& band_tile, const BordTile& bord_tile) {
  auto live = [&](int g) { return g < Gm && (g >= GB || g < tq) && gnz[g]; };
  const int nb2 = (Gm + 1) >> 1, nblk = nb2 * (nb2 + 1) / 2;
  for (int p = c.warp - 1; p < nblk; p += c.nwarp - 1) {
    const int bi = s_pairs[p] >> 8, bj = s_pairs[p] & 255;
    const int gi[2] = {2 * bi, 2 * bi + 1}, gj[2] = {2 * bj, 2 * bj + 1};
    const bool vi[2] = {live(gi[0]), live(gi[1])}, vj[2] = {live(gj[0]), live(gj[1])};
    if (!(vi[0] || vi[1]) || !(vj[0] || vj[1])) continue;
    chd_kkt_update_block(c, gi, gj, vi, vj, bi == bj, GB, band_tile, bord_tile);
  }
}

// C. tiled band LDL^T with dense border, block column by block column: panel, stream-in of the next block row, trailing
// updates.  Sets s_fail on a bad pivot of a diagonal tile.
template <bool WS>
__device__ __forceinline__ void chd_kkt_factor(const ChdKktCtx& c, int& s_fail) {
  const ChdKT& K = c.K;
  const int tid = c.tid, nt = c.nt, lane = c.lane, warp = c.warp, nwarp = c.nwarp;
  const int Qs = c.Qs, Q = c.Q, nbt = c.nbt, nbp8 = c.nbp8, nbc = c.nbc, nbt_s = c.nbt_s;
  double *cc = c.cc, *ypan = c.ypan, *xpan = c.xpan, *dinv = c.dinv, *win = c.win, *bwin = c.bwin;
  // corner (incl. rhs row) to shared memory; initial window: band tiles (I, J), 0 <= J <= I <= q and border columns 0..q
  for (int i = tid; i < nbp8 * nbp8; i += nt) cc[i] = K.corn[i];
  // (without the shared-memory window the factorisation runs in place on Kwork: no window copy, no stream-in)
  if (WS) {
    for (int idx = tid; idx < Q * Q * 64; idx += nt) {
      const int e = idx & 63, pr = idx >> 6, J = pr / Q, t = pr % Q;
      if (J + t < Q && J < nbc && J + t < nbc) win[chd_win_slot(J + t, J, Q) * 64 + e] = K.band[((size_t)J * Qs + t) * 64 + e];
    }
    for (int idx = tid; idx < Q * nbt * 64; idx += nt) {
      const int J = idx / (nbt * 64);
      if (J < nbc) bwin[idx] = K.bord[(size_t)J * nbt * 64 + idx % (nbt * 64)];
    }
  }
  __syncthreads();
  // index tables: pair list of the 2 x 2 blocks of the trailing update (built once; panel groups = band groups 0..q-1,
  // border groups q..q+nbt-1), window slot of every band group of the current block column (double buffered, no
  // integer division)
  __shared__ int s_rs[2][96];
  __shared__ int s_gnz[2][96];   // per panel group: any non-zero entry in the X tile (zero tiles skip their trailing updates)
  // pair table: at most 64 panel groups with the shared-memory window, 96 with the global one (its static shared memory
  // is not needed for a window).  The 2 x 2 blocks use the first (Gm+1)/2 * ((Gm+1)/2 + 1) / 2 entries; the sizes are
  // the static shared memory the KKT plan budgets for each kernel.
  constexpr int kPairs = WS ? 3000 : CHD_KKT_GROUPS_MAX * (CHD_KKT_GROUPS_MAX + 1) / 2;
  __shared__ unsigned short s_pairs[kPairs];
  __shared__ unsigned char s_cmp[CHD_KKT_THREADS / 32][64];   // per warp: rank -> id of the non-zero panel groups
  __shared__ __align__(16) double s_winv[2][64];   // inverse of the current / next diagonal tile factor, fragment order
#ifdef CHD_PROFILE
  // phase (c) of every block column: warp 0's update and LDL^T of the next diagonal tile (prof[6]), and the time until the
  // last update warp is done (prof[7]) -- the larger of the two bounds the block column
  __shared__ unsigned long long s_upd_end;
  double prof_diag = 0.0, prof_upd = 0.0;
  if (tid == 0) s_upd_end = 0;
#endif
  // block pairs (bi >= bj) of the 2 x 2 blocks of the trailing update, row by row
  const int GB = K.q, Gm = K.q + nbt_s, nb2 = (Gm + 1) >> 1, npairs = nb2 * (nb2 + 1) / 2;
  for (int p = tid; p < npairs && p < kPairs; p += nt) {
    int gi = (int)((sqrt(8.0 * p + 1.0) - 1.0) * 0.5);
    while (gi * (gi + 1) / 2 > p) --gi;
    while ((gi + 1) * (gi + 2) / 2 <= p) ++gi;
    s_pairs[p] = (unsigned short)((gi << 8) | (p - gi * (gi + 1) / 2));
  }
  auto tri = [](int a_, int b_) { return a_ > b_ ? a_ * (a_ + 1) / 2 + b_ : b_ * (b_ + 1) / 2 + a_; };
  for (int g = tid; g < GB; g += nt) s_rs[0][g] = (1 + g) % Q;
  for (int g = tid; g < 96; g += nt) s_gnz[0][g] = 0, s_gnz[1][g] = 0;
  if (warp == 0) {
    const bool ok = chd_tile_ldl(WS ? win : K.band, dinv, s_winv[0], lane);   // tile (0,0) sits in slot 0
    if (!ok && lane == 0) s_fail = 1;
  }
  __syncthreads();
  int kslot = 0, cur = 0;  // kslot = Kc % Q
  for (int Kc = 0; Kc < nbc; ++Kc, cur ^= 1) {
    const int tq = min(K.q, nbc - 1 - Kc);          // band tiles below the diagonal tile
    const int* rs = s_rs[cur];
    // tile addresses: circular triangular window in shared memory, or in place in the global band / border storage
    auto band_tile = [&](int gi, int gj) -> double* {     // tile (Kc+1+gi, Kc+1+gj), gi >= gj
      return WS ? win + (size_t)tri(rs[gi], rs[gj]) * 64 : K.band + ((size_t)(Kc + 1 + gj) * Qs + (gi - gj)) * 64;
    };
    auto bord_tile = [&](int bi, int gj) -> double* {     // border tile bi of block column Kc+1+gj
      return WS ? bwin + ((size_t)rs[gj] * nbt + bi) * 64 : K.bord + ((size_t)(Kc + 1 + gj) * nbt + bi) * 64;
    };
    double* Tkk = WS ? win + (size_t)tri(kslot, kslot) * 64 : K.band + (size_t)Kc * Qs * 64;
    double* Bk = WS ? bwin + (size_t)kslot * nbt * 64 : K.bord + (size_t)Kc * nbt * 64;
    const double* dv = dinv + 8 * cur;
    // with a single band tile per block column (half bandwidth 0) no trailing update reaches the next diagonal tile, so
    // warp 0 does not factor it in (c): it is factored here, once the previous block column has streamed it in
    if (GB == 0 && Kc > 0) {
      if (warp == 0) {
        const bool ok = chd_tile_ldl(Tkk, dinv + 8 * cur, s_winv[cur], lane);
        if (!ok && lane == 0) s_fail = 1;
      }
      __syncthreads();
    }
    // (b) panel: Y = A L0^-T = A W^T (W = L0^-1 from the diagonal-tile factorisation) as one tensor-core product per
    //     pair of 8x8 panel tiles (stacked rows of an m16n8k8), X = Y D^-1; both go to the panel buffers in fragment
    //     order, X also to global (final L); the diagonal tile goes to global as well
    {
      const double* wv = s_winv[cur];
      const int r = lane >> 2, k = lane & 3, ng = tq + nbt_s;
      const double2 wf = *reinterpret_cast<const double2*>(wv + 2 * lane);
      const double d0 = dv[2 * k], d1 = dv[2 * k + 1];
      const int f0 = r * 8 + chd_frag_col(2 * k), f1 = r * 8 + chd_frag_col(2 * k + 1);
      for (int g0 = 2 * warp; g0 < ng; g0 += 2 * nwarp) {
        double2 a[2], y[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int g = g0 + h;
          const double* A = g < tq ? (WS ? win + (size_t)tri(rs[g], kslot) * 64 : K.band + ((size_t)Kc * Qs + 1 + g) * 64) : Bk + (g - tq) * 64;
          a[h] = g < ng ? make_double2(A[r * 8 + k], A[r * 8 + k + 4]) : make_double2(0.0, 0.0);
          y[h] = make_double2(0.0, 0.0);
        }
        chd_mma_16x8x8(y[0], y[1], a[0], a[1], wf);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int g = g0 + h;
          if (g >= ng) break;
          const bool band_t = g < tq;
          const int pg = band_t ? g : GB + (g - tq);                   // group id inside the panel buffers
          const double x0 = y[h].x * d0, x1 = y[h].y * d1;
          ypan[pg * 64 + f0] = y[h].x, ypan[pg * 64 + f1] = y[h].y;
          xpan[pg * 64 + f0] = x0, xpan[pg * 64 + f1] = x1;
          double* G = band_t ? K.band + ((size_t)Kc * Qs + 1 + g) * 64 : K.bord + ((size_t)Kc * nbt + (g - tq)) * 64;
          *reinterpret_cast<double2*>(G + r * 8 + 2 * k) = make_double2(x0, x1);
          const bool nz = __any_sync(0xffffffffu, x0 != 0.0 || x1 != 0.0);
          if (lane == 0 && nz) s_gnz[cur][pg] = 1;
        }
      }
    }
    if (WS)
      for (int e = tid; e < 64; e += nt) K.band[(size_t)Kc * Qs * 64 + e] = Tkk[e];
    __syncthreads();
    // (c) stream in block row Kc + Q (its slots are dead now), trailing updates on the fp64 tensor core;
    //     warp 0 takes the pair that completes the next diagonal tile and factors it right away
    const int In = Kc + Q;
#ifdef CHD_PROFILE
    const long long tc0 = clock64();
#endif
    if (WS && In < nbc) {
      // 16-byte cp.async chunks by the warps 1..15; warp 0 goes straight to the diagonal tile.  (A TMA producer warp, bulk
      // copies issued by a lane of an updating warp and dynamically dealt update blocks were slower: DESIGN.md section 9)
      for (int idx = tid - 32; idx < Q * 32 + nbt_s * 32; idx += nt - 32) {
        if (idx < 0) break;
        const int tile = idx >> 5, off = (idx & 31) * 2;
        if (tile < Q) {
          const int J = tile < GB ? Kc + 1 + tile : In;
          double* dst = tile < GB ? win + (size_t)tri(kslot, rs[tile]) * 64 : Tkk;
          chd_copy16(dst + off, K.band + ((size_t)J * Qs + (In - J)) * 64 + off, WS);
        } else {
          chd_copy16(Bk + (tile - Q) * 64 + off, K.bord + (size_t)In * nbt * 64 + (tile - Q) * 64 + off, WS);
        }
      }
    }
    if (warp == 0) {
      if (tq >= 1) {
        double* Tn = band_tile(0, 0);
        chd_tile_sub_xyT(Tn, xpan, ypan, lane);
        __syncwarp();
        const bool ok = chd_tile_ldl(Tn, dinv + 8 * (cur ^ 1), s_winv[cur ^ 1], lane);
        if (!ok && lane == 0) s_fail = 1;
      }
#ifdef CHD_PROFILE
      if (lane == 0) prof_diag += (double)(clock64() - tc0);
#endif
    } else {
      if (warp == 1) {
        for (int g = lane; g < GB; g += 32) {   // slot table of the next block column
          int v = kslot + 2 + g;
          while (v >= Q) v -= Q;
          s_rs[cur ^ 1][g] = v;
        }
        for (int g = lane; g < Gm; g += 32) s_gnz[cur ^ 1][g] = 0;
      }
      // every shared-memory window has Gm <= 64 (batch creation checks Q - 1 + nbt <= 64)
      if (!WS && Gm > 64) chd_kkt_update_wide(c, s_pairs, s_gnz[cur], GB, Gm, tq, band_tile, bord_tile);
      else chd_kkt_update_compact(c, s_pairs, s_cmp[warp], s_gnz[cur], GB, Gm, tq, band_tile, bord_tile);
#ifdef CHD_PROFILE
      if (lane == 0) atomicMax(&s_upd_end, (unsigned long long)clock64());
#endif
    }
    chd_copy_wait(WS);
    __syncthreads();
#ifdef CHD_PROFILE
    if (tid == 0) prof_upd += (double)((long long)s_upd_end - tc0);
#endif
    kslot = kslot + 1 == Q ? 0 : kslot + 1;
  }
#ifdef CHD_PROFILE
  if (tid == 0) c.I->prof[6] += prof_diag, c.I->prof[7] += prof_upd;
#endif
}

// dense LDL^T of the border Schur complement S = cc[0..nbl)^2 and solve S xb = rb (rb = row NBR of cc); xb goes to
// xs[8*nbc_max ..) and to the solution vector.  Sets s_fail on a bad pivot.
__device__ __forceinline__ void chd_kkt_border(const ChdDev& D, const ChdKktCtx& c, int& s_fail) {
  const int tid = c.tid, nt = c.nt, lane = c.lane, warp = c.warp, nbl = c.nbl, nbp8 = c.nbp8, NBR = c.NBR, Na = c.K.Na;
  double* cc = c.cc;
  for (int k = 0; k < nbl; ++k) {
    const double dk = cc[k * nbp8 + k];
    if (tid == 0 && !(dk > 0.0 && isfinite(dk))) s_fail = 1;
    __syncthreads();
    const double ik = 1.0 / dk;
    const int rem = nbl - k - 1;
    for (int idx = tid; idx < rem * rem; idx += nt) {
      const int i = k + 1 + idx / rem, j = k + 1 + idx % rem;
      if (j <= i) cc[i * nbp8 + j] -= cc[i * nbp8 + k] * ik * cc[j * nbp8 + k];
    }
    for (int j = k + 1 + tid; j < nbl; j += nt) cc[NBR * nbp8 + j] -= cc[j * nbp8 + k] * ik * cc[NBR * nbp8 + k];
    __syncthreads();
  }
  double* xb = c.xs + 8 * D.nbc_max;  // border solution
  if (warp == 0) {
    // column-oriented back-substitution by one warp: x_k = acc_k / d_k, then acc_j -= (L d)[k][j] x_k for j < k
    // (row k of cc holds the unscaled column entries; one division per unknown instead of one per matrix entry)
    for (int j = lane; j < nbl; j += 32) xb[j] = cc[NBR * nbp8 + j];
    __syncwarp();
    for (int k = nbl - 1; k >= 0; --k) {
      const double xk = xb[k] / cc[k * nbp8 + k];
      __syncwarp();
      for (int j = lane; j < k; j += 32) xb[j] -= cc[k * nbp8 + j] * xk;
      if (lane == 0) xb[k] = xk;
      __syncwarp();
    }
  }
  __syncthreads();
  for (int i = tid; i < nbl; i += nt) D.sol[(size_t)c.b * (D.Na_max + D.nb_max) + Na + i] = xb[i];
}

// backward substitution of the band, column oriented: acc = u - Lb^T xb; for K descending: x_K = L0^-T acc_K (warp 0),
// then acc_J -= L(K,J)^T x_K for the block row K (all threads).  Tiles are staged two block rows ahead.  The band
// solution goes to xs and to the solution vector.
template <bool WS>
__device__ __forceinline__ void chd_kkt_backsub(const ChdDev& D, const ChdKktCtx& c) {
  const ChdKT& K = c.K;
  const int tid = c.tid, nt = c.nt, lane = c.lane, warp = c.warp, Q = c.Q, Qs = c.Qs, nbt = c.nbt, nbl = c.nbl, nbc = c.nbc;
  const int NBR = c.NBR, Na = K.Na;
  double *xs = c.xs, *sol = D.sol + (size_t)c.b * (D.Na_max + D.nb_max);
  const double* xb = xs + 8 * D.nbc_max;
  double* accv = c.xs2;
  for (int i = tid; i < K.Np; i += nt) {
    const double* bt = K.bord + (size_t)(i >> 3) * nbt * 64 + (i & 7);
    double v = bt[NBR * 8];
    for (int q2 = 0; q2 < nbl; ++q2) v -= bt[q2 * 8] * xb[q2];
    accv[i] = v;
  }
  // staging buffers in the (now free) window + border window: two chunks of R block rows each,
  // row slot = diag tile | tiles (K, K-1-g), g = 0..q-1.  Warp 0 alone walks through a chunk (the recursion is
  // sequential anyway; without block barriers a block row costs ~0.5 k cycles instead of 1.4 k) while the other
  // warps prefetch the next chunk; one barrier per chunk.
  const int per = Q * 64;
  const int R = max(1, (int)((c.win_region - (WS ? c.n_even + c.xs_len : 0)) / 64) / (2 * Q));
  double* stg = c.win;
  auto stage_chunk = [&](int Ktop, int buf, int t0, int tstep) {   // block rows Ktop, Ktop-1, ... (R of them)
    for (int idx = t0; idx < R * Q * 32; idx += tstep) {
      const int rr = idx / (Q * 32), rem = idx - rr * (Q * 32);
      const int Kr = Ktop - rr;
      if (Kr < 0) break;
      const int tile = rem >> 5, off = (rem & 31) * 2;
      const int J = tile == 0 ? Kr : Kr - tile;     // tile 0: diagonal; tile g+1: (Kr, Kr-1-g)
      if (J < 0) continue;
      chd_copy16(stg + ((size_t)buf * R + rr) * per + tile * 64 + off, K.band + ((size_t)J * Qs + (Kr - J)) * 64 + off, WS);
    }
  };
  stage_chunk(nbc - 1, 0, tid, nt);
  chd_copy_wait(WS);
  __syncthreads();
  int buf = 0;
  for (int Ktop = nbc - 1; Ktop >= 0; Ktop -= R, buf ^= 1) {
    if (warp != 0) {
      stage_chunk(Ktop - R, buf ^ 1, tid - 32, nt - 32);
    } else {
      for (int rr = 0; rr < R && Ktop - rr >= 0; ++rr) {
        const int Kc = Ktop - rr;
        const double* T0 = stg + ((size_t)buf * R + rr) * per;
        double xk[8];
#pragma unroll
        for (int cl = 7; cl >= 0; --cl) {
          double v = accv[Kc * 8 + cl];
#pragma unroll
          for (int p = 7; p > cl; --p) v -= T0[p * 8 + cl] * xk[p];   // oldest unknown first: only the last link waits for xk[cl+1]
          xk[cl] = v;
        }
        if (lane < 8) {
          const int gi = Kc * 8 + lane;
          double v = xk[0];
#pragma unroll
          for (int cl = 1; cl < 8; ++cl) v = lane == cl ? xk[cl] : v;
          xs[gi] = v;
          if (gi < Na) sol[gi] = v;
        }
        const int nrow = min(K.q, Kc);   // tiles (Kc, Kc-1-g), g < nrow
        for (int idx = lane; idx < nrow * 8; idx += 32) {
          const int g = idx >> 3, cl = idx & 7;
          const double* T = T0 + (g + 1) * 64;
          double v = 0.0;
#pragma unroll
          for (int r = 0; r < 8; ++r) v += T[r * 8 + cl] * xk[r];
          accv[(Kc - 1 - g) * 8 + cl] -= v;
        }
        __syncwarp();
      }
    }
    chd_copy_wait(WS);
    __syncthreads();
  }
}

// No step from this factorisation: a coupling left the band (the stage fails) or a pivot broke down (the regularisation
// goes up and the iteration is repeated).  Returns true in either case.
__device__ __forceinline__ bool chd_kkt_no_step(const ChdDev& D, const ChdKktCtx& c, const int& s_fail) {
  ChdIpm& I = *c.I;
  const int tid = c.tid, nt = c.nt, n = c.n, m = c.m;
  const size_t ro = c.ro, vo = c.vo;
  if (I.band_ovf) {
    // a coupling left the band (stage 3 moved a polynomial boundary further than the layout allows): the stage fails and
    // the schedule goes on with the fixed-duration stage 4, as the reference does after a failed stage 3
    __syncthreads();
    if (tid == 0) I.status = -2, chd_stage_advance(D, I, -2, c.sg.snap_after);
    return true;
  }
  if (s_fail) {
    // numerical breakdown: raise the primal regularisation and retry next iteration (no step is taken)
    if (tid == 0) {
      I.delta_w = fmin(fmax(I.delta_w * 100.0, 1e-4), CHD_DW_MAX * 10);
      I.a_pr = 0.0, I.a_du = 0.0, I.dphi = 0.0;
      I.ls_fail += 1;
      I.step_ready = 1;
      I.kw_req = 1;
      if (I.delta_w > CHD_DW_MAX) I.status = -2, chd_stage_advance(D, I, -2, c.sg.snap_after);
    }
    for (int i = tid; i < n; i += nt) D.dx[vo + i] = 0.0;
    for (int r = tid; r < m; r += nt) D.ds[ro + r] = 0.0, D.dy[ro + r] = 0.0, D.dzL[ro + r] = 0.0, D.dzU[ro + r] = 0.0;
    return true;
  }
  return false;
}

// D. recover the full step, fraction-to-the-boundary, line-search inputs
__device__ __forceinline__ void chd_kkt_recover(const ChdDev& D, const ChdKktCtx& c) {
  ChdIpm& I = *c.I;
  const ChdSeq* h = c.h;
  const int b = c.b, tid = c.tid, nt = c.nt, n = c.n, m = c.m, n_act = c.n_act;
  const size_t ro = c.ro, vo = c.vo;
  const int *rf = c.rf, *vk = c.vk, *rk = c.rk, *ep = c.ep, *ec = c.ec;
  const double *Jv = c.Jv, *grad = c.grad, *sol = D.sol + (size_t)c.b * (D.Na_max + D.nb_max), sf = c.sf, mu = c.mu, tau = c.tau;
  double *vecn = c.vecn, *red = c.red;
  double* dx = D.dx + vo;
  for (int i = tid; i < n; i += nt) {
    const int k = vk[i];
    const double v = (k >= 0 && i < n_act) ? sol[k] : 0.0;
    dx[i] = v;
    vecn[i] = v;   // step in the unknowns (switch times for the durations): what the Jacobian columns refer to
  }
  __syncthreads();
  if (c.sg.opt_dur) {   // the line search moves x, i.e. phase durations: dd_k = dtau_k - dtau_{k-1}
    for (int ee = 0; ee < h->n_ee; ++ee)
      for (int k = 1 + tid; k < h->n_phases[ee] - 1; k += nt) dx[h->dur_xoff[ee] + k] = vecn[h->dur_xoff[ee] + k] - vecn[h->dur_xoff[ee] + k - 1];
  }
  double a_pr = 1.0, a_du = 1.0, a_dphi = 0.0, a_phi = 0.0;
  for (int i = tid; i < n; i += nt) a_dphi += sf * grad[i] * vecn[i];
  for (int r = tid; r < m; r += nt) {
    const int f = rf[r];
    if (!(f & CHD_ROW_ACTIVE)) continue;
    if (f & CHD_ROW_EQ) {
      D.dy[ro + r] = sol[rk[r]];
      D.ds[ro + r] = 0.0;
      continue;
    }
    const double sc = D.sc[ro + r], s = D.s[ro + r];
    double Jdx = 0.0;
    for (int e = ep[r]; e < ep[r + 1]; ++e) {
      const int col = ec[e];
      if (col >= 0) Jdx += Jv[e] * vecn[col];
    }
    const double riq = chd_row_res(f, sc * D.g[ro + r], D.dL[ro + r], s);
    const double ds = sc * Jdx + riq;
    const bool hl = f & CHD_ROW_HASL, hu = f & CHD_ROW_HASU;
    const ChdGaps gap = chd_row_gaps(f, s, D.dL[ro + r], D.dU[ro + r]);
    const double zL = D.zL[ro + r], zU = D.zU[ro + r];
    const ChdSigma sig = chd_row_sigma(f, gap, zL, zU);
    const double bvec = (hl ? mu / gap.L : 0.0) - (hu ? mu / gap.U : 0.0);   // mu times chd_row_mu_coef, rounded per bound
    const double dy = sig.sum() * ds - D.y[ro + r] - bvec;
    const double dzL = hl ? mu / gap.L - zL - sig.L * ds : 0.0;
    const double dzU = hu ? mu / gap.U - zU + sig.U * ds : 0.0;
    D.ds[ro + r] = ds, D.dy[ro + r] = dy, D.dzL[ro + r] = dzL, D.dzU[ro + r] = dzU;
    if (hl && ds < 0) a_pr = fmin(a_pr, -tau * gap.L / ds);
    if (hu && ds > 0) a_pr = fmin(a_pr, tau * gap.U / ds);
    if (hl && dzL < 0) a_du = fmin(a_du, -tau * zL / dzL);
    if (hu && dzU < 0) a_du = fmin(a_du, -tau * zU / dzU);
    if (hl) a_dphi -= mu * ds / gap.L;
    if (hu) a_dphi += mu * ds / gap.U;
    chd_row_barrier(f, mu, gap, a_phi);
  }
  a_pr = chd_block_min(a_pr, red);
  a_du = chd_block_min(a_du, red);
  const double dphi = chd_block_sum(a_dphi, red);
  const double phib = chd_block_sum(a_phi, red);
  if (tid == 0) {
    I.a_pr = a_pr, I.a_du = a_du, I.dphi = dphi;
    I.phi0 = sf * D.cost[2 * b] + phib;
    I.step_ready = 1;
    I.kw_req = 1;
  }
}

// One interior-point iteration of the sequence of this CTA: the phases above in order, each ending on a block barrier.
template <bool WS>
__device__ __forceinline__ void chd_kkt_body(const ChdDev& D) {
  __shared__ int s_fail;
  ChdIpm& I = D.ipm[blockIdx.x];
  if (I.phase != CHD_PH_RUN) return;
  ChdKktCtx c;
  chd_kkt_ctx_init<WS>(D, I, c);
  // per-phase cycle counters (scripts/prof_stage.py): compiled in only with -DCHD_PROFILE (extra barriers + clock reads)
#ifdef CHD_PROFILE
  long long tk0 = clock64();
#define CHD_PROF(slot) do { __syncthreads(); if (c.tid == 0) { long long t_ = clock64(); I.prof[slot] += (double)(t_ - tk0); tk0 = t_; } } while (0)
#else
#define CHD_PROF(slot) do { } while (0)
#endif
  if (chd_kkt_errors(D, c, s_fail)) return;
  CHD_PROF(0);
  chd_kkt_assemble(D, c);
  __syncthreads();
  CHD_PROF(1);
  chd_kkt_factor<WS>(c, s_fail);
  CHD_PROF(2);
  chd_kkt_border(D, c, s_fail);
  CHD_PROF(3);
  chd_kkt_backsub<WS>(D, c);
  CHD_PROF(4);
  if (chd_kkt_no_step(D, c, s_fail)) return;
  __syncthreads();
  chd_kkt_recover(D, c);
  CHD_PROF(5);
}
#undef CHD_PROF

// Kwork <- Kbase for the sequences whose KKT kernel asked for it; runs on a side stream, overlapped with the line
// search / evaluation kernels of the next iteration, on the SMs the one-CTA-per-sequence kernels leave idle
__global__ void __launch_bounds__(256) chd_k_kcopy(ChdDev D) {
  const int b = blockIdx.y;
  if (!D.ipm[b].kw_req) return;
  if (blockIdx.x == 0) chd_rhs_clear(D, b);
  if (chd_stage(D, b, D.ipm[b].stage).opt_dur && D.ipm[b].phase == CHD_PH_RUN) {
    // stage 3: the cost Hessian moves with the durations; chd_k_hess_dur rebuilds it into a cleared Kwork after the line search
    chd_hess_clear(D, b, D.Kwork + (size_t)b * D.kstride, blockIdx.x, gridDim.x);
    return;
  }
  const size_t cnt2 = D.kstride / 2, per = (cnt2 + gridDim.x - 1) / gridDim.x;
  const size_t lo = (size_t)blockIdx.x * per, hi = lo + per < cnt2 ? lo + per : cnt2;
  const double2* src = reinterpret_cast<const double2*>(D.Kbase + (size_t)b * D.kstride);
  double2* dst = reinterpret_cast<double2*>(D.Kwork + (size_t)b * D.kstride);
  const size_t nt = blockDim.x;
  size_t i = lo + threadIdx.x;
  for (; i + 3 * nt < hi; i += 4 * nt) {   // four independent 16-byte loads in flight per thread
    const double2 v0 = src[i], v1 = src[i + nt], v2 = src[i + 2 * nt], v3 = src[i + 3 * nt];
    dst[i] = v0, dst[i + nt] = v1, dst[i + 2 * nt] = v2, dst[i + 3 * nt] = v3;
  }
  for (; i < hi; i += nt) dst[i] = src[i];
}

// distance-row curvature terms of the next iteration (needs the iterate the line search just accepted); side stream,
// after chd_k_kcopy, grid (G, B)
__global__ void __launch_bounds__(256) chd_k_curv(ChdDev D) {
  __shared__ double s_ws[8 * 192];
  const int b = blockIdx.y;
  const ChdIpm& I = D.ipm[b];
  if (!I.kw_req || I.phase != CHD_PH_RUN) return;
  ChdKT K;
  chd_kt_init(D, D.seq + b, D.Kwork + (size_t)b * D.kstride, K);
  K.ovf = &D.ipm[b].band_ovf;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  chd_curv_rows(D, b, K, chd_stage(D, b, I.stage), blockIdx.x * 8 + warp, gridDim.x * 8, lane, s_ws + warp * 192);
}

// Jacobian-dependent matrix entries and right-hand side of every running sequence, on a Kwork that holds the cost
// Hessian and the distance-row curvature (chd_k_hess_zero / chd_k_hess_base on the first iteration of a stage,
// chd_k_kcopy / chd_k_hess_dur / chd_k_curv afterwards) and zeroed rhs0 / rhs1: grid (G, B), launched right before
// chd_k_kkt.  The reductions into L2 are the cost, so G CTAs per sequence on the SMs the one-CTA-per-sequence kernels
// leave idle take 1/G of the time.
__global__ void __launch_bounds__(256) chd_k_asm(ChdDev D) {
  const int b = blockIdx.y;
  const ChdIpm& I = D.ipm[b];
  if (I.phase != CHD_PH_RUN) return;
  ChdKT K;
  chd_kt_init(D, D.seq + b, D.Kwork + (size_t)b * D.kstride, K);
  K.ovf = &D.ipm[b].band_ovf;
  // the band chd_k_kkt factors in a fixed-duration stage: a Jacobian coupling outside it (stage 4 on the durations a
  // failed stage 3 left behind) fails the stage instead of being left out of the factorisation
  if (!chd_stage(D, b, I.stage).opt_dur) K.q = D.Qfix - 1;
  const size_t go = (size_t)b * (D.Na_max + D.nb_max);
  chd_assemble(D, b, K, I.delta_w, I.sf, blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x, D.rhs0 + go, D.rhs1 + go);
}

// fp64 throughput probe for the roofline denominators: mode 0 = DFMA chains, mode 1 = DMMA in the shape of the KKT
// factorisation's panel and trailing updates (mma.sync m16n8k8 f64, DMMA.16x8x8)
__global__ void __launch_bounds__(256) chd_k_fp64_peak(int mode, int iters, double* sink) {
  const double s = 1.0 + 1e-9 * threadIdx.x;
  double2 a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = make_double2(0.5 + i, 1.5 + i);
  if (mode == 0) {
    for (int it = 0; it < iters; ++it) {
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i].x = fma(a[i].x, s, 1e-3);
    }
  } else {
    const double2 x = make_double2(s, s), y = make_double2(1.0 - 1e-9 * threadIdx.x, 1.0);
    for (int it = 0; it < iters; ++it) {
#pragma unroll
      for (int i = 0; i < 4; ++i) chd_mma_16x8x8(a[2 * i], a[2 * i + 1], x, x, y);
    }
  }
  double t = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) t += a[i].x + a[i].y;
  if (t == 123.456) sink[threadIdx.x] = t;
}

// the elimination window lives in shared memory (WS) or, for very wide bands, in a global scratch buffer
__global__ void __launch_bounds__(CHD_KKT_THREADS) chd_k_kkt(ChdDev D) { chd_kkt_body<true>(D); }
__global__ void __launch_bounds__(CHD_KKT_THREADS) chd_k_kkt_gwin(ChdDev D) { chd_kkt_body<false>(D); }
