// Shared host/device definitions for the batched phys-optim NLP (product code, sm_90a).
//
// What this replaces: the per-iteration evaluation the reference performs through ifopt's virtual
// ConstraintSet/CostTerm interface (towr_phys_optim/src/constraints/*.cpp, src/costs/*.cpp,
// src/models/humanoid_rigid_body_dynamics.cpp) on top of TOWR's NodeSpline / EulerConverter.
// Here the spline algebra is table driven: every sequence carries flat per-spline tables (polynomial
// durations, cumulative end times, node -> variable index) built once on the host (chd_layout.cpp), and
// every constraint row / cost sample is an independent work item.
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define CHD_HD __host__ __device__ __forceinline__
#else
#define CHD_HD inline
#endif

#define CHD_MAX_EE 4
#define CHD_MAX_SPLINES (2 + 2 * CHD_MAX_EE)

// constraint-set types in the master row order
enum ChdSetType : int {
  CHD_SET_ACC = 0,      // towr SplineAccConstraint (nlp_formulation.cpp:349-360); a = spline id
  CHD_SET_TERRAIN = 1,  // towr TerrainConstraint   (nlp_formulation.cpp:321-331); a = ee
  CHD_SET_ROM = 2,      // leg_length_constraint.cpp;                              a = ee
  CHD_SET_DYN = 3,      // humanoid_dynamic_constraint.cpp
  CHD_SET_FORCE = 4,    // towr ForceConstraint     (nlp_formulation.cpp:334-346); a = ee
  CHD_SET_HEEL = 5,     // ee_dist_constraint.cpp;                                 a,b = ee pair
  CHD_SET_HEIGHT = 6,   // height_constraint.cpp;                                  a = ee
  CHD_SET_TOTTIME = 7,  // total_duration_constraint.cpp:60-82 (stage 3 only);     a = ee, one row
  CHD_SET_DURPOS = 8,   // PhaseDurations bounds (0, 500) of parameters.cpp:60 as rows d_k >= 0 (stage 3 only); a = ee
};
#define CHD_TAU_TRUST 0.04   /* [s] stage 3 keeps every switch time within this distance of its input value: the layout sizes the
                                band for the polynomials that can move onto a sample time within it (line-search trials beyond are refused) */
#define CHD_MAX_DUR 96   /* most phase-duration variables (sum over feet of P-1) stage 3 handles as dense border unknowns
                            (more need banded switch times: chd_phys_options) */
// stage bit masks over set types (phys_optim.cpp:554-749, SURVEY Appendix B)
#define CHD_MASK(t) (1u << (t))
enum ChdStage : int { CHD_STAGE_11 = 0, CHD_STAGE_12 = 1, CHD_STAGE_21 = 2, CHD_STAGE_22 = 3, CHD_STAGE_3 = 4, CHD_STAGE_4 = 5 };

struct ChdSet {
  int type, a, b;
  int row0;     // first row in the master row vector
  int nitems;   // work items (rows = nitems * rows_per_item(type))
  int tab;      // offset into the per-sequence int table (node id lists) where needed
};

CHD_HD int chd_rows_per_item(int type) { return type == CHD_SET_ACC ? 3 : (type == CHD_SET_DYN ? 6 : (type == CHD_SET_FORCE ? 5 : 1)); }
CHD_HD int chd_slots_per_row(int type, int n_ee) {
  switch (type) {
    case CHD_SET_ACC: return 6;
    case CHD_SET_TERRAIN: return 3;
    case CHD_SET_FORCE: return 3;
    // time-located rows end with two switch-time slots per foot they touch (stage 3; columns -1 otherwise)
    case CHD_SET_ROM: return 36 + 2;
    case CHD_SET_DYN: return 24 + 24 * n_ee + 2 * n_ee;
    case CHD_SET_HEEL: return 24 + 4;
    case CHD_SET_TOTTIME: return 1;
    case CHD_SET_DURPOS: return 2;
    default: return 12 + 2;  // HEIGHT
  }
}

// Per-sequence header.  All "off" members index batch-global flat arrays.
struct ChdSeq {
  int n_ee, F, n_splines;
  int n;          // optimisation variables (ifopt stacking: base_lin, base_ang, ee motion.., ee force..)
  int m;          // rows of the master constraint vector
  int nsets;
  int nslots;     // Jacobian value slots
  int n_dyn, n_rom, n_smooth;
  int Na, nb, w;  // KKT: banded unknowns, border unknowns (stance positions, then the switch times), half bandwidth
  int n_dur;      // phase-duration variables (0: stage 3 not available for this sequence), the last n_dur entries of x
  int nb_fix;     // border unknowns of the fixed-duration stages (= nb - n_dur, or nb when dur_band)
  int w_fix;      // half bandwidth of the fixed-duration stages (static pattern); w additionally covers the polynomials
                  // stage 3 may move onto a sample time
  int dur_band;   // 1: the switch times are band unknowns (time ordered) instead of the last n_dur border unknowns; the
                  // fixed-duration stages give them a unit diagonal and no couplings
  int dur_xoff[CHD_MAX_EE];   // first duration variable of every foot (P - 1 of them)
  double dt, T, mass, grav, mu, max_leg, max_heel, heel_dist, force_limit;
  double normal[3], point[3], gvec[3], nrm[3], tan1[3], tan2[3], dhdx, dhdy;
  int sp_npoly[CHD_MAX_SPLINES];
  int sp_xoff[CHD_MAX_SPLINES];   // first variable of the spline's set in x
  int sp_nvar[CHD_MAX_SPLINES];
  int start_contact[CHD_MAX_EE], n_phases[CHD_MAX_EE];
};

// spline ids: 0 base_lin, 1 base_ang, 2+ee motion, 2+n_ee+ee force
CHD_HD int chd_sp_motion(int ee) { return 2 + ee; }
CHD_HD int chd_sp_force(int n_ee, int ee) { return 2 + n_ee + ee; }

// ---------------------------------------------------------------------------------------------
// Cubic Hermite segment: value/derivative weights of the four node values (p0, v0, p1, v1) at local
// time t of a segment of duration T (closed forms: SURVEY 8(c); towr CubicHermitePolynomial).
// w[deriv][k], k = 0:p0 1:v0 2:p1 3:v1
// ---------------------------------------------------------------------------------------------
struct ChdBasis {
  double w[3][4];
};
CHD_HD void chd_basis(double t, double T, ChdBasis& b) {
  const double iT = 1.0 / T, iT2 = iT * iT, iT3 = iT2 * iT;
  const double t2 = t * t, t3 = t2 * t;
  b.w[0][0] = 2 * t3 * iT3 - 3 * t2 * iT2 + 1;
  b.w[0][1] = t - 2 * t2 * iT + t3 * iT2;
  b.w[0][2] = 3 * t2 * iT2 - 2 * t3 * iT3;
  b.w[0][3] = t3 * iT2 - t2 * iT;
  b.w[1][0] = 6 * t2 * iT3 - 6 * t * iT2;
  b.w[1][1] = 3 * t2 * iT2 - 4 * t * iT + 1;
  b.w[1][2] = 6 * t * iT2 - 6 * t2 * iT3;
  b.w[1][3] = 3 * t2 * iT2 - 2 * t * iT;
  b.w[2][0] = 12 * t * iT3 - 6 * iT2;
  b.w[2][1] = 6 * t * iT2 - 4 * iT;
  b.w[2][2] = 6 * iT2 - 12 * t * iT3;
  b.w[2][3] = 6 * t * iT2 - 2 * iT;
}

// Segment lookup (towr Spline::GetSegmentID): first segment with cumulative end >= t - 1e-10.
// tend[] holds the sequentially accumulated end times.
CHD_HD int chd_locate(const double* tend, int npoly, double t, double* tl) {
  const double tt = t - 1e-10;
  int lo = 0, hi = npoly - 1;
  while (lo < hi) {  // first i with tend[i] >= tt
    int mid = (lo + hi) >> 1;
    if (tend[mid] >= tt) hi = mid; else lo = mid + 1;
  }
  *tl = t - (lo > 0 ? tend[lo - 1] : 0.0);
  return lo;
}

// ---------------------------------------------------------------------------------------------
// Euler ZYX kinematics (towr EulerConverter, SURVEY 8(c)): R = Rz(z) Ry(y) Rx(x), omega = M(e) edot.
// ---------------------------------------------------------------------------------------------
struct ChdTrig {
  double sx, cx, sy, cy, sz, cz;
};
CHD_HD void chd_trig(const double e[3], ChdTrig& t) {
  t.sx = sin(e[0]); t.cx = cos(e[0]); t.sy = sin(e[1]); t.cy = cos(e[1]); t.sz = sin(e[2]); t.cz = cos(e[2]);
}
CHD_HD void chd_R(const ChdTrig& t, double R[9]) {
  R[0] = t.cy * t.cz; R[1] = t.cz * t.sx * t.sy - t.cx * t.sz; R[2] = t.sx * t.sz + t.cx * t.cz * t.sy;
  R[3] = t.cy * t.sz; R[4] = t.cx * t.cz + t.sx * t.sy * t.sz; R[5] = t.cx * t.sy * t.sz - t.cz * t.sx;
  R[6] = -t.sy;       R[7] = t.cy * t.sx;                      R[8] = t.cx * t.cy;
}
// dR/de_k, k = 0(x) 1(y) 2(z)
CHD_HD void chd_dR(const ChdTrig& t, int k, double D[9]) {
  if (k == 0) {
    D[0] = 0; D[1] = t.cz * t.cx * t.sy + t.sx * t.sz;  D[2] = t.cx * t.sz - t.sx * t.cz * t.sy;
    D[3] = 0; D[4] = -t.sx * t.cz + t.cx * t.sy * t.sz; D[5] = -t.sx * t.sy * t.sz - t.cz * t.cx;
    D[6] = 0; D[7] = t.cy * t.cx;                       D[8] = -t.sx * t.cy;
  } else if (k == 1) {
    D[0] = -t.sy * t.cz; D[1] = t.cz * t.sx * t.cy; D[2] = t.cx * t.cz * t.cy;
    D[3] = -t.sy * t.sz; D[4] = t.sx * t.cy * t.sz; D[5] = t.cx * t.cy * t.sz;
    D[6] = -t.cy;        D[7] = -t.sy * t.sx;       D[8] = -t.cx * t.sy;
  } else {
    D[0] = -t.cy * t.sz; D[1] = -t.sz * t.sx * t.sy - t.cx * t.cz; D[2] = t.sx * t.cz - t.cx * t.sz * t.sy;
    D[3] = t.cy * t.cz;  D[4] = -t.cx * t.sz + t.sx * t.sy * t.cz; D[5] = t.cx * t.sy * t.cz + t.sz * t.sx;
    D[6] = 0; D[7] = 0; D[8] = 0;
  }
}
CHD_HD void chd_M(const ChdTrig& t, double M[9]) {
  M[0] = t.cy * t.cz; M[1] = -t.sz; M[2] = 0;
  M[3] = t.cy * t.sz; M[4] = t.cz;  M[5] = 0;
  M[6] = -t.sy;       M[7] = 0;     M[8] = 1;
}
// dM/de_y, dM/de_z (dM/de_x = 0)
CHD_HD void chd_dM_y(const ChdTrig& t, double D[9]) {
  D[0] = -t.sy * t.cz; D[1] = 0; D[2] = 0; D[3] = -t.sy * t.sz; D[4] = 0; D[5] = 0; D[6] = -t.cy; D[7] = 0; D[8] = 0;
}
CHD_HD void chd_dM_z(const ChdTrig& t, double D[9]) {
  D[0] = -t.cy * t.sz; D[1] = -t.cz; D[2] = 0; D[3] = t.cy * t.cz; D[4] = -t.sz; D[5] = 0; D[6] = 0; D[7] = 0; D[8] = 0;
}
// second derivatives d2M/dy2, d2M/dydz, d2M/dz2
CHD_HD void chd_d2M(const ChdTrig& t, double Dyy[9], double Dyz[9], double Dzz[9]) {
  for (int i = 0; i < 9; ++i) Dyy[i] = Dyz[i] = Dzz[i] = 0.0;
  Dyy[0] = -t.cy * t.cz; Dyy[3] = -t.cy * t.sz; Dyy[6] = t.sy;
  Dyz[0] = t.sy * t.sz;  Dyz[3] = -t.sy * t.cz;
  Dzz[0] = -t.cy * t.cz; Dzz[1] = t.sz; Dzz[3] = -t.cy * t.sz; Dzz[4] = -t.cz;
}

CHD_HD void chd_mv(const double A[9], const double v[3], double r[3]) {
  r[0] = A[0] * v[0] + A[1] * v[1] + A[2] * v[2];
  r[1] = A[3] * v[0] + A[4] * v[1] + A[5] * v[2];
  r[2] = A[6] * v[0] + A[7] * v[1] + A[8] * v[2];
}
CHD_HD void chd_mtv(const double A[9], const double v[3], double r[3]) {  // A^T v
  r[0] = A[0] * v[0] + A[3] * v[1] + A[6] * v[2];
  r[1] = A[1] * v[0] + A[4] * v[1] + A[7] * v[2];
  r[2] = A[2] * v[0] + A[5] * v[1] + A[8] * v[2];
}
CHD_HD void chd_cross(const double a[3], const double b[3], double r[3]) {
  r[0] = a[1] * b[2] - a[2] * b[1];
  r[1] = a[2] * b[0] - a[0] * b[2];
  r[2] = a[0] * b[1] - a[1] * b[0];
}
CHD_HD double chd_dot(const double a[3], const double b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
