// Block-banded Cholesky solve of the kinematic initialisation's damped Gauss-Newton systems (see include/chd.h,
// chd_kin_solve).  One CTA per clip; per frame f of the clip (87 x 87 blocks padded to 88 = 11 tiles of 8):
//
//   A      = D_f + lam diag(max(diag D_f, 1e-12)) - L1_{f-1} L1_{f-1}^T - L2_{f-2} L2_{f-2}^T
//   A      = L0_f L0_f^T                                    tiled right-looking Cholesky (chd_tile_ldl per diagonal tile)
//   y_f    = L0_f^-1 (g_f - L1_{f-1} y_{f-1} - L2_{f-2} y_{f-2})
//   L1_f   = (B1_f - L2_{f-1} L1_{f-1}^T) L0_f^-T,   L2_f = B2_f L0_f^-T
//
// then s_f = L0_f^-T (y_f - L1_f^T s_{f+1} - L2_f^T s_{f+2}) backwards.  Every block product is a sum of 8 x 8 tile
// products on the fp64 tensor core (chd_tile_mma).  Blocks live in shared memory as 121 tiles in fragment order; three
// block slots (186 KB) hold the active blocks, and L0, L1, L2 of every frame go to `work` for the backward sweep and the
// next frames.  The diagonal tiles of a stored L0 hold the inverse of the Cholesky factor's diagonal tile instead of the
// tile itself: both sweeps only ever need that inverse.  No atomics: each clip's result depends only on its own inputs.
#include <cuda_runtime.h>

#include <cstdio>

#include "../../include/chd.h"
#include "chd_kkt_tiles.cuh"

#define KIN_N 87                 // unknowns per frame (root translation + 28 Euler triples)
#define KIN_P 88                 // padded block order
#define KIN_T 11                 // tiles per block row
#define KIN_BLK (KIN_P * KIN_P)  // doubles per padded block (121 tiles)
#define KIN_WARPS 16
#define KIN_THREADS (KIN_WARPS * 32)

// smem layout (doubles): three block slots | diagonal-tile scratch (row-major tile, W = L^-1, 1/d) |
// right-hand side, three solution vectors, two partial-sum vectors (88 each)
#define KIN_SMEM_DOUBLES (3 * KIN_BLK + 64 + 64 + 8 + 6 * KIN_P)

__device__ __forceinline__ double* kin_tile(double* S, int I, int J) { return S + (I * KIN_T + J) * 64; }
__device__ __forceinline__ const double* kin_tile(const double* S, int I, int J) { return S + (I * KIN_T + J) * 64; }
// element (R, C) of a block in tile / fragment order
__device__ __forceinline__ int kin_at(int R, int C) { return ((R >> 3) * KIN_T + (C >> 3)) * 64 + (R & 7) * 8 + chd_frag_col(C & 7); }

// accumulator of one tile: lane holds (r = lane>>2, c = 2k, 2k+1) with k = lane&3
__device__ __forceinline__ void kin_ld(const double* T, int lane, double& c0, double& c1) {
  const int r = lane >> 2, k = lane & 3;
  c0 = T[r * 8 + chd_frag_col(2 * k)];
  c1 = T[r * 8 + chd_frag_col(2 * k + 1)];
}
__device__ __forceinline__ void kin_st(double* T, int lane, double c0, double c1) {
  const int r = lane >> 2, k = lane & 3;
  T[r * 8 + chd_frag_col(2 * k)] = c0;
  T[r * 8 + chd_frag_col(2 * k + 1)] = c1;
}

// input block (87 x 87 row major, global) -> padded slot; diag: add the damping and put 1 on the padding diagonal
__device__ void kin_load_input(double* S, const double* src, bool diag, double lam) {
  for (int e = threadIdx.x; e < KIN_BLK; e += KIN_THREADS) {
    const int R = e / KIN_P, C = e - R * KIN_P;
    double v;
    if (R < KIN_N && C < KIN_N) {
      v = src[R * KIN_N + C];
      if (diag && R == C) v = __dadd_rn(v, __dmul_rn(lam, fmax(v, 1e-12)));   // rounded like the host's D + lam * diag
    } else {
      v = (diag && R == C) ? 1.0 : 0.0;
    }
    S[kin_at(R, C)] = v;
  }
}

__device__ void kin_copy(double* dst, const double* src) {
  const double2* s2 = reinterpret_cast<const double2*>(src);
  double2* d2 = reinterpret_cast<double2*>(dst);
  for (int e = threadIdx.x; e < KIN_BLK / 2; e += KIN_THREADS) d2[e] = s2[e];
}

// lower tiles (I >= J) of A -= X X^T (+ Y Y^T)
__device__ void kin_syrk(double* A, const double* X, const double* Y) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int idx = warp; idx < KIN_T * (KIN_T + 1) / 2; idx += KIN_WARPS) {
    int I = 0;
    while ((I + 1) * (I + 2) / 2 <= idx) ++I;
    const int J = idx - I * (I + 1) / 2;
    double c0, c1;
    kin_ld(kin_tile(A, I, J), lane, c0, c1);
    for (int K = 0; K < KIN_T; ++K) chd_tile_mma(c0, c1, kin_tile(X, I, K), kin_tile(X, J, K), lane);
    if (Y)
      for (int K = 0; K < KIN_T; ++K) chd_tile_mma(c0, c1, kin_tile(Y, I, K), kin_tile(Y, J, K), lane);
    kin_st(kin_tile(A, I, J), lane, c0, c1);
  }
}

// all tiles of A -= X Y^T
__device__ void kin_gemm_nt(double* A, const double* X, const double* Y) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int idx = warp; idx < KIN_T * KIN_T; idx += KIN_WARPS) {
    const int I = idx / KIN_T, J = idx - I * KIN_T;
    double c0, c1;
    kin_ld(kin_tile(A, I, J), lane, c0, c1);
    for (int K = 0; K < KIN_T; ++K) chd_tile_mma(c0, c1, kin_tile(X, I, K), kin_tile(Y, J, K), lane);
    kin_st(kin_tile(A, I, J), lane, c0, c1);
  }
}

// In-place tiled Cholesky of the lower tiles of A; the diagonal tiles receive the inverse of the factor's diagonal tiles.
// Returns false (uniformly over the CTA) when a pivot is not positive and finite.
__device__ bool kin_potrf(double* A, double* scr, double* winv, double* dinv, int* flag) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t = 0; t < KIN_T; ++t) {
    if (warp == 0) {
      double* Tt = kin_tile(A, t, t);
      for (int e = lane; e < 64; e += 32) scr[e] = Tt[(e >> 3) * 8 + chd_frag_col(e & 7)];
      __syncwarp();
      bool ok = chd_tile_ldl(scr, dinv, winv, lane);
      __syncwarp();
      ok = __all_sync(0xffffffffu, ok && (lane >= 8 || dinv[lane] > 0.0));
      // Cholesky factor of the tile = L D^1/2, its inverse = D^-1/2 L^-1: rows of W scaled by 1/sqrt(d)
      for (int e = lane; e < 64; e += 32) Tt[e] = winv[e] * sqrt(dinv[e >> 3]);
      if (lane == 0) *flag = ok ? 0 : 1;
    }
    __syncthreads();
    if (*flag) return false;
    // panel: A(I, t) <- A(I, t) Winv_t^T
    for (int I = t + 1 + warp; I < KIN_T; I += KIN_WARPS) {
      double c0 = 0.0, c1 = 0.0;
      chd_tile_mma(c0, c1, kin_tile(A, I, t), kin_tile(A, t, t), lane);
      __syncwarp();
      kin_st(kin_tile(A, I, t), lane, -c0, -c1);
    }
    __syncthreads();
    // trailing update of the lower tiles t < J <= I
    const int n = KIN_T - 1 - t;
    for (int idx = warp; idx < n * (n + 1) / 2; idx += KIN_WARPS) {
      int i = 0;
      while ((i + 1) * (i + 2) / 2 <= idx) ++i;
      const int I = t + 1 + i, J = t + 1 + idx - i * (i + 1) / 2;
      double c0, c1;
      kin_ld(kin_tile(A, I, J), lane, c0, c1);
      chd_tile_mma(c0, c1, kin_tile(A, I, t), kin_tile(A, J, t), lane);
      kin_st(kin_tile(A, I, J), lane, c0, c1);
    }
    __syncthreads();
  }
  return true;
}

// X <- X L^-T for up to two blocks X (L = factor in L0 storage), one warp per tile row, left looking over the columns
__device__ void kin_trsm(double* X0, double* X1, const double* L) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = X1 ? 2 * KIN_T : KIN_T;
  for (int task = warp; task < rows; task += KIN_WARPS) {
    double* X = task < KIN_T ? X0 : X1;
    const int I = task < KIN_T ? task : task - KIN_T;
    for (int J = 0; J < KIN_T; ++J) {
      double c0, c1;
      kin_ld(kin_tile(X, I, J), lane, c0, c1);
      for (int K = 0; K < J; ++K) chd_tile_mma(c0, c1, kin_tile(X, I, K), kin_tile(L, J, K), lane);
      kin_st(kin_tile(X, I, J), lane, c0, c1);
      __syncwarp();
      double e0 = 0.0, e1 = 0.0;
      chd_tile_mma(e0, e1, kin_tile(X, I, J), kin_tile(L, J, J), lane);
      __syncwarp();
      kin_st(kin_tile(X, I, J), lane, -e0, -e1);
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(KIN_THREADS, 1)
chd_k_kin_solve(const double* __restrict__ Dg, const double* __restrict__ B1g, const double* __restrict__ B2g,
                const double* __restrict__ g, const int32_t* __restrict__ seg, const double* __restrict__ lam,
                const int32_t* __restrict__ sel, int32_t K, int32_t F_total, double* __restrict__ work,
                double* __restrict__ s, int32_t* __restrict__ status) {
  extern __shared__ __align__(16) double sm[];
  __shared__ int flag;
  const int k = sel ? sel[blockIdx.x] : (int)blockIdx.x;
  if (k < 0 || k >= K) return;
  const int f0 = seg[k], F = seg[k + 1] - f0;
  if (f0 < 0 || F < 0 || f0 + F > F_total) {
    if (threadIdx.x == 0) status[k] = -1;
    return;
  }
  const int tid = threadIdx.x;
  double* slot[3] = {sm, sm + KIN_BLK, sm + 2 * KIN_BLK};
  double* scr = sm + 3 * KIN_BLK;
  double* winv = scr + 64;
  double* dinv = winv + 64;
  double* vb = dinv + 8;          // right-hand side being reduced
  double* vy[3] = {vb + KIN_P, vb + 2 * KIN_P, vb + 3 * KIN_P};   // y (forward) / s (backward) of the last three frames
  double* vp = vb + 4 * KIN_P;   // partial sums
  const double lk = lam[k];
  auto wblk = [&](int f, int which) { return work + ((size_t)(f0 + f) * 3 + which) * KIN_BLK; };

  // ---- factorisation and forward substitution ----
  double *SA = slot[0], *S1 = slot[1], *ST = slot[2];   // current diagonal, L1_{f-1}, scratch
  for (int f = 0; f < F; ++f) {
    const size_t gf = (size_t)(f0 + f);
    kin_load_input(SA, Dg + gf * KIN_N * KIN_N, true, lk);
    if (f >= 2) kin_copy(ST, wblk(f - 2, 2));
    __syncthreads();
    if (f >= 1) kin_syrk(SA, S1, f >= 2 ? ST : nullptr);
    __syncthreads();
    if (!kin_potrf(SA, scr, winv, dinv, &flag)) {
      if (tid == 0) status[k] = f + 1;
      return;
    }
    // forward: b = g_f - L1_{f-1} y_{f-1} - L2_{f-2} y_{f-2}
    double* y1 = vy[(f + 2) % 3];
    double* y2 = vy[(f + 1) % 3];
    double* y0 = vy[f % 3];
    if (tid < 2 * KIN_P) {
      const int r = tid % KIN_P, h = tid / KIN_P;
      double v = 0.0;
      if (h == 0 && f >= 1)
        for (int c = 0; c < KIN_P; ++c) v += S1[kin_at(r, c)] * y1[c];
      if (h == 1 && f >= 2)
        for (int c = 0; c < KIN_P; ++c) v += ST[kin_at(r, c)] * y2[c];
      vp[tid] = v;
    }
    __syncthreads();
    if (tid < KIN_P) vb[tid] = (tid < KIN_N ? g[gf * KIN_N + tid] : 0.0) - vp[tid] - vp[KIN_P + tid];
    __syncthreads();
    for (int J = 0; J < KIN_T; ++J) {
      if (tid < 8) {
        double v = 0.0;
        for (int c = 0; c < 8; ++c) v += SA[kin_at(8 * J + tid, 8 * J + c)] * vb[8 * J + c];
        y0[8 * J + tid] = v;
      }
      __syncthreads();
      if (tid >= 8 * (J + 1) && tid < KIN_P) {
        double v = vb[tid];
        for (int c = 0; c < 8; ++c) v -= SA[kin_at(tid, 8 * J + c)] * y0[8 * J + c];
        vb[tid] = v;
      }
      __syncthreads();
    }
    if (tid < KIN_N) s[gf * KIN_N + tid] = y0[tid];
    // L1_f = (B1_f - L2_{f-1} L1_{f-1}^T) L0^-T and L2_f = B2_f L0^-T
    const bool h1 = f + 1 < F, h2 = f + 2 < F;
    if (h1) {
      kin_load_input(ST, B1g + gf * KIN_N * KIN_N, false, 0.0);
      __syncthreads();
      if (f >= 1) kin_gemm_nt(ST, wblk(f - 1, 2), S1);
      __syncthreads();
    }
    if (h2) {
      kin_load_input(S1, B2g + gf * KIN_N * KIN_N, false, 0.0);
      __syncthreads();
    }
    if (h1) kin_trsm(ST, h2 ? S1 : nullptr, SA);
    __syncthreads();
    kin_copy(wblk(f, 0), SA);
    if (h1) kin_copy(wblk(f, 1), ST);
    if (h2) kin_copy(wblk(f, 2), S1);
    __syncthreads();
    double* t = S1;   // L1_f becomes the coupling block of the next frame
    S1 = ST;
    ST = t;
  }
  __syncthreads();   // work written above is read back below by other threads

  // ---- backward substitution ----
  for (int f = F - 1; f >= 0; --f) {
    const size_t gf = (size_t)(f0 + f);
    const bool h1 = f + 1 < F, h2 = f + 2 < F;
    double* s0 = vy[f % 3];
    double* s1 = vy[(f + 1) % 3];
    double* s2 = vy[(f + 2) % 3];
    kin_copy(slot[0], wblk(f, 0));
    if (h1) kin_copy(slot[1], wblk(f, 1));
    if (h2) kin_copy(slot[2], wblk(f, 2));
    __syncthreads();
    // b = y_f - L1_f^T s_{f+1} - L2_f^T s_{f+2}
    if (tid < 2 * KIN_P) {
      const int c = tid % KIN_P, h = tid / KIN_P;
      double v = 0.0;
      if (h == 0 && h1)
        for (int r = 0; r < KIN_P; ++r) v += slot[1][kin_at(r, c)] * s1[r];
      if (h == 1 && h2)
        for (int r = 0; r < KIN_P; ++r) v += slot[2][kin_at(r, c)] * s2[r];
      vp[tid] = v;
    }
    __syncthreads();
    if (tid < KIN_P) vb[tid] = (tid < KIN_N ? s[gf * KIN_N + tid] : 0.0) - vp[tid] - vp[KIN_P + tid];
    __syncthreads();
    const double* L = slot[0];
    for (int J = KIN_T - 1; J >= 0; --J) {
      if (tid < 8) {
        double v = 0.0;
        for (int r = 0; r < 8; ++r) v += L[kin_at(8 * J + r, 8 * J + tid)] * vb[8 * J + r];
        s0[8 * J + tid] = v;
      }
      __syncthreads();
      if (tid < 8 * J) {
        double v = vb[tid];
        for (int r = 0; r < 8; ++r) v -= L[kin_at(8 * J + r, tid)] * s0[8 * J + r];
        vb[tid] = v;
      }
      __syncthreads();
    }
    if (tid < KIN_N) s[gf * KIN_N + tid] = s0[tid];
    __syncthreads();
  }
  if (tid == 0) status[k] = 0;
}

extern "C" int64_t chd_kin_work_bytes(int32_t F_total) {
  if (F_total < 0) return -1;
  return (int64_t)F_total * 3 * KIN_BLK * (int64_t)sizeof(double);
}

extern "C" int chd_kin_solve(const double* D, const double* B1, const double* B2, const double* g, const int32_t* seg,
                             const double* lam, const int32_t* sel, int32_t n_sel, int32_t K, int32_t F_total, double* work,
                             double* s, int32_t* status, void* stream) {
  if (K < 0 || F_total < 0 || n_sel < 0) return -1;
  if (!seg || !lam || !status) return -1;
  if (F_total > 0 && (!D || !g || !work || !s)) return -1;
  if ((F_total > 1 && !B1) || (F_total > 2 && !B2)) return -1;
  if (sel && n_sel > K) return -1;
  const int n = sel ? n_sel : K;
  if (n == 0) return 0;
  const size_t smem = KIN_SMEM_DOUBLES * sizeof(double);
  cudaError_t e = cudaFuncSetAttribute(chd_k_kin_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) {
    fprintf(stderr, "libchd: chd_kin_solve: %s\n", cudaGetErrorString(e));
    return -100 - (int)e;
  }
  chd_k_kin_solve<<<n, KIN_THREADS, smem, (cudaStream_t)stream>>>(D, B1, B2, g, seg, lam, sel, K, F_total, work, s, status);
  e = cudaGetLastError();
  if (e != cudaSuccess) {
    fprintf(stderr, "libchd: chd_kin_solve: %s\n", cudaGetErrorString(e));
    return -100 - (int)e;
  }
  return 0;
}
