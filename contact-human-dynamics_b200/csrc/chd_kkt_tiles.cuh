// Tiled (8x8) symmetric arrowhead storage of the condensed KKT matrix and its factorisation primitives
// (product code, device only).
//
//   [ A  B^T ]   A : banded, order Np (= Na padded to a multiple of 8 with identity), half bandwidth <= 8*q
//   [ B  C   ]   B : dense border rows (long-lived stance-position variables) + the right-hand side as one more row
//
// Global layout per sequence (doubles):  band | bord | corn
//   band : block column J (8 columns) holds Q = q+1 tiles (I = J .. J+q), tile = 8x8 row major
//   bord : block column J holds nbt tiles of border rows (row b -> tile b>>3, r = b&7)
//   corn : nbp8 x nbp8 dense, row major (nbp8 = 8*nbt)
// The right-hand side is stored as the border row right behind the border unknowns of the stage (chd_k_kkt).
// The factorisation is an unpivoted block LDL^T (the matrix is quasi-definite by construction, DESIGN.md):
// per block column: 8x8 diagonal LDL^T (warp shuffles) that also yields the inverse of its unit factor, the panel as one
// FP64 tensor-core (mma.sync m8n8k4) product per tile, and rank-8 tensor-core trailing updates of the elimination window
// (shared memory, or in place in global memory for wide bands).
#pragma once
#include "chd_dev.h"

struct ChdKT {
  int Na, Np, nbc, q, Q, nbt, nbp8;
  double *band, *bord, *corn;
  int* ovf;   // set when a coupling falls outside the band (run-time patterns of stage 3), nullptr: not checked
};

__device__ __forceinline__ void chd_kt_init(const ChdDev& D, const ChdSeq* h, double* base, ChdKT& K) {
  K.Na = h->Na;
  K.Np = (h->Na + 7) & ~7;
  K.nbc = K.Np >> 3;
  K.Q = D.Q;
  K.q = D.Q - 1;
  K.nbt = D.nbt;
  K.nbp8 = 8 * D.nbt;
  K.ovf = nullptr;
  K.band = base;
  K.bord = base + (size_t)D.nbc_max * D.Q * 64;
  K.corn = K.bord + (size_t)D.nbc_max * D.nbt * 64;
}

// add v at position (i, j) of the symmetric matrix (lower triangle storage); unknown index >= Na = border
__device__ __forceinline__ void chd_kadd(const ChdKT& K, int i, int j, double v) {
  if (i < j) { int t = i; i = j; j = t; }
  if (i < K.Na) {
    const int J = j >> 3;
    if ((i >> 3) - J > K.q) {   // outside the band the layout sized: only possible once stage 3 has moved a polynomial boundary far
      if (K.ovf) *K.ovf = 1;
      return;
    }
    atomicAdd(K.band + ((size_t)J * K.Q + ((i >> 3) - J)) * 64 + (i & 7) * 8 + (j & 7), v);
  } else if (j < K.Na) {
    const int b = i - K.Na;
    atomicAdd(K.bord + ((size_t)(j >> 3) * K.nbt + (b >> 3)) * 64 + (b & 7) * 8 + (j & 7), v);
  } else {
    atomicAdd(K.corn + (size_t)(i - K.Na) * K.nbp8 + (j - K.Na), v);
  }
}
// diagonal element (k, k), unknown index as in chd_kadd (k >= Na: border); band = true addresses the band for any
// k < Np, the identity padding rows Na .. Np-1 included
__device__ __forceinline__ double* chd_kdiag(const ChdKT& K, int k, bool band = false) {
  if (band || k < K.Na) return K.band + ((size_t)(k >> 3) * K.Q) * 64 + (k & 7) * 9;
  return K.corn + (size_t)(k - K.Na) * (K.nbp8 + 1);
}

// D(8x8) = C - X * Y^T for row-major 8x8 tiles X, Y (fp64 tensor core, two k-steps of m8n8k4).
// Fragment layout (PTX ISA, mma.m8n8k4 f64): A[row = lane>>2][k = lane&3], B[k = lane&3][col = lane>>2],
// C/D[row = lane>>2][col = 2*(lane&3) + {0,1}].
// accumulator form: (c0, c1) -= (X Y^T)[r][2k, 2k+1].
// X and Y are panel tiles in *fragment order*: element (row r, column c) of the 8x8 tile sits at
// r*8 + chd_frag_col(c), so that lane (r = lane>>2, k = lane&3) finds its two operands {c = k, c = k+4} of both
// k-steps in one aligned 16-byte word at [2*lane] -- a conflict-free LDS.128 instead of two 4-way bank-conflicted
// 8-byte loads per operand (the trailing updates were shared-memory bound on exactly those conflicts).
__device__ __forceinline__ int chd_frag_col(int c) { return ((c & 3) << 1) | (c >> 2); }
__device__ __forceinline__ void chd_tile_mma(double& c0, double& c1, const double* X, const double* Y, int lane) {
  const double2 xa = *reinterpret_cast<const double2*>(X + 2 * lane);
  const double2 yb = *reinterpret_cast<const double2*>(Y + 2 * lane);
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(-xa.x), "d"(yb.x));
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(-xa.y), "d"(yb.y));
}
__device__ __forceinline__ void chd_tile_sub_xyT(double* C, const double* X, const double* Y, int lane) {
  const int r = lane >> 2, k = lane & 3;
  double c0 = C[r * 8 + 2 * k], c1 = C[r * 8 + 2 * k + 1];
  chd_tile_mma(c0, c1, X, Y, lane);
  C[r * 8 + 2 * k] = c0;
  C[r * 8 + 2 * k + 1] = c1;
}

// In-place LDL^T of the lower triangle of an 8x8 row-major tile by one warp (lanes replicate rows r = lane&7).
// On exit: strict lower part = unit L, diagonal = d.  dinv[8] receives 1/d and winv[64] the inverse W = L^-1
// (unit lower triangular) in fragment order, so that the panel below the tile becomes one tensor-core product
// Y = A W^T per 8x8 panel tile instead of a scalar triangular solve per row.  Returns false on a bad pivot.
__device__ __forceinline__ bool chd_tile_ldl(double* T, double* dinv, double* winv, int lane) {
  const int r = lane & 7;
  double a[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) a[c] = c <= r ? T[r * 8 + c] : 0.0;
  bool ok = true;
  // W = L^-1 by forward substitution on the rows, w = e_r - sum_{j<r} L[r][j] W[j][:], interleaved with the
  // elimination: column p of L is final after pivot p and row p of W after step p-1, so step p of the recurrence has no
  // dependence on the next pivot's divide -> multiply -> fma chain and fills its latency
  double w[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) w[c] = c == r ? 1.0 : 0.0;
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const double dp = __shfl_sync(0xffffffffu, a[p], p, 8);
    ok = ok && (fabs(dp) > 1e-300) && isfinite(dp);
    const double inv = 1.0 / dp;   // correctly rounded, as in the CPU oracle (DESIGN §9 item 0)
    const double lr = a[p] * inv;
#pragma unroll
    for (int c = p + 1; c < 8; ++c) {
      const double acp = __shfl_sync(0xffffffffu, a[p], c, 8);  // unscaled A[c][p]
      if (r >= c) a[c] -= lr * acp;
    }
    if (r > p) a[p] = lr;
    if (lane == p) dinv[p] = inv;
    if (p < 7) {
#pragma unroll
      for (int c = 0; c <= p; ++c) {
        const double wpc = __shfl_sync(0xffffffffu, w[c], p, 8);
        if (r > p) w[c] -= lr * wpc;
      }
    }
  }
  if (lane < 8) {
#pragma unroll
    for (int c = 0; c < 8; ++c)
      if (c <= r) T[r * 8 + c] = a[c];
  }
  if (lane < 8) {
#pragma unroll
    for (int j = 0; j < 4; ++j) reinterpret_cast<double2*>(winv + r * 8)[j] = make_double2(w[j], w[j + 4]);   // fragment order
  }
  return ok;
}

// 16-byte copy global -> window.  With the window in shared memory this is an asynchronous cp.async (LDGSTS);
// chd_copy_wait() must precede the barrier that publishes the data.
__device__ __forceinline__ void chd_copy16(double* dst, const double* src, int smem) {
  if (smem) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(src) : "memory");
  } else {
    dst[0] = src[0];
    dst[1] = src[1];
  }
}
__device__ __forceinline__ void chd_copy_wait(int smem) {
  if (smem) asm volatile("cp.async.wait_all;" ::: "memory");
}

// window slot of band tile (I, J), I >= J, both inside a sliding window of Q block rows/columns
__device__ __forceinline__ int chd_win_slot(int I, int J, int Q) {
  const int a = I % Q, b = J % Q;
  const int hi = a > b ? a : b, lo = a > b ? b : a;
  return hi * (hi + 1) / 2 + lo;
}
