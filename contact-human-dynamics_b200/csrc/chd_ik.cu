// Damped least-squares full-body IK for K clips of one skeleton in one launch per iteration (see include/chd.h,
// chd_ik_solve).  One CTA per frame; per frame and iteration, with the frame's local rotations R and translations P:
//
//   FK (level by level over the joint depth), e = euler_of(R), world rotation axes w_ka = parentR_k ax_a(e_k),
//   err    = goal - p_targets
//   A      = J J^T + lam^2 I           3T x 3T, packed lower triangle in shared memory, built block by block from the
//                                      ancestor structure: block (t1, t2) sums the rotation columns of the strict common
//                                      ancestors of t1 and t2 and the translation columns of lca(t1, t2) and its ancestors
//   A      = L L^T                     scalar right-looking Cholesky, one warp per trailing row
//   y      = A^-1 err,   dx = J^T y    dx[k] sums over the targets below k (bit masks over the targets)
//   x      = [e; P] + dx + s (x_{f-1} + x_{f+1} - 2 x),   R = rot_of(x[:3J]),  P = x[3J:]
//
// The Jacobian is never formed.  The state is double-buffered in `work`, so a frame reads its neighbours' previous
// iterate without a grid-wide barrier; no atomics, so each clip's result is bitwise independent of the batch.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../include/chd.h"

#define IK_THREADS 512
#define IK_MAX_J 128
#define IK_MAX_T 64

struct IkParams {
  int J, T, maxdepth, translate;
  double lam2, smooth;
  const unsigned long long* mstrict;   // [J] bit t: target t is a strict descendant of joint k
  const unsigned long long* mall;      // [J] bit t: target t is joint k or below it
  const int* parents;                  // [J]
  const int* depth;                    // [J]
  const int* targets;                  // [T]
  const int* lca;                      // [T * T] lowest common ancestor of two targets (-1: none)
  const int* lo;                       // [F_total] first frame of the frame's clip
  const int* hi;                       // [F_total] last frame of the frame's clip
};

// work layout: tables (see IkParams, 256-byte aligned) | R0 | P0 | R1 | P1 (state ping-pong, F_total x J x 9 / x 3)
static size_t ik_table_bytes(int F_total, int J, int T) {
  const size_t b = 16 * (size_t)J + 4 * (2 * (size_t)J + T + (size_t)T * T) + 8 * (size_t)F_total;
  return (b + 255) & ~(size_t)255;
}

static size_t ik_smem_bytes(int J, int T) {
  const size_t n = 3 * (size_t)T;
  return 16 * (size_t)J + 8 * (n * (n + 1) / 2 + 54 * (size_t)J + 2 * n) + 4 * (2 * (size_t)J + T);
}

__device__ __forceinline__ double ik_euler_c(const double* R, int c) {   // x, y, z with R = Rz Ry Rx
  if (c == 0) return atan2(R[7], R[8]);
  if (c == 1) return -asin(fmin(fmax(R[6], -1.0), 1.0));
  return atan2(R[3], R[0]);
}

__global__ void __launch_bounds__(IK_THREADS, 1)
chd_k_ik_iter(const IkParams p, const double* __restrict__ Rs, const double* __restrict__ Ps, double* __restrict__ Rd,
              double* __restrict__ Pd, const double* __restrict__ goal) {
  extern __shared__ __align__(16) double sm[];
  const int J = p.J, T = p.T, n = 3 * T;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int f = blockIdx.x;
  unsigned long long* ms = reinterpret_cast<unsigned long long*>(sm);
  unsigned long long* ma = ms + J;
  double* A = reinterpret_cast<double*>(ma + J);
  double* Rl = A + n * (n + 1) / 2;   // local rotations; reused for the new Euler angles
  double* Pl = Rl + 9 * J;
  double* e = Pl + 3 * J;
  double* gR = e + 3 * J;
  double* gP = gR + 9 * J;
  double* W = gP + 3 * J;             // world rotation axes: W[9k + 3a + i]
  double* prs = W + 9 * J;            // parent's global rotation (identity for a root), row major
  double* M = prs + 9 * J;            // prs prs^T
  double* b = M + 9 * J;              // err, then L^-1 err in place
  double* y = b + n;
  int* par = reinterpret_cast<int*>(y + n);
  int* dep = par + J;
  int* tgt = dep + J;

  for (int i = tid; i < J; i += IK_THREADS) {
    ms[i] = p.mstrict[i];
    ma[i] = p.mall[i];
    par[i] = p.parents[i];
    dep[i] = p.depth[i];
  }
  for (int i = tid; i < T; i += IK_THREADS) tgt[i] = p.targets[i];
  const double* Rf = Rs + (size_t)f * J * 9;
  const double* Pf = Ps + (size_t)f * J * 3;
  for (int i = tid; i < 9 * J; i += IK_THREADS) Rl[i] = Rf[i];
  for (int i = tid; i < 3 * J; i += IK_THREADS) Pl[i] = Pf[i];
  __syncthreads();

  // ---- Euler angles and forward kinematics ----
  if (tid < J)
    for (int c = 0; c < 3; ++c) e[3 * tid + c] = ik_euler_c(Rl + 9 * tid, c);
  for (int d = 0; d <= p.maxdepth; ++d) {
    if (tid < J && dep[tid] == d) {
      const int j = tid, q = par[j];
      if (q < 0) {
        for (int i = 0; i < 9; ++i) gR[9 * j + i] = Rl[9 * j + i];
        for (int i = 0; i < 3; ++i) gP[3 * j + i] = Pl[3 * j + i];
      } else {
        const double* G = gR + 9 * q;
        const double* L = Rl + 9 * j;
        const double* t = Pl + 3 * j;
        for (int r = 0; r < 3; ++r) {
          for (int c = 0; c < 3; ++c) gR[9 * j + 3 * r + c] = G[3 * r] * L[c] + G[3 * r + 1] * L[3 + c] + G[3 * r + 2] * L[6 + c];
          gP[3 * j + r] = gP[3 * q + r] + (G[3 * r] * t[0] + G[3 * r + 1] * t[1] + G[3 * r + 2] * t[2]);
        }
      }
    }
    __syncthreads();
  }

  // ---- parent rotations, world axes, error ----
  if (tid < J) {
    const int j = tid, q = par[j];
    double pr[9];
    for (int i = 0; i < 9; ++i) pr[i] = q < 0 ? (i % 4 == 0 ? 1.0 : 0.0) : gR[9 * q + i];
    const double cz = cos(e[3 * j + 2]), sz = sin(e[3 * j + 2]), cy = cos(e[3 * j + 1]), sy = sin(e[3 * j + 1]);
    const double ax[3][3] = {{cz * cy, sz * cy, -sy}, {-sz, cz, 0.0}, {0.0, 0.0, 1.0}};
    for (int a = 0; a < 3; ++a)
      for (int i = 0; i < 3; ++i) W[9 * j + 3 * a + i] = pr[3 * i] * ax[a][0] + pr[3 * i + 1] * ax[a][1] + pr[3 * i + 2] * ax[a][2];
    for (int i = 0; i < 3; ++i)
      for (int k = 0; k < 3; ++k) M[9 * j + 3 * i + k] = pr[3 * i] * pr[3 * k] + pr[3 * i + 1] * pr[3 * k + 1] + pr[3 * i + 2] * pr[3 * k + 2];
    for (int i = 0; i < 9; ++i) prs[9 * j + i] = pr[i];
  }
  for (int i = tid; i < n; i += IK_THREADS) {
    const int t = i / 3, c = i - 3 * t;
    b[i] = goal[((size_t)f * T + t) * 3 + c] - gP[3 * tgt[t] + c];
  }
  __syncthreads();

  // ---- A = J J^T + lam^2 I, one 3 x 3 block (t1 >= t2) per thread ----
  for (int q = tid; q < T * (T + 1) / 2; q += IK_THREADS) {
    int t1 = (int)((sqrtf(8.0f * q + 1.0f) - 1.0f) * 0.5f);
    while (t1 * (t1 + 1) / 2 > q) --t1;
    while ((t1 + 1) * (t1 + 2) / 2 <= q) ++t1;
    const int t2 = q - t1 * (t1 + 1) / 2;
    const int j1 = tgt[t1], j2 = tgt[t2], l = p.lca[t1 * T + t2];
    const double* p1 = gP + 3 * j1;
    const double* p2 = gP + 3 * j2;
    double acc[9];
    for (int i = 0; i < 9; ++i) acc[i] = 0.0;
    // rotation columns: joints strictly above both targets
    for (int k = (l == j1 || l == j2) ? (l >= 0 ? par[l] : -1) : l; k >= 0; k = par[k]) {
      const double* pk = gP + 3 * k;
      const double r1[3] = {p1[0] - pk[0], p1[1] - pk[1], p1[2] - pk[2]};
      const double r2[3] = {p2[0] - pk[0], p2[1] - pk[1], p2[2] - pk[2]};
      for (int a = 0; a < 3; ++a) {
        const double* w = W + 9 * k + 3 * a;
        const double c1[3] = {w[1] * r1[2] - w[2] * r1[1], w[2] * r1[0] - w[0] * r1[2], w[0] * r1[1] - w[1] * r1[0]};
        const double c2[3] = {w[1] * r2[2] - w[2] * r2[1], w[2] * r2[0] - w[0] * r2[2], w[0] * r2[1] - w[1] * r2[0]};
        for (int i = 0; i < 3; ++i)
          for (int j = 0; j < 3; ++j) acc[3 * i + j] += c1[i] * c2[j];
      }
    }
    // translation columns: the common ancestor and everything above it
    if (p.translate)
      for (int k = l; k >= 0; k = par[k])
        for (int i = 0; i < 9; ++i) acc[i] += M[9 * k + i];
    for (int i = 0; i < 3; ++i) {
      const int r = 3 * t1 + i;
      for (int j = 0; j < 3 && (t1 != t2 || j <= i); ++j) {
        const int c = 3 * t2 + j;
        A[r * (r + 1) / 2 + c] = r == c ? acc[3 * i + j] + p.lam2 : acc[3 * i + j];
      }
    }
  }
  __syncthreads();

  // ---- Cholesky: step j updates the trailing triangle with the unscaled column j (A_ik -= A_ij A_kj / A_jj) and
  //      scales column j - 1, which no thread reads in step j ----
  double piv_prev = 1.0;
  for (int j = 0; j < n; ++j) {
    const double piv = A[j * (j + 1) / 2 + j];
    const double rp = 1.0 / piv;
    for (int i = j + 1 + warp; i < n; i += IK_THREADS / 32) {
      double* Ai = A + i * (i + 1) / 2;
      const double aij = Ai[j] * rp;
      for (int k = j + 1 + lane; k <= i; k += 32) Ai[k] -= aij * A[k * (k + 1) / 2 + j];
    }
    if (j > 0) {
      const double s = sqrt(piv_prev);
      for (int i = j - 1 + tid; i < n; i += IK_THREADS) {
        double& v = A[i * (i + 1) / 2 + j - 1];
        v = i == j - 1 ? s : v / s;
      }
    }
    piv_prev = piv;
    __syncthreads();
  }
  if (tid == 0) A[(n - 1) * n / 2 + n - 1] = sqrt(piv_prev);
  __syncthreads();

  // ---- y = L^-T L^-1 err on warp 0: forward by rows, backward by columns (row j of L is contiguous) ----
  if (warp == 0) {
    for (int i = 0; i < n; ++i) {
      const double* Li = A + i * (i + 1) / 2;
      double s = 0.0;
      for (int k = lane; k < i; k += 32) s += Li[k] * b[k];
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) b[i] = (b[i] - s) / Li[i];
      __syncwarp();
    }
    for (int j = n - 1; j >= 0; --j) {
      const double* Lj = A + j * (j + 1) / 2;
      const double yj = b[j] / Lj[j];
      __syncwarp();
      for (int i = lane; i < j; i += 32) b[i] -= Lj[i] * yj;
      if (lane == 0) y[j] = yj;
      __syncwarp();
    }
  }
  __syncthreads();

  // ---- dx = J^T y and the smoothed update, one thread per (joint, axis) ----
  const int f_lo = p.lo[f], f_hi = p.hi[f];
  const int fp = f > f_lo ? f - 1 : f, fa = f < f_hi ? f + 1 : f;
  double* xn = Rl;   // R is not read again in this iteration
  if (tid < 3 * J) {
    const int k = tid / 3, a = tid - 3 * k;
    const double* w = W + 9 * k + 3 * a;
    const double* pk = gP + 3 * k;
    double dr = 0.0;
    for (unsigned long long m = ms[k]; m; m &= m - 1) {
      const int t = __ffsll((long long)m) - 1;
      const double* pt = gP + 3 * tgt[t];
      const double r[3] = {pt[0] - pk[0], pt[1] - pk[1], pt[2] - pk[2]};
      const double u[3] = {w[1] * r[2] - w[2] * r[1], w[2] * r[0] - w[0] * r[2], w[0] * r[1] - w[1] * r[0]};
      dr += u[0] * y[3 * t] + u[1] * y[3 * t + 1] + u[2] * y[3 * t + 2];
    }
    const double xr = e[3 * k + a];
    const double xrp = ik_euler_c(Rs + ((size_t)fp * J + k) * 9, a), xra = ik_euler_c(Rs + ((size_t)fa * J + k) * 9, a);
    xn[3 * k + a] = xr + dr + p.smooth * (xrp + xra - 2.0 * xr);
    const double xt = Pl[3 * k + a];
    double pn = xt;
    if (p.translate) {
      const double* pr = prs + 9 * k;
      double dt = 0.0;
      for (unsigned long long m = ma[k]; m; m &= m - 1) {
        const int t = __ffsll((long long)m) - 1;
        dt += pr[a] * y[3 * t] + pr[3 + a] * y[3 * t + 1] + pr[6 + a] * y[3 * t + 2];
      }
      const double xtp = Ps[((size_t)fp * J + k) * 3 + a], xta = Ps[((size_t)fa * J + k) * 3 + a];
      pn = xt + dt + p.smooth * (xtp + xta - 2.0 * xt);
    }
    Pd[((size_t)f * J + k) * 3 + a] = pn;
  }
  __syncthreads();
  if (tid < J) {
    const double* x = xn + 3 * tid;
    const double cx = cos(x[0]), sx = sin(x[0]), cy = cos(x[1]), sy = sin(x[1]), cz = cos(x[2]), sz = sin(x[2]);
    double* R = Rd + ((size_t)f * J + tid) * 9;
    R[0] = cz * cy;
    R[1] = cz * sy * sx - sz * cx;
    R[2] = cz * sy * cx + sz * sx;
    R[3] = sz * cy;
    R[4] = sz * sy * sx + cz * cx;
    R[5] = sz * sy * cx - cz * sx;
    R[6] = -sy;
    R[7] = cy * sx;
    R[8] = cy * cx;
  }
}

extern "C" int64_t chd_ik_work_bytes(int32_t F_total, int32_t J, int32_t T) {
  if (F_total < 0 || J < 1 || J > IK_MAX_J || T < 1 || T > IK_MAX_T) return -1;
  return (int64_t)(ik_table_bytes(F_total, J, T) + 2 * (size_t)F_total * J * 12 * sizeof(double));
}

static int ik_cuda_error(cudaError_t e) {
  fprintf(stderr, "libchd: chd_ik_solve: %s\n", cudaGetErrorString(e));
  return -100 - (int)e;
}

extern "C" int chd_ik_solve(int32_t J, const int32_t* parents, int32_t T, const int32_t* targets, const int32_t* seg, int32_t K,
                            int32_t F_total, double* R, double* P, const double* goal, int32_t iterations, double damping,
                            double smoothness, int32_t translate, double* work, void* stream) {
  // ---- validation (host arrays only; nothing is launched on a bad argument) ----
  if (J < 1 || J > IK_MAX_J || T < 1 || T > IK_MAX_T || K < 0 || F_total < 0 || iterations < 0) return -1;
  if (!parents || !targets || !seg) return -1;
  if (parents[0] != -1) return -1;
  for (int j = 1; j < J; ++j)
    if (parents[j] < -1 || parents[j] >= j) return -1;
  for (int t = 0; t < T; ++t)
    if (targets[t] < 0 || targets[t] >= J) return -1;
  if (seg[0] != 0 || seg[K] != F_total) return -1;
  for (int k = 0; k < K; ++k)
    if (seg[k + 1] < seg[k]) return -1;
  if (F_total > 0 && (!R || !P || !goal || !work)) return -1;
  if (F_total == 0 || iterations == 0) return 0;

  // ---- ancestor tables ----
  std::vector<unsigned char> tab(ik_table_bytes(F_total, J, T), 0);
  unsigned long long* mstrict = reinterpret_cast<unsigned long long*>(tab.data());
  unsigned long long* mall = mstrict + J;
  int* par = reinterpret_cast<int*>(mall + J);
  int* dep = par + J;
  int* tg = dep + J;
  int* lca = tg + T;
  int* lo = lca + T * T;
  int* hi = lo + F_total;
  int maxdepth = 0;
  for (int j = 0; j < J; ++j) {
    par[j] = parents[j];
    dep[j] = par[j] < 0 ? 0 : dep[par[j]] + 1;
    maxdepth = dep[j] > maxdepth ? dep[j] : maxdepth;
  }
  for (int t = 0; t < T; ++t) {
    tg[t] = targets[t];
    mall[targets[t]] |= 1ull << t;
    for (int k = par[targets[t]]; k >= 0; k = par[k]) {
      mstrict[k] |= 1ull << t;
      mall[k] |= 1ull << t;
    }
  }
  for (int t1 = 0; t1 < T; ++t1)
    for (int t2 = 0; t2 < T; ++t2) {
      int a = tg[t1], c = tg[t2];
      while (a != c && a >= 0 && c >= 0) {
        if (dep[a] >= dep[c]) a = par[a];
        else c = par[c];
      }
      lca[t1 * T + t2] = (a == c) ? a : -1;
    }
  for (int k = 0; k < K; ++k)
    for (int fr = seg[k]; fr < seg[k + 1]; ++fr) {
      lo[fr] = seg[k];
      hi[fr] = seg[k + 1] - 1;
    }

  cudaStream_t st = (cudaStream_t)stream;
  char* wb = reinterpret_cast<char*>(work);
  const size_t nR = (size_t)F_total * J * 9, nP = (size_t)F_total * J * 3;
  double* bufR[2] = {reinterpret_cast<double*>(wb + tab.size()), nullptr};
  double* bufP[2] = {bufR[0] + nR, nullptr};
  bufR[1] = bufP[0] + nP;
  bufP[1] = bufR[1] + nR;
  IkParams p;
  p.J = J;
  p.T = T;
  p.maxdepth = maxdepth;
  p.translate = translate ? 1 : 0;
  const double lam = damping * (1.0 / (1.0 + 0.001));
  p.lam2 = lam * lam;
  p.smooth = smoothness;
  p.mstrict = reinterpret_cast<const unsigned long long*>(wb);
  p.mall = p.mstrict + J;
  p.parents = reinterpret_cast<const int*>(p.mall + J);
  p.depth = p.parents + J;
  p.targets = p.depth + J;
  p.lca = p.targets + T;
  p.lo = p.lca + T * T;
  p.hi = p.lo + F_total;

  const size_t smem = ik_smem_bytes(J, T);
  cudaError_t e = cudaFuncSetAttribute(chd_k_ik_iter, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return ik_cuda_error(e);
  if ((e = cudaMemcpyAsync(work, tab.data(), tab.size(), cudaMemcpyHostToDevice, st)) != cudaSuccess) return ik_cuda_error(e);
  if ((e = cudaMemcpyAsync(bufR[0], R, nR * sizeof(double), cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return ik_cuda_error(e);
  if ((e = cudaMemcpyAsync(bufP[0], P, nP * sizeof(double), cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return ik_cuda_error(e);
  for (int it = 0; it < iterations; ++it) {
    const int s = it & 1;
    chd_k_ik_iter<<<F_total, IK_THREADS, smem, st>>>(p, bufR[s], bufP[s], bufR[s ^ 1], bufP[s ^ 1], goal);
    if ((e = cudaGetLastError()) != cudaSuccess) return ik_cuda_error(e);
  }
  const int s = iterations & 1;
  if ((e = cudaMemcpyAsync(R, bufR[s], nR * sizeof(double), cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return ik_cuda_error(e);
  if ((e = cudaMemcpyAsync(P, bufP[s], nP * sizeof(double), cudaMemcpyDeviceToDevice, st)) != cudaSuccess) return ik_cuda_error(e);
  return 0;
}
