// TEST INFRASTRUCTURE ONLY -- kernel-level harness of the KKT factorisation and solve (csrc/chd_kkt.cu) for
// tests/test_kkt_factor_gpu.py.  Two kernels, one per elimination window (shared memory / global scratch), run the
// product's own phase functions in the order chd_kkt_body runs them -- context, right-hand side, band LDL^T, border
// Schur complement, back-substitution -- on tile-format matrices the test packs, without the error measures, the
// no-step test and the step recovery.  Never loaded by the product; adds nothing to libchd.so.
//
// C ABI (ctypes):
//   chd_kkt_harness_plan : the ChdKktPlan batch creation would make for these strides, with this library's kernels'
//                          static shared memory, for a given per-block opt-in limit
//   chd_kkt_harness_run  : one launch over a batch of B sequences; returns the factored tile buffers, the solutions,
//                          the per-sequence fail flags and the kernel that ran.  Every allocation is freed on return.
#include <cstdio>
#include <cstring>

#include "../../contact-human-dynamics_b200/csrc/chd_kkt.cu"

template <bool WS>
__global__ void __launch_bounds__(CHD_KKT_THREADS) chd_kkt_harness(ChdDev D, const double* mu, int* fail) {
  __shared__ int s_fail;
  ChdIpm& I = D.ipm[blockIdx.x];
  ChdKktCtx c;
  chd_kkt_ctx_init<WS>(D, I, c);
  if (c.tid == 0) s_fail = 0;
  c.mu = mu[blockIdx.x];
  c.tau = 1.0;
  c.polish = false;
  c.delta_w = I.delta_w;
  __syncthreads();
  chd_kkt_assemble(D, c);
  __syncthreads();
  chd_kkt_factor<WS>(c, s_fail);
  chd_kkt_border(D, c, s_fail);
  chd_kkt_backsub<WS>(D, c);
  __syncthreads();
  if (c.tid == 0) fail[blockIdx.x] = s_fail;
}

static int harness_err(char* err, int len, const char* what, cudaError_t e) {
  if (err && len > 0) snprintf(err, len, "%s: %s", what, cudaGetErrorString(e));
  return -1;
}
#define HCUDA(x)                                          \
  do {                                                    \
    cudaError_t e_ = (x);                                 \
    if (e_ != cudaSuccess) {                              \
      rc = harness_err(err, errlen, #x, e_);              \
      goto done;                                          \
    }                                                     \
  } while (0)

static cudaError_t harness_plan(int Na_max, int nb_max, int w_max, int w_fix_max, int n_max, long long optin, ChdKktPlan* P) {
  cudaFuncAttributes fa_kkt, fa_gwin;
  cudaError_t e = cudaFuncGetAttributes(&fa_kkt, chd_kkt_harness<true>);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa_gwin, chd_kkt_harness<false>);
  if (e != cudaSuccess) return e;
  *P = chd_kkt_plan(Na_max, nb_max, w_max, w_fix_max, n_max, fa_kkt.sharedSizeBytes, fa_gwin.sharedSizeBytes, (size_t)optin);
  return cudaSuccess;
}

extern "C" int chd_kkt_harness_plan_size() { return (int)sizeof(ChdKktPlan); }

// optin <= 0: the device's per-block opt-in limit.  Returns 0, or -1 with a message in err.
extern "C" int chd_kkt_harness_plan(int Na_max, int nb_max, int w_max, int w_fix_max, int n_max, long long optin, ChdKktPlan* out,
                                    char* err, int errlen) {
  int rc = 0;
  if (optin <= 0) {
    int dev = 0, v = 0;
    HCUDA(cudaGetDevice(&dev));
    HCUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    optin = v;
  }
  HCUDA(harness_plan(Na_max, nb_max, w_max, w_fix_max, n_max, optin, out));
done:
  return rc;
}

// K: B x kstride tile-format matrices (band | bord | corn), factored in place on return.  rhs0 / rhs1: B x (Na_max +
// nb_max) as chd_k_asm leaves them (band unknowns first, border unknowns from Na_max).  sol: B x (Na_max + nb_max).
// Na / nb / nb_fix / opt_dur per sequence (opt_dur 0: a fixed-duration stage, which solves for nb_fix border unknowns
// and Qfix band tiles per block column).  which: 1 = chd_k_kkt's shared-memory window ran, 0 = the global one.
// Returns 0; -1 on a CUDA error, -2 when the plan does not fit (message in err).
extern "C" int chd_kkt_harness_run(int B, int Na_max, int nb_max, int w_max, int w_fix_max, int n_max, long long optin,
                                   const int* Na, const int* nb, const int* nb_fix, const int* opt_dur, double* K,
                                   const double* rhs0, const double* rhs1, const double* mu, double* sol, int* fail, int* which,
                                   char* err, int errlen) {
  int rc = 0;
  ChdKktPlan P;
  ChdDev D;
  memset(&D, 0, sizeof(D));
  ChdSeq* hseq = nullptr;
  ChdIpm* hipm = nullptr;
  double* d_mu = nullptr;
  int* d_fail = nullptr;
  const size_t nv = (size_t)Na_max + nb_max;
  if (optin <= 0) {
    int dev = 0, v = 0;
    HCUDA(cudaGetDevice(&dev));
    HCUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    optin = v;
  }
  HCUDA(harness_plan(Na_max, nb_max, w_max, w_fix_max, n_max, optin, &P));
  if (P.status != CHD_KKT_FITS) {
    if (err && errlen > 0) snprintf(err, errlen, "KKT plan status %d (Q=%d nbt=%d)", P.status, P.Q, P.nbt);
    return -2;
  }
  *which = P.win_smem;
  D.B = B, D.n_max = n_max, D.Na_max = Na_max, D.nb_max = nb_max, D.w_max = w_max;
  D.win_smem = P.win_smem, D.nbc_max = P.nbc_max, D.Q = P.Q, D.Qfix = P.Qfix, D.nbt = P.nbt, D.win_tiles = P.win_tiles;
  D.pan_doubles = P.pan_doubles, D.kstride = P.kstride, D.scratch_stride = P.scratch_stride;
  hseq = new ChdSeq[B];
  hipm = new ChdIpm[B];
  memset(hseq, 0, sizeof(ChdSeq) * B);
  memset(hipm, 0, sizeof(ChdIpm) * B);
  for (int b = 0; b < B; ++b) {
    hseq[b].Na = Na[b], hseq[b].nb = nb[b], hseq[b].nb_fix = nb_fix[b], hseq[b].n_dur = nb[b] - nb_fix[b];
    hipm[b].phase = CHD_PH_RUN, hipm[b].stage = opt_dur[b] ? 1 : 0, hipm[b].sf = 1.0;
  }
  {
    ChdStageDev hst[2];
    memset(hst, 0, sizeof(hst));
    hst[1].opt_dur = 1;
    HCUDA(cudaMalloc((void**)&D.stages, sizeof(hst)));
    HCUDA(cudaMemcpy((void*)D.stages, hst, sizeof(hst), cudaMemcpyHostToDevice));
  }
  HCUDA(cudaMalloc((void**)&D.seq, sizeof(ChdSeq) * B));
  HCUDA(cudaMemcpy((void*)D.seq, hseq, sizeof(ChdSeq) * B, cudaMemcpyHostToDevice));
  HCUDA(cudaMalloc((void**)&D.ipm, sizeof(ChdIpm) * B));
  HCUDA(cudaMemcpy(D.ipm, hipm, sizeof(ChdIpm) * B, cudaMemcpyHostToDevice));
  HCUDA(cudaMalloc((void**)&D.Kwork, sizeof(double) * B * P.kstride));
  HCUDA(cudaMemcpy(D.Kwork, K, sizeof(double) * B * P.kstride, cudaMemcpyHostToDevice));
  HCUDA(cudaMalloc((void**)&D.rhs0, sizeof(double) * B * nv));
  HCUDA(cudaMemcpy(D.rhs0, rhs0, sizeof(double) * B * nv, cudaMemcpyHostToDevice));
  HCUDA(cudaMalloc((void**)&D.rhs1, sizeof(double) * B * nv));
  HCUDA(cudaMemcpy(D.rhs1, rhs1, sizeof(double) * B * nv, cudaMemcpyHostToDevice));
  HCUDA(cudaMalloc((void**)&D.sol, sizeof(double) * B * nv));
  HCUDA(cudaMemset(D.sol, 0, sizeof(double) * B * nv));
  if (P.scratch_stride) {
    HCUDA(cudaMalloc((void**)&D.scratch, sizeof(double) * B * P.scratch_stride));
    HCUDA(cudaMemset(D.scratch, 0, sizeof(double) * B * P.scratch_stride));
  }
  HCUDA(cudaMalloc((void**)&d_mu, sizeof(double) * B));
  HCUDA(cudaMemcpy(d_mu, mu, sizeof(double) * B, cudaMemcpyHostToDevice));
  HCUDA(cudaMalloc((void**)&d_fail, sizeof(int) * B));
  HCUDA(cudaMemset(d_fail, 0xff, sizeof(int) * B));
  if (P.win_smem) {
    HCUDA(cudaFuncSetAttribute(chd_kkt_harness<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P.smem_bytes));
    chd_kkt_harness<true><<<B, CHD_KKT_THREADS, P.smem_bytes>>>(D, d_mu, d_fail);
  } else {
    HCUDA(cudaFuncSetAttribute(chd_kkt_harness<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P.smem_bytes));
    chd_kkt_harness<false><<<B, CHD_KKT_THREADS, P.smem_bytes>>>(D, d_mu, d_fail);
  }
  HCUDA(cudaGetLastError());
  HCUDA(cudaDeviceSynchronize());
  HCUDA(cudaMemcpy(K, D.Kwork, sizeof(double) * B * P.kstride, cudaMemcpyDeviceToHost));
  HCUDA(cudaMemcpy(sol, D.sol, sizeof(double) * B * nv, cudaMemcpyDeviceToHost));
  HCUDA(cudaMemcpy(fail, d_fail, sizeof(int) * B, cudaMemcpyDeviceToHost));
done:
  cudaFree((void*)D.stages);
  cudaFree((void*)D.seq);
  cudaFree(D.ipm);
  cudaFree(D.Kwork);
  cudaFree(D.rhs0);
  cudaFree(D.rhs1);
  cudaFree(D.sol);
  cudaFree(D.scratch);
  cudaFree(d_mu);
  cudaFree(d_fail);
  delete[] hseq;
  delete[] hipm;
  return rc;
}
