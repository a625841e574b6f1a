// Contact classifier, 3xTF32 fast mode (CHD_CONTACT_TF32X3): the three large layers 352 -> 1024 -> 512 -> 128 on the
// sm_90a tensor core.
//
// wgmma has no fp32-input kind, and a single TF32 product perturbs the logits by about 1e-3 relative, enough to flip
// labels whose logits sit near zero.  So every fp32 operand x is split into two TF32 values, hi = rna(x) and
// lo = rna(x - hi), and each product is summed as lo_a*hi_b + hi_a*lo_b + hi_a*hi_b in one fp32 accumulator (the
// dropped lo*lo term is about 2^-22 relative).
//   chd_k_contact_split     : W [K][N] fp32 -> hi, lo [N][K] (once, when the mode is switched on)
//   chd_k_contact_gather_tc : the windows of chd_k_contact_gather (same arithmetic), written as hi and lo planes
//   chd_k_contact_gemm_tc   : one Linear + eval BatchNorm + ReLU layer; 128 x 128 CTA tile, K tiles of 32 fp32 (one
//                             128-byte row, 128-byte swizzle) loaded by TMA into a 3-stage ring of hi+lo tiles (64 KB a
//                             stage), one producer warp and two consumer warpgroups each issuing
//                             wgmma.m64n128k8.f32.tf32.tf32 from shared-memory descriptors.  The epilogue writes the next
//                             layer's hi and lo planes (plain fp32 after the last layer, for chd_k_contact_tail).
// wgmma takes tf32 operands K-major only, which the activations [M][K] are; the weights get their own [N][K] copies.
#include "chd_contact_tc.h"

#include <cudaTypedefs.h>

#include <cstdint>
#include <cstdio>

#define TC_WIN 9
#define TC_J 13
#define TC_IN 351
#define TC_K0 352
#define TC_BM 128
#define TC_BN 128
#define TC_BK 32                                // fp32 per K tile: one 128-byte row
#define TC_STAGES 3
#define TC_TILE_BYTES (TC_BM * TC_BK * 4)       // 16 KB: one operand plane of one stage
#define TC_STAGE_BYTES (4 * TC_TILE_BYTES)      // A hi, A lo, W hi, W lo
#define TC_SMEM (TC_STAGES * TC_STAGE_BYTES + 1024)
#define TC_THREADS 288                          // two consumer warpgroups + one producer warp

static __device__ __constant__ int c_tc_lower_joints[TC_J] = {8, 9, 10, 11, 12, 13, 14, 19, 20, 21, 22, 23, 24};

#define TC_CUDA(x)                                                                           \
  do {                                                                                       \
    cudaError_t e_ = (x);                                                                    \
    if (e_ != cudaSuccess) {                                                                 \
      fprintf(stderr, "libchd: CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      return -100 - (int)e_;                                                                 \
    }                                                                                        \
  } while (0)

static __device__ __forceinline__ float tc_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// ------------------------------------------------------------------ mbarrier / TMA / wgmma -----------------------
static __device__ __forceinline__ void tc_mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
static __device__ __forceinline__ void tc_mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
static __device__ __forceinline__ void tc_mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
static __device__ __forceinline__ void tc_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// 2-D tile {32 fp32 of K, 128 rows} at (k, row) -> shared memory, completion counted on bar
static __device__ __forceinline__ void tc_tma_load(uint32_t dst, const CUtensorMap* map, int k, int row, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(k), "r"(row), "r"(bar)
      : "memory");
}
// Shared-memory matrix descriptor of a K-major tile with 128-byte swizzle: rows of 128 bytes, 8-row groups 1024 bytes
// apart (stride byte offset), leading byte offset unused for this layout; the tile base is 1024-byte aligned.
static __device__ __forceinline__ uint64_t tc_desc(uint32_t addr) {
  return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
#define TC_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
// d[64] += A (64 x 8, tf32) * B (8 x 128, tf32), both from shared memory
static __device__ __forceinline__ void tc_wgmma(float* d, uint64_t da, uint64_t db) {
  asm volatile(
      "{\n .reg .pred p;\n setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
      "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}\n"
      : TC_D8(0), TC_D8(8), TC_D8(16), TC_D8(24), TC_D8(32), TC_D8(40), TC_D8(48), TC_D8(56)
      : "l"(da), "l"(db), "r"(1));
}

// ------------------------------------------------------------------ kernels ---------------------------------------
// W [K][N] fp32 -> hi, lo [N][K]
__global__ void __launch_bounds__(256) chd_k_contact_split(const float* __restrict__ W, int K, int N, float* __restrict__ hi,
                                                           float* __restrict__ lo) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)K * N) return;
  const int n = (int)(idx / K), k = (int)(idx % K);
  const float x = W[(size_t)k * N + n], h = tc_tf32(x);
  hi[idx] = h;
  lo[idx] = tc_tf32(x - h);
}

// chd_k_contact_gather with the window value split into hi [Mp][352] and lo [Mp][352]
__global__ void __launch_bounds__(256) chd_k_contact_gather_tc(const double* __restrict__ frames, int V, int Fmax, int g0, int Mp,
                                                               float* __restrict__ A_hi, float* __restrict__ A_lo) {
  const int Wn = Fmax - (TC_WIN - 1), total = V * Wn;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)Mp * TC_K0) return;
  const int m = (int)(idx / TC_K0), k = (int)(idx % TC_K0), g = g0 + m;
  float val = 0.f;
  if (g < total && k < TC_IN) {
    const int v = g / Wn, w = g % Wn;
    const int f = k / (TC_J * 3), rem = k % (TC_J * 3), j = rem / 3, c = rem % 3;
    const int joint = c_tc_lower_joints[j];
    const double* fr = frames + (((size_t)v * Fmax + w + f) * 25 + joint) * 3;
    if (c == 2) {
      val = (float)fr[2];
    } else {
      const double root = frames[(((size_t)v * Fmax + w + TC_WIN / 2) * 25 + 8) * 3 + c];
      val = (f == TC_WIN / 2 && joint == 8) ? (float)root : (float)(fr[c] - root);
    }
  }
  const float h = tc_tf32(val);
  A_hi[idx] = h;
  A_lo[idx] = tc_tf32(val - h);
}

// C[Mp][N] = relu(bn(A[Mp][K] W^T + bias)) with A = A_hi + A_lo, W = W_hi + W_lo given as [N][K] planes through the
// tensor maps; Mp % 128 == 0, N % 128 == 0, K % 32 == 0.  C_lo != nullptr: C is written as hi / lo planes
// (C_hi, C_lo), else as plain fp32 into C_hi.
__global__ void __launch_bounds__(TC_THREADS, 1)
    chd_k_contact_gemm_tc(const __grid_constant__ CUtensorMap tA_hi, const __grid_constant__ CUtensorMap tA_lo,
                          const __grid_constant__ CUtensorMap tW_hi, const __grid_constant__ CUtensorMap tW_lo, int K, int N,
                          const float* __restrict__ bias, const float* __restrict__ scale, const float* __restrict__ mean,
                          const float* __restrict__ beta, float* __restrict__ C_hi, float* __restrict__ C_lo) {
  extern __shared__ unsigned char tc_smem[];
  __shared__ __align__(8) uint64_t bar_full[TC_STAGES], bar_empty[TC_STAGES];
  const uint32_t base = ((uint32_t)__cvta_generic_to_shared(tc_smem) + 1023u) & ~1023u;
  const uint32_t full0 = (uint32_t)__cvta_generic_to_shared(bar_full), empty0 = (uint32_t)__cvta_generic_to_shared(bar_empty);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.y * TC_BM, n0 = blockIdx.x * TC_BN, KT = K / TC_BK;
  if (threadIdx.x == 0) {
    for (int s = 0; s < TC_STAGES; ++s) {
      tc_mbar_init(full0 + 8 * s, 1);             // the producer's arrive.expect_tx
      tc_mbar_init(empty0 + 8 * s, 256);          // every consumer thread
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == 8) {                                // producer
    if (lane == 0) {
      for (int kt = 0; kt < KT; ++kt) {
        const int s = kt % TC_STAGES;
        if (kt >= TC_STAGES) tc_mbar_wait(empty0 + 8 * s, (kt / TC_STAGES - 1) & 1);
        const uint32_t st = base + s * TC_STAGE_BYTES, fb = full0 + 8 * s;
        tc_mbar_expect_tx(fb, TC_STAGE_BYTES);
        tc_tma_load(st, &tA_hi, kt * TC_BK, m0, fb);
        tc_tma_load(st + TC_TILE_BYTES, &tA_lo, kt * TC_BK, m0, fb);
        tc_tma_load(st + 2 * TC_TILE_BYTES, &tW_hi, kt * TC_BK, n0, fb);
        tc_tma_load(st + 3 * TC_TILE_BYTES, &tW_lo, kt * TC_BK, n0, fb);
      }
    }
    return;
  }
  const int wg = warp >> 2;                       // consumer warpgroup: rows 64 wg .. 64 wg + 63 of the tile
  float d[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  for (int kt = 0; kt < KT; ++kt) {
    const int s = kt % TC_STAGES;
    tc_mbar_wait(full0 + 8 * s, (kt / TC_STAGES) & 1);
    const uint32_t st = base + s * TC_STAGE_BYTES;
    const uint64_t ah = tc_desc(st + wg * (64 * 128)), al = tc_desc(st + TC_TILE_BYTES + wg * (64 * 128));
    const uint64_t bh = tc_desc(st + 2 * TC_TILE_BYTES), bl = tc_desc(st + 3 * TC_TILE_BYTES);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int kk = 0; kk < TC_BK / 8; ++kk) {      // k8 steps are 32 bytes along the swizzled row: +2 in the address field
      tc_wgmma(d, al + 2 * kk, bh + 2 * kk);
      tc_wgmma(d, ah + 2 * kk, bl + 2 * kk);
      tc_wgmma(d, ah + 2 * kk, bh + 2 * kk);
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");   // this stage's MMAs may still run; the previous one's are done
    if (kt > 0) tc_mbar_arrive(empty0 + 8 * ((kt - 1) % TC_STAGES));
  }
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
  // epilogue: bias, eval BatchNorm as (y - mean) * scale + beta, ReLU.  Accumulator fragment of m64n128: register
  // 4j + 2h + e holds row 16 (warp % 4) + lane / 4 + 8h, column 8j + 2 (lane % 4) + e.
  const int r0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int n = n0 + 8 * j + 2 * (lane & 3);
    const float2 bj = *reinterpret_cast<const float2*>(bias + n), sc = *reinterpret_cast<const float2*>(scale + n);
    const float2 mu = *reinterpret_cast<const float2*>(mean + n), be = *reinterpret_cast<const float2*>(beta + n);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const size_t o = (size_t)(r0 + 8 * h) * N + n;
      float2 y;
      y.x = fmaxf((d[4 * j + 2 * h] + bj.x - mu.x) * sc.x + be.x, 0.f);
      y.y = fmaxf((d[4 * j + 2 * h + 1] + bj.y - mu.y) * sc.y + be.y, 0.f);
      if (C_lo) {
        const float2 yh = make_float2(tc_tf32(y.x), tc_tf32(y.y));
        *reinterpret_cast<float2*>(C_hi + o) = yh;
        *reinterpret_cast<float2*>(C_lo + o) = make_float2(tc_tf32(y.x - yh.x), tc_tf32(y.y - yh.y));
      } else {
        *reinterpret_cast<float2*>(C_hi + o) = y;
      }
    }
  }
}

// ------------------------------------------------------------------ host side -------------------------------------
static const int kTcK[3] = {TC_K0, 1024, 512}, kTcN[3] = {1024, 512, 128};

// cuTensorMapEncodeTiled through the runtime's driver entry point: libchd links only libcudart.
static PFN_cuTensorMapEncodeTiled_v12000 tc_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (PFN_cuTensorMapEncodeTiled_v12000)p;
  }
  return fn;
}

// [rows][K] fp32 plane, boxes of 32 x 128 with the 128-byte swizzle wgmma's descriptors expect
static int tc_map(CUtensorMap* map, const float* plane, int rows, int K) {
  PFN_cuTensorMapEncodeTiled_v12000 enc = tc_encode_fn();
  if (!enc) {
    fprintf(stderr, "libchd: cuTensorMapEncodeTiled is not available from the driver\n");
    return -100 - (int)cudaErrorNotSupported;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)K * sizeof(float)};
  const cuuint32_t box[2] = {TC_BK, TC_BM}, estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)plane, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "libchd: cuTensorMapEncodeTiled failed (%d) for a %d x %d plane\n", (int)r, rows, K);
    return -100 - (int)r;
  }
  return 0;
}

size_t chd_contact_tc_ws_floats(int rows) { return (size_t)rows * (2 * (TC_K0 + 1024 + 512) + 128); }

int chd_contact_tc_split(const float* W, int K, int N, float* hi, float* lo, cudaStream_t s) {
  chd_k_contact_split<<<(unsigned)(((size_t)K * N + 255) / 256), 256, 0, s>>>(W, K, N, hi, lo);
  TC_CUDA(cudaGetLastError());
  return 0;
}

int chd_contact_tc_plan(const ChdContactTcNet* net, float* ws, int rows, ChdContactTcPlan* plan) {
  float* p = ws;
  for (int l = 0; l < 3; ++l) {
    plan->act_hi[l] = p, p += (size_t)rows * kTcK[l];
    plan->act_lo[l] = p, p += (size_t)rows * kTcK[l];
  }
  plan->a3 = p;
  plan->net = net;
  int rc;
  for (int l = 0; l < 3; ++l)
    if ((rc = tc_map(&plan->a_hi[l], plan->act_hi[l], rows, kTcK[l])) || (rc = tc_map(&plan->a_lo[l], plan->act_lo[l], rows, kTcK[l])) ||
        (rc = tc_map(&plan->w_hi[l], net->w_hi[l], kTcN[l], kTcK[l])) || (rc = tc_map(&plan->w_lo[l], net->w_lo[l], kTcN[l], kTcK[l])))
      return rc;
  TC_CUDA(cudaFuncSetAttribute(chd_k_contact_gemm_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
  return 0;
}

int chd_contact_tc_layers(const ChdContactTcPlan& plan, const double* frames, int V, int Fmax, int g0, int Mp, cudaStream_t s) {
  const ChdContactTcNet& n = *plan.net;
  chd_k_contact_gather_tc<<<(unsigned)(((size_t)Mp * TC_K0 + 255) / 256), 256, 0, s>>>(frames, V, Fmax, g0, Mp, plan.act_hi[0], plan.act_lo[0]);
  for (int l = 0; l < 3; ++l)
    chd_k_contact_gemm_tc<<<dim3(kTcN[l] / TC_BN, Mp / TC_BM), TC_THREADS, TC_SMEM, s>>>(
        plan.a_hi[l], plan.a_lo[l], plan.w_hi[l], plan.w_lo[l], kTcK[l], kTcN[l], n.bias[l], n.scale[l], n.mean[l], n.beta[l],
        l < 2 ? plan.act_hi[l + 1] : plan.a3, l < 2 ? plan.act_lo[l + 1] : nullptr);
  TC_CUDA(cudaGetLastError());
  return 0;
}
