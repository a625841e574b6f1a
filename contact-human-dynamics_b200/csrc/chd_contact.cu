// Foot-contact classifier of contact-human-dynamics on sm_90a (product code).
//
// Replaces, for inference, src/contact_learning/test.py:51-152 (val_full_video) +
// src/contact_learning/models/openpose_only.py:29-78 + the window construction of
// src/contact_learning/data/real_video_dataset.py:206-276:
//   chd_k_contact_gather : the 9-frame x 13-joint x (x,y,conf) windows straight from the per-frame keypoints
//                          (root-relative as the dataset does it, fp64 subtraction then fp32)
//   chd_k_contact_gemm   : one Linear + eval BatchNorm + ReLU layer over a slab of windows, 128x128x16 tiles,
//                          8x8 outputs per thread, double-buffered shared-memory tiles (layers 351-1024-512-128)
//   chd_k_contact_tail   : the two small layers 128-32-20
//   chd_k_contact_vote   : sigmoid > 0.5, 5-vote aggregation, edge thresholds, 2-frame padding, int64 labels
// Windows are processed in slabs of 16384 (activations of a slab: 132 MB, in HBM rather than shared memory; a slab
// small enough for the 50 MB L2 would leave the 128-wide layer with fewer tiles than SMs); every output is one fp32
// accumulator summed over k in ascending order (fmaf), the same arithmetic as a plain loop.  fp32 FFMA, no tf32/bf16:
// the integer labels must match the reference's fp32 forward away from the logit-0 boundary (SURVEY 8(a)-D note;
// wgmma has no fp32-input kind).  The opt-in 3xTF32 tensor-core mode of the three large layers (CHD_CONTACT_TF32X3)
// is in chd_contact_tc.cu; this file's kernels are the default FP32 mode.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../include/chd.h"
#include "chd_contact_tc.h"

#define CT_WIN 9
#define CT_PRED 5
#define CT_J 13
#define CT_IN 351
#define CT_K0 352        // first layer's K padded to the tile depth
#define CT_SLAB 16384    // windows per slab
#define GM 128
#define GN 128
#define GK 16

static __device__ __constant__ int c_lower_joints[CT_J] = {8, 9, 10, 11, 12, 13, 14, 19, 20, 21, 22, 23, 24};  // openpose_dataset.py:38

struct ContactDev {
  const float* W[5];   // [in][out] (transposed on the host; layer 0 has CT_K0 rows, the last one zero)
  const float* b[5];
  const float* bn_scale[4];  // gamma / sqrt(var + eps)
  const float* bn_mean[4];
  const float* bn_beta[4];
};

// frames: [V][Fmax][25][3] fp64 (scaled, gap-interpolated, normalised keypoints) -> A0 [Mp][CT_K0] fp32 for the
// windows g0 .. g0+Mp-1 (rows past the last window and column 351 are zero), real_video_dataset.py:240-252
__global__ void __launch_bounds__(256) chd_k_contact_gather(const double* __restrict__ frames, int V, int Fmax, int g0, int Mp,
                                                            float* __restrict__ A0) {
  const int Wn = Fmax - (CT_WIN - 1), total = V * Wn;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)Mp * CT_K0) return;
  const int m = (int)(idx / CT_K0), k = (int)(idx % CT_K0), g = g0 + m;
  float val = 0.f;
  if (g < total && k < CT_IN) {
    const int v = g / Wn, w = g % Wn;
    const int f = k / (CT_J * 3), rem = k % (CT_J * 3), j = rem / 3, c = rem % 3;
    const int joint = c_lower_joints[j];
    const double* fr = frames + (((size_t)v * Fmax + w + f) * 25 + joint) * 3;
    if (c == 2) {
      val = (float)fr[2];
    } else {
      const double root = frames[(((size_t)v * Fmax + w + CT_WIN / 2) * 25 + 8) * 3 + c];
      val = (f == CT_WIN / 2 && joint == 8) ? (float)root : (float)(fr[c] - root);
    }
  }
  A0[idx] = val;
}

// C[Mp][N] = relu(bn(A[Mp][K] W[K][N] + bias)); Mp % 128 == 0, N % 128 == 0, K % 16 == 0.
// 256 threads; thread (ty, tx) owns rows {4ty..4ty+3, 64+4ty..} x columns {4tx..4tx+3, 64+4tx..}.
__global__ void __launch_bounds__(256) chd_k_contact_gemm(const float* __restrict__ A, const float* __restrict__ W, int K, int N,
                                                          const float* __restrict__ bias, const float* __restrict__ scale,
                                                          const float* __restrict__ mean, const float* __restrict__ beta,
                                                          float* __restrict__ C) {
  __shared__ __align__(16) float As[2][GK][GM];   // transposed A tile
  __shared__ __align__(16) float Bs[2][GK][GN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * GM, n0 = blockIdx.x * GN;
  // global -> register staging: A tile 128 x 16 = 512 float4 (2 per thread), B tile 16 x 128 = 512 float4
  const int ar = tid >> 2, ac = (tid & 3) * 4;          // A rows ar, ar + 64; k offset ac
  const int br = tid >> 5, bc = (tid & 31) * 4;         // B rows br, br + 8; column offset bc
  const float* Ap = A + (size_t)(m0 + ar) * K + ac;
  const float* Bp = W + (size_t)br * N + n0 + bc;
  float4 ra0, ra1, rb0, rb1;
  auto gload = [&](int k0) {
    ra0 = *reinterpret_cast<const float4*>(Ap + k0);
    ra1 = *reinterpret_cast<const float4*>(Ap + (size_t)64 * K + k0);
    rb0 = __ldg(reinterpret_cast<const float4*>(Bp + (size_t)k0 * N));
    rb1 = __ldg(reinterpret_cast<const float4*>(Bp + (size_t)(k0 + 8) * N));
  };
  auto sstore = [&](int buf) {
    As[buf][ac + 0][ar] = ra0.x, As[buf][ac + 1][ar] = ra0.y, As[buf][ac + 2][ar] = ra0.z, As[buf][ac + 3][ar] = ra0.w;
    As[buf][ac + 0][ar + 64] = ra1.x, As[buf][ac + 1][ar + 64] = ra1.y, As[buf][ac + 2][ar + 64] = ra1.z, As[buf][ac + 3][ar + 64] = ra1.w;
    *reinterpret_cast<float4*>(&Bs[buf][br][bc]) = rb0;
    *reinterpret_cast<float4*>(&Bs[buf][br + 8][bc]) = rb1;
  };
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  gload(0);
  sstore(0);
  __syncthreads();
  int buf = 0;
  for (int k0 = 0; k0 < K; k0 += GK, buf ^= 1) {
    const bool more = k0 + GK < K;
    if (more) gload(k0 + GK);
#pragma unroll
    for (int kk = 0; kk < GK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (more) sstore(buf ^ 1);
    __syncthreads();
  }
  // epilogue: bias, eval BatchNorm as (y - mean) * scale + beta, ReLU
#pragma unroll
  for (int jh = 0; jh < 2; ++jh) {
    const int n = n0 + jh * 64 + tx * 4;
    const float4 bj = *reinterpret_cast<const float4*>(bias + n), sc = *reinterpret_cast<const float4*>(scale + n);
    const float4 mu = *reinterpret_cast<const float4*>(mean + n), be = *reinterpret_cast<const float4*>(beta + n);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int m = m0 + (i >> 2) * 64 + ty * 4 + (i & 3);
      float4 y;
      y.x = fmaxf((acc[i][jh * 4 + 0] + bj.x - mu.x) * sc.x + be.x, 0.f);
      y.y = fmaxf((acc[i][jh * 4 + 1] + bj.y - mu.y) * sc.y + be.y, 0.f);
      y.z = fmaxf((acc[i][jh * 4 + 2] + bj.z - mu.z) * sc.z + be.z, 0.f);
      y.w = fmaxf((acc[i][jh * 4 + 3] + bj.w - mu.w) * sc.w + be.w, 0.f);
      *reinterpret_cast<float4*>(C + (size_t)m * N + n) = y;
    }
  }
}

// layers 128 -> 32 (BN + ReLU) -> 20 for 32 windows per CTA; logits [total][20]
__global__ void __launch_bounds__(256) chd_k_contact_tail(ContactDev net, const float* __restrict__ A3, int g0, int total,
                                                          float* __restrict__ logits) {
  __shared__ float sA[32][129];
  __shared__ float sW3[128 * 32];
  __shared__ float sH[32][33];
  __shared__ float sW4[32 * 20];
  const int tid = threadIdx.x, m0 = blockIdx.x * 32;
  for (int i = tid; i < 32 * 128; i += 256) sA[i >> 7][i & 127] = A3[(size_t)(m0 + (i >> 7)) * 128 + (i & 127)];
  for (int i = tid; i < 128 * 32; i += 256) sW3[i] = net.W[3][i];
  for (int i = tid; i < 32 * 20; i += 256) sW4[i] = net.W[4][i];
  __syncthreads();
  {
    const int n = tid & 31;
    const float bj = net.b[3][n], sc = net.bn_scale[3][n], mu = net.bn_mean[3][n], be = net.bn_beta[3][n];
    for (int m = tid >> 5; m < 32; m += 8) {
      float acc = 0.f;
#pragma unroll 8
      for (int k = 0; k < 128; ++k) acc = fmaf(sA[m][k], sW3[k * 32 + n], acc);
      sH[m][n] = fmaxf((acc + bj - mu) * sc + be, 0.f);
    }
  }
  __syncthreads();
  for (int i = tid; i < 32 * 20; i += 256) {
    const int m = i / 20, n = i % 20, g = g0 + m0 + m;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) acc = fmaf(sH[m][k], sW4[k * 20 + n], acc);
    if (g < total) logits[(size_t)g * 20 + n] = acc + net.b[4][n];
  }
}

// The 0.5 vote of frame f, contact c of one video whose window logits are lg [Fmax-8][20] (test.py:88-122); the one
// rule behind the labels of chd_k_contact_vote and the merged counts of chd_k_contact_score.  mabs, when given, takes
// the min of the |logit| of every prediction that entered the vote.
static __device__ __forceinline__ bool ct_vote(const float* __restrict__ lg, int Fmax, int f, int c, float* mabs = nullptr) {
  const int Wn = Fmax - (CT_WIN - 1), nv = Wn + 2 * (CT_PRED / 2);   // frames that receive votes
  const int off = (CT_WIN - CT_PRED) / 2;                            // copies padded on each side
  int fv = f - off;                        // index into the voted array, clamped = repeat first/last row
  fv = fv < 0 ? 0 : (fv >= nv ? nv - 1 : fv);
  int votes = 0;
  for (int p = 0; p < CT_PRED; ++p) {      // window w = fv - p contributes its prediction for offset p
    const int w = fv - p;
    if (w < 0 || w >= Wn) continue;
    const float x = lg[w * 20 + p * 4 + c];
    const float prob = 1.0f / (1.0f + expf(-x));   // openpose_only.py:75-78: sigmoid(x) > 0.5
    votes += prob > 0.5f ? 1 : 0;
    if (mabs) *mabs = fminf(*mabs, fabsf(x));
  }
  int thresh = (CT_PRED + 1) / 2;          // test.py:101-104
  const int e0 = fv, e1 = nv - 1 - fv;
  if (e0 < CT_PRED - 1) thresh = e0 / 2 + 1;
  if (e1 < CT_PRED - 1) thresh = e1 / 2 + 1;
  return votes >= thresh;
}

// labels [V][Fmax][4] int64; rows >= seq_len are zeroed (the reference trims them, test.py:149-152)
__global__ void chd_k_contact_vote(const float* __restrict__ logits, int V, int Fmax, const int* __restrict__ seq_lens,
                                   long long* __restrict__ labels, float* __restrict__ min_abs) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  float mabs = 3.4e38f;
  if (idx < V * Fmax * 4) {
    const int c = idx & 3, f = (idx >> 2) % Fmax, v = (idx >> 2) / Fmax;
    const bool vote = ct_vote(logits + (size_t)v * (Fmax - (CT_WIN - 1)) * 20, Fmax, f, c, &mabs);
    labels[idx] = f < seq_lens[v] ? (vote ? 1 : 0) : 0;
  }
  // block min of |logit|
  for (int o = 16; o > 0; o >>= 1) mabs = fminf(mabs, __shfl_xor_sync(0xffffffffu, mabs, o));
  if ((threadIdx.x & 31) == 0 && mabs < 3.0e38f) atomicMin(reinterpret_cast<int*>(min_abs), __float_as_int(mabs));  // positive floats order as ints
}

// Scores the logits of every window against ground-truth contacts (test.py:64-140 val_full_video with labels: the
// OpenPoseModel.loss / .accuracy calls and the merged-label count).  One CTA per video, CT_SCORE_THREADS threads; a
// multiple of 20 and of 4, so a thread always sees the same (predicted frame, contact) pair in the window pass and the
// same contact in the frame pass and keeps four counters.  Video v's truth rows are truth[toffs[v] .. toffs[v+1]), padded
// with their last row or trimmed to Fmax (fix_data_len, real_video_dataset.py:165-191); a video without rows gets zeros.
//   loss_sum[v]          sum over windows x 5 x 4 of BCE-with-logits (1 - y) x - log_sigmoid(x), fp32 terms, fp64 sum
//   conf_frames[v][p][.] (tp, fp, fn, tn) of sigmoid(x) > thresh against truth row w + 2 + p of window w
//   conf_merged[v][.]    (tp, fp, fn, tn) over all Fmax x 4 of the 0.5 vote before trimming (ct_vote again: the vote
//                        kernel zeroes rows >= seq_len) against truth row clamp(f, 2, Fmax - 3), test.py:124-140
// Fixed-order reductions, no atomics: a video's outputs depend only on its own logits, truth and Fmax.
#define CT_SCORE_THREADS 320
__global__ void __launch_bounds__(CT_SCORE_THREADS) chd_k_contact_score(const float* __restrict__ logits, int Fmax, const int* __restrict__ truth,
                                                                       const int* __restrict__ toffs, float thresh, double* __restrict__ loss_sum,
                                                                       long long* __restrict__ conf_frames, long long* __restrict__ conf_merged) {
  __shared__ int s_cnt[CT_SCORE_THREADS][4];
  __shared__ double s_loss[CT_SCORE_THREADS / 32];
  const int v = blockIdx.x, tid = threadIdx.x;
  const int Wn = Fmax - (CT_WIN - 1), off = (CT_WIN - CT_PRED) / 2;
  const int t0 = toffs[v], nrow = toffs[v + 1] - t0;
  const float* lg = logits + (size_t)v * Wn * 20;
  auto label = [&](int r, int c) { return truth[(size_t)(t0 + (r < nrow ? r : nrow - 1)) * 4 + c] != 0; };
  // ---- per window: loss and per-frame counts; this thread's (p, c) = (tid % 20) / 4, tid % 4 ----
  int cnt[4] = {0, 0, 0, 0};
  double loss = 0.0;
  if (nrow > 0) {
    const int p = (tid % 20) / 4, c = tid % 4;
    for (int i = tid; i < Wn * 20; i += CT_SCORE_THREADS) {
      const float x = lg[i];
      const bool y = label(i / 20 + off + p, c);
      const float log_sig = fminf(x, 0.f) - log1pf(expf(-fabsf(x)));        // torch's log_sigmoid
      loss += (double)((y ? 0.f : x) - log_sig);                               // (1 - y) * x - log_sigmoid(x)
      const bool pred = 1.0f / (1.0f + expf(-x)) > thresh;                     // the vote kernel's predicate
      ++cnt[pred ? (y ? 0 : 1) : (y ? 2 : 3)];
    }
  }
  for (int q = 0; q < 4; ++q) s_cnt[tid][q] = cnt[q];
  for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
  if ((tid & 31) == 0) s_loss[tid >> 5] = loss;
  __syncthreads();
  if (tid < CT_PRED * 4) {    // tid = (p, q): sum over the contacts c and the threads c + 4p, c + 4p + 20, ...
    const int p = tid / 4, q = tid % 4;
    long long sum = 0;
    for (int c = 0; c < 4; ++c)
      for (int t = p * 4 + c; t < CT_SCORE_THREADS; t += 20) sum += s_cnt[t][q];
    conf_frames[(size_t)v * 20 + tid] = sum;
  }
  if (tid == 0) {
    double s = 0.0;
    for (int w = 0; w < CT_SCORE_THREADS / 32; ++w) s += s_loss[w];
    loss_sum[v] = s;
  }
  __syncthreads();
  // ---- per frame: merged counts ----
  int mc[4] = {0, 0, 0, 0};
  if (nrow > 0) {
    for (int i = tid; i < Fmax * 4; i += CT_SCORE_THREADS) {
      const int c = i & 3, f = i >> 2;
      const bool pred = ct_vote(lg, Fmax, f, c);
      const bool y = label(f < off ? off : (f > Fmax - 1 - off ? Fmax - 1 - off : f), c);
      ++mc[pred ? (y ? 0 : 1) : (y ? 2 : 3)];
    }
  }
  for (int q = 0; q < 4; ++q) s_cnt[tid][q] = mc[q];
  __syncthreads();
  if (tid < 4) {              // count q over all threads (every contact)
    long long sum = 0;
    for (int t = 0; t < CT_SCORE_THREADS; ++t) sum += s_cnt[t][tid];
    conf_merged[(size_t)v * 4 + tid] = sum;
  }
}

// Grow-only device buffers (ct_reserve): the host entry points' buffers and the slab workspaces of the two modes,
// IO_WS = A0 [rows][352] | A1 [rows][1024] | A2 [rows][512] | A3 [rows][128] of the FP32 kernels and IO_TC_WS = the
// tensor-core layers' planes (chd_contact_tc_ws_floats).
enum { IO_FRAMES, IO_LENS, IO_LABELS, IO_LOGITS, IO_MIN, IO_RAW, IO_OFFS, IO_PACKED, IO_TRUTH, IO_TOFFS, IO_SCORE, IO_WS, IO_TC_WS, IO_COUNT };

struct chd_contact_net {
  std::vector<void*> allocs;
  ContactDev dev;
  cudaStream_t stream = nullptr;
  int64_t launches = 0;
  // no allocation per call, nothing to leak on an error path
  void* io[IO_COUNT] = {};
  size_t io_bytes[IO_COUNT] = {};
  // CHD_CONTACT_TF32X3: split weight planes (one allocation)
  int precision = CHD_CONTACT_FP32;
  ChdContactTcNet tc = {};
  float* tc_w = nullptr;
};

#define CT_CUDA(x)                                                                           \
  do {                                                                                       \
    cudaError_t e_ = (x);                                                                    \
    if (e_ != cudaSuccess) {                                                                 \
      fprintf(stderr, "libchd: CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      return -100 - (int)e_;                                                                 \
    }                                                                                        \
  } while (0)

// ------------------------------------------------------------------ keypoint preprocessing -----------------------
// RealVideoDataset.__init__ (real_video_dataset.py:132-163) + process_openpose_data (openpose_dataset.py:49-121) on the
// device: one thread per (video, joint) walks the frames of its joint.  raw: concatenated (sum F, 25, 3) [x, y, conf]
// of the OpenPose json files, offs: V+1 frame offsets.  out: (V, Fmax, 25, 3) -- videos padded to the longest one
// by repeating their last frame, xy scaled by 1280 / width, low-confidence (< thresh) runs of a joint replaced (leading /
// trailing runs: nearest valid frame; interior runs: linear interpolation whose weight accumulates `cur += step` like the
// reference loop), xy divided by the training normalisation.  Same fp64 operation order as the numpy reference
// (explicit round-to-nearest multiplies / adds: no FMA contraction), so the result is bit identical.
__global__ void chd_k_contact_prep(const double* __restrict__ raw, const int* __restrict__ offs, int V, int Fmax, double scale,
                                   double norm, double thresh, double* __restrict__ out, int* __restrict__ seq_lens) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= V * 25) return;
  const int v = idx / 25, j = idx % 25;
  const int f0 = offs[v], len = offs[v + 1] - f0;
  if (j == 0) seq_lens[v] = len;
  auto src = [&](int t, int c) { return raw[((size_t)(f0 + (t < len ? t : len - 1)) * 25 + j) * 3 + c]; };
  auto X = [&](int t, int c) { return __dmul_rn(src(t, c), scale); };   // a[:, :, :2] *= scale
  double* o = out + ((size_t)v * Fmax * 25 + j) * 3;
  const size_t fs = 25 * 3;
  int t = 0;
  while (t < Fmax) {
    if (src(t, 2) < thresh) {
      int nxt = t + 1;
      while (nxt < Fmax && src(nxt, 2) < thresh) ++nxt;
      const int init = t - 1;
      for (int ct = t; ct < nxt; ++ct) {
        double x, y;
        if (t == 0 && nxt == Fmax) x = X(ct, 0), y = X(ct, 1);                    // never seen with confidence: left alone
        else if (t == 0) x = X(nxt, 0), y = X(nxt, 1);                          // leading run: first valid frame
        else if (nxt == Fmax) x = X(init, 0), y = X(init, 1);                   // trailing run: last valid frame
        else {
          const double step = 1.0 / (nxt - init);
          double cur = step;
          for (int q = t; q < ct; ++q) cur += step;                             // accumulated exactly like the reference loop
          const double w0 = 1.0 - cur;
          x = __dadd_rn(__dmul_rn(w0, X(init, 0)), __dmul_rn(cur, X(nxt, 0)));
          y = __dadd_rn(__dmul_rn(w0, X(init, 1)), __dmul_rn(cur, X(nxt, 1)));
        }
        o[(size_t)ct * fs + 0] = x / norm, o[(size_t)ct * fs + 1] = y / norm, o[(size_t)ct * fs + 2] = src(ct, 2);
      }
      t = nxt;
    } else {
      o[(size_t)t * fs + 0] = X(t, 0) / norm, o[(size_t)t * fs + 1] = X(t, 1) / norm, o[(size_t)t * fs + 2] = src(t, 2);
      ++t;
    }
  }
}
// (V, Fmax, 4) labels -> concatenated (sum F, 4), the rows foot_contacts.npy keeps (test.py:149-152)
__global__ void chd_k_contact_pack(const long long* __restrict__ lab, const int* __restrict__ offs, int V, int Fmax, long long* __restrict__ out) {
  const int v = blockIdx.y;
  const int f0 = offs[v], len = offs[v + 1] - f0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < len * 4; i += gridDim.x * blockDim.x) out[(size_t)f0 * 4 + i] = lab[(size_t)v * Fmax * 4 + i];
}

static int ct_reserve(chd_contact_net* net, int slot, size_t bytes) {
  if (bytes <= net->io_bytes[slot]) return 0;
  if (net->io[slot]) cudaFree(net->io[slot]);
  net->io[slot] = nullptr, net->io_bytes[slot] = 0;
  cudaError_t e = cudaMalloc(&net->io[slot], bytes);
  if (e != cudaSuccess) {
    fprintf(stderr, "libchd: CUDA error %s (contact io buffer %d, %zu bytes)\n", cudaGetErrorString(e), slot, bytes);
    return -100 - (int)e;
  }
  net->io_bytes[slot] = bytes;
  return 0;
}

extern "C" {

int chd_contact_create(const float* weights, const float* biases, const float* bn, float bn_eps, int32_t device, chd_contact_net** out) {
  if (!weights || !biases || !bn || !out) return -1;
  if (device >= 0) CT_CUDA(cudaSetDevice(device));
  const int dims[6] = {CT_IN, 1024, 512, 128, 32, 20};
  chd_contact_net* net = new chd_contact_net();
  CT_CUDA(cudaStreamCreate(&net->stream));
  auto up = [&](const std::vector<float>& h, const float** d) -> int {
    void* p = nullptr;
    CT_CUDA(cudaMalloc(&p, h.size() * sizeof(float)));
    net->allocs.push_back(p);
    CT_CUDA(cudaMemcpy(p, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
    *d = (const float*)p;
    return 0;
  };
  const float* w = weights;
  const float* b = biases;
  const float* q = bn;
  for (int l = 0; l < 5; ++l) {
    const int in = dims[l], o = dims[l + 1];
    std::vector<float> wt((size_t)(l == 0 ? CT_K0 : in) * o, 0.f), bb(b, b + o);
    for (int i = 0; i < o; ++i)
      for (int k = 0; k < in; ++k) wt[(size_t)k * o + i] = w[(size_t)i * in + k];   // torch [out][in] -> [in][out]
    int rc;
    if ((rc = up(wt, &net->dev.W[l])) || (rc = up(bb, &net->dev.b[l]))) return rc;
    w += (size_t)in * o;
    b += o;
    if (l < 4) {
      std::vector<float> sc(o), mu(o), be(o);
      for (int i = 0; i < o; ++i) {
        const float gamma = q[i], beta = q[o + i], mean = q[2 * o + i], var = q[3 * o + i];
        sc[i] = gamma / sqrtf(var + bn_eps);
        mu[i] = mean;
        be[i] = beta;
      }
      if ((rc = up(sc, &net->dev.bn_scale[l])) || (rc = up(mu, &net->dev.bn_mean[l])) || (rc = up(be, &net->dev.bn_beta[l]))) return rc;
      q += 4 * o;
    }
  }
  *out = net;
  return 0;
}

void chd_contact_destroy(chd_contact_net* net) {
  if (!net) return;
  for (void* p : net->allocs) cudaFree(p);
  if (net->tc_w) cudaFree(net->tc_w);
  for (int q = 0; q < IO_COUNT; ++q)
    if (net->io[q]) cudaFree(net->io[q]);
  if (net->stream) cudaStreamDestroy(net->stream);
  delete net;
}

int chd_contact_forward_device(chd_contact_net* net, const double* frames_dev, int32_t V, int32_t Fmax, const int32_t* seq_lens_dev,
                               int64_t* labels_dev, float* logits_dev, float* min_abs_dev, void* stream) {
  if (!net || !frames_dev || !seq_lens_dev || !labels_dev || !logits_dev || !min_abs_dev || Fmax < CT_WIN) return -1;   // all device buffers are required
  cudaStream_t s = stream ? (cudaStream_t)stream : net->stream;
  const int Wn = Fmax - (CT_WIN - 1), total = V * Wn;
  const float big = 3.4e38f;
  CT_CUDA(cudaMemcpyAsync(min_abs_dev, &big, sizeof(float), cudaMemcpyHostToDevice, s));
  const int rows = std::min(CT_SLAB, (total + GM - 1) / GM * GM);
  const ContactDev& d = net->dev;
  int rc;
  if (net->precision == CHD_CONTACT_TF32X3) {
    // per slab: split gather, three tensor-core layers, FFMA tail (chd_contact_tc.cu)
    ChdContactTcPlan plan;
    if ((rc = ct_reserve(net, IO_TC_WS, chd_contact_tc_ws_floats(rows) * sizeof(float))) ||
        (rc = chd_contact_tc_plan(&net->tc, (float*)net->io[IO_TC_WS], rows, &plan)))
      return rc;
    for (int g0 = 0; g0 < total; g0 += CT_SLAB) {
      const int Mp = (std::min(CT_SLAB, total - g0) + GM - 1) / GM * GM;
      if ((rc = chd_contact_tc_layers(plan, frames_dev, V, Fmax, g0, Mp, s))) return rc;
      chd_k_contact_tail<<<Mp / 32, 256, 0, s>>>(d, plan.a3, g0, total, logits_dev);
      net->launches += 5;
    }
  } else {
    if ((rc = ct_reserve(net, IO_WS, (size_t)rows * (CT_K0 + 1024 + 512 + 128) * sizeof(float)))) return rc;
    float* A0 = (float*)net->io[IO_WS];
    float* A1 = A0 + (size_t)rows * CT_K0;
    float* A2 = A1 + (size_t)rows * 1024;
    float* A3 = A2 + (size_t)rows * 512;
    for (int g0 = 0; g0 < total; g0 += CT_SLAB) {
      const int Mp = (std::min(CT_SLAB, total - g0) + GM - 1) / GM * GM;
      chd_k_contact_gather<<<(unsigned)(((size_t)Mp * CT_K0 + 255) / 256), 256, 0, s>>>(frames_dev, V, Fmax, g0, Mp, A0);
      chd_k_contact_gemm<<<dim3(1024 / GN, Mp / GM), 256, 0, s>>>(A0, d.W[0], CT_K0, 1024, d.b[0], d.bn_scale[0], d.bn_mean[0], d.bn_beta[0], A1);
      chd_k_contact_gemm<<<dim3(512 / GN, Mp / GM), 256, 0, s>>>(A1, d.W[1], 1024, 512, d.b[1], d.bn_scale[1], d.bn_mean[1], d.bn_beta[1], A2);
      chd_k_contact_gemm<<<dim3(128 / GN, Mp / GM), 256, 0, s>>>(A2, d.W[2], 512, 128, d.b[2], d.bn_scale[2], d.bn_mean[2], d.bn_beta[2], A3);
      chd_k_contact_tail<<<Mp / 32, 256, 0, s>>>(d, A3, g0, total, logits_dev);
      net->launches += 5;
    }
  }
  chd_k_contact_vote<<<(V * Fmax * 4 + 255) / 256, 256, 0, s>>>(logits_dev, V, Fmax, seq_lens_dev, (long long*)labels_dev, min_abs_dev);
  net->launches += 1;
  CT_CUDA(cudaGetLastError());
  return 0;
}

int chd_contact_forward(chd_contact_net* net, const double* frames, int32_t V, int32_t Fmax, const int32_t* seq_lens, int64_t* labels,
                        float* logits, float* min_abs_logit) {
  if (!net || !frames || !seq_lens || !labels || V <= 0 || Fmax < CT_WIN) return -1;
  const size_t nfr = (size_t)V * Fmax * 75, Wn = Fmax - (CT_WIN - 1), nlog = (size_t)V * Wn * 20, nlab = (size_t)V * Fmax * 4;
  int rc;
  if ((rc = ct_reserve(net, IO_FRAMES, nfr * sizeof(double))) || (rc = ct_reserve(net, IO_LENS, V * sizeof(int))) ||
      (rc = ct_reserve(net, IO_LABELS, nlab * sizeof(long long))) || (rc = ct_reserve(net, IO_LOGITS, nlog * sizeof(float))) ||
      (rc = ct_reserve(net, IO_MIN, sizeof(float))))
    return rc;
  double* d_fr = (double*)net->io[IO_FRAMES];
  int* d_len = (int*)net->io[IO_LENS];
  long long* d_lab = (long long*)net->io[IO_LABELS];
  float *d_log = (float*)net->io[IO_LOGITS], *d_min = (float*)net->io[IO_MIN];
  CT_CUDA(cudaMemcpyAsync(d_fr, frames, nfr * sizeof(double), cudaMemcpyHostToDevice, net->stream));
  CT_CUDA(cudaMemcpyAsync(d_len, seq_lens, V * sizeof(int), cudaMemcpyHostToDevice, net->stream));
  rc = chd_contact_forward_device(net, d_fr, V, Fmax, d_len, (int64_t*)d_lab, d_log, d_min, net->stream);
  if (rc) return rc;
  CT_CUDA(cudaMemcpyAsync(labels, d_lab, nlab * sizeof(long long), cudaMemcpyDeviceToHost, net->stream));
  if (logits) CT_CUDA(cudaMemcpyAsync(logits, d_log, nlog * sizeof(float), cudaMemcpyDeviceToHost, net->stream));
  if (min_abs_logit) CT_CUDA(cudaMemcpyAsync(min_abs_logit, d_min, sizeof(float), cudaMemcpyDeviceToHost, net->stream));
  CT_CUDA(cudaStreamSynchronize(net->stream));
  return 0;
}

// raw OpenPose keypoints -> preprocessed frames on the device (shared by chd_contact_preprocess / _detect):
// xy multiplied by `scale`, gaps interpolated, xy divided by `norm`
static int ct_prep_device(chd_contact_net* net, const double* raw, const int32_t* offs, int32_t V, double scale, double norm, int* Fmax_out) {
  int Fmax = 0, total = offs[V];
  for (int v = 0; v < V; ++v) {
    if (offs[v + 1] <= offs[v]) return -1;
    Fmax = std::max(Fmax, offs[v + 1] - offs[v]);
  }
  if (Fmax < CT_WIN) return -1;
  int rc;
  if ((rc = ct_reserve(net, IO_RAW, (size_t)total * 75 * sizeof(double))) || (rc = ct_reserve(net, IO_OFFS, (V + 1) * sizeof(int))) ||
      (rc = ct_reserve(net, IO_FRAMES, (size_t)V * Fmax * 75 * sizeof(double))) || (rc = ct_reserve(net, IO_LENS, V * sizeof(int))))
    return rc;
  CT_CUDA(cudaMemcpyAsync(net->io[IO_RAW], raw, (size_t)total * 75 * sizeof(double), cudaMemcpyHostToDevice, net->stream));
  CT_CUDA(cudaMemcpyAsync(net->io[IO_OFFS], offs, (V + 1) * sizeof(int), cudaMemcpyHostToDevice, net->stream));
  chd_k_contact_prep<<<(V * 25 + 127) / 128, 128, 0, net->stream>>>((const double*)net->io[IO_RAW], (const int*)net->io[IO_OFFS], V, Fmax, scale,
                                                                    norm, 0.2, (double*)net->io[IO_FRAMES], (int*)net->io[IO_LENS]);
  net->launches += 1;
  CT_CUDA(cudaGetLastError());
  *Fmax_out = Fmax;
  return 0;
}

int chd_contact_preprocess(chd_contact_net* net, const double* raw, const int32_t* seq_offsets, int32_t V, double scale, double norm,
                           double* frames_out, int32_t* seq_lens_out) {
  if (!net || !raw || !seq_offsets || V <= 0 || !(scale > 0) || !(norm > 0) || !frames_out) return -1;
  int Fmax = 0;
  int rc = ct_prep_device(net, raw, seq_offsets, V, scale, norm, &Fmax);
  if (rc) return rc;
  CT_CUDA(cudaMemcpyAsync(frames_out, net->io[IO_FRAMES], (size_t)V * Fmax * 75 * sizeof(double), cudaMemcpyDeviceToHost, net->stream));
  if (seq_lens_out) CT_CUDA(cudaMemcpyAsync(seq_lens_out, net->io[IO_LENS], V * sizeof(int), cudaMemcpyDeviceToHost, net->stream));
  CT_CUDA(cudaStreamSynchronize(net->stream));
  return 0;
}

int chd_contact_score_device(chd_contact_net* net, const float* logits_dev, int32_t V, int32_t Fmax, const int32_t* truth_dev,
                             const int32_t* truth_offsets_dev, float classify_thresh, double* loss_sum_dev, int64_t* conf_frames_dev,
                             int64_t* conf_merged_dev, void* stream) {
  if (!net || !logits_dev || !truth_offsets_dev || !loss_sum_dev || !conf_frames_dev || !conf_merged_dev || V <= 0 || Fmax < CT_WIN) return -1;
  cudaStream_t s = stream ? (cudaStream_t)stream : net->stream;
  chd_k_contact_score<<<V, CT_SCORE_THREADS, 0, s>>>(logits_dev, Fmax, truth_dev, truth_offsets_dev, classify_thresh, loss_sum_dev,
                                                     (long long*)conf_frames_dev, (long long*)conf_merged_dev);
  net->launches += 1;
  CT_CUDA(cudaGetLastError());
  return 0;
}

int chd_contact_detect(chd_contact_net* net, const double* raw, const int32_t* seq_offsets, int32_t V, double scale, double norm,
                       const int32_t* truth, const int32_t* truth_offsets, float classify_thresh, int64_t* labels_out, double* loss_sum,
                       int64_t* conf_frames, int64_t* conf_merged, float* min_abs_logit) {
  if (!net || !raw || !seq_offsets || V <= 0 || !(scale > 0) || !(norm > 0) || !labels_out) return -1;
  const bool scored = truth_offsets != nullptr;
  double* d_loss = nullptr;          // IO_SCORE: loss_sum [V] | conf_frames [V][20] | conf_merged [V][4]
  int64_t *d_frames = nullptr, *d_merged = nullptr;
  int rc;
  if (scored) {
    if (!loss_sum || !conf_frames || !conf_merged || truth_offsets[0] != 0) return -1;
    for (int v = 0; v < V; ++v)
      if (truth_offsets[v + 1] < truth_offsets[v]) return -1;
    const size_t nrows = truth_offsets[V];
    if (nrows > 0 && !truth) return -1;
    // the truth goes up first: the prep / forward reservations below do not touch these slots
    if ((rc = ct_reserve(net, IO_TRUTH, std::max<size_t>(nrows, 1) * 4 * sizeof(int))) || (rc = ct_reserve(net, IO_TOFFS, (V + 1) * sizeof(int))) ||
        (rc = ct_reserve(net, IO_SCORE, (size_t)V * (1 + 20 + 4) * 8)))
      return rc;
    d_loss = (double*)net->io[IO_SCORE], d_frames = (int64_t*)(d_loss + V), d_merged = d_frames + (size_t)V * 20;
    if (nrows) CT_CUDA(cudaMemcpyAsync(net->io[IO_TRUTH], truth, nrows * 4 * sizeof(int), cudaMemcpyHostToDevice, net->stream));
    CT_CUDA(cudaMemcpyAsync(net->io[IO_TOFFS], truth_offsets, (V + 1) * sizeof(int), cudaMemcpyHostToDevice, net->stream));
  }
  int Fmax = 0;
  if ((rc = ct_prep_device(net, raw, seq_offsets, V, scale, norm, &Fmax))) return rc;
  const size_t total = seq_offsets[V], Wn = Fmax - (CT_WIN - 1), nlog = (size_t)V * Wn * 20, nlab = (size_t)V * Fmax * 4;
  if ((rc = ct_reserve(net, IO_LABELS, nlab * sizeof(long long))) || (rc = ct_reserve(net, IO_LOGITS, nlog * sizeof(float))) ||
      (rc = ct_reserve(net, IO_MIN, sizeof(float))) || (rc = ct_reserve(net, IO_PACKED, total * 4 * sizeof(long long))))
    return rc;
  if ((rc = chd_contact_forward_device(net, (const double*)net->io[IO_FRAMES], V, Fmax, (const int*)net->io[IO_LENS], (int64_t*)net->io[IO_LABELS],
                                       (float*)net->io[IO_LOGITS], (float*)net->io[IO_MIN], net->stream)))
    return rc;
  if (scored && (rc = chd_contact_score_device(net, (const float*)net->io[IO_LOGITS], V, Fmax, (const int*)net->io[IO_TRUTH],
                                               (const int*)net->io[IO_TOFFS], classify_thresh, d_loss, d_frames, d_merged, net->stream)))
    return rc;
  // (V, Fmax, 4) labels -> the rows foot_contacts.npy keeps, then one download
  chd_k_contact_pack<<<dim3(4, V), 256, 0, net->stream>>>((const long long*)net->io[IO_LABELS], (const int*)net->io[IO_OFFS], V, Fmax,
                                                          (long long*)net->io[IO_PACKED]);
  net->launches += 1;
  CT_CUDA(cudaGetLastError());
  CT_CUDA(cudaMemcpyAsync(labels_out, net->io[IO_PACKED], total * 4 * sizeof(long long), cudaMemcpyDeviceToHost, net->stream));
  if (min_abs_logit) CT_CUDA(cudaMemcpyAsync(min_abs_logit, net->io[IO_MIN], sizeof(float), cudaMemcpyDeviceToHost, net->stream));
  if (scored) {
    CT_CUDA(cudaMemcpyAsync(loss_sum, d_loss, V * sizeof(double), cudaMemcpyDeviceToHost, net->stream));
    CT_CUDA(cudaMemcpyAsync(conf_frames, d_frames, (size_t)V * 20 * sizeof(int64_t), cudaMemcpyDeviceToHost, net->stream));
    CT_CUDA(cudaMemcpyAsync(conf_merged, d_merged, (size_t)V * 4 * sizeof(int64_t), cudaMemcpyDeviceToHost, net->stream));
  }
  CT_CUDA(cudaStreamSynchronize(net->stream));
  return 0;
}

int64_t chd_contact_launch_count(const chd_contact_net* net) { return net ? net->launches : 0; }

int chd_contact_set_precision(chd_contact_net* net, int32_t precision) {
  if (!net || (precision != CHD_CONTACT_FP32 && precision != CHD_CONTACT_TF32X3)) return -1;
  if (precision == CHD_CONTACT_FP32) {             // the FP32 kernels never read the fast mode's buffers
    if (net->tc_w) cudaFree(net->tc_w);
    if (net->io[IO_TC_WS]) cudaFree(net->io[IO_TC_WS]);
    net->tc_w = nullptr, net->io[IO_TC_WS] = nullptr, net->io_bytes[IO_TC_WS] = 0, net->tc = ChdContactTcNet{};
  } else if (!net->tc_w) {                         // split the weights of the three large layers once
    const int K[3] = {CT_K0, 1024, 512}, N[3] = {1024, 512, 128};
    size_t n = 0;
    for (int l = 0; l < 3; ++l) n += 2 * (size_t)K[l] * N[l];
    float* w = nullptr;
    CT_CUDA(cudaMalloc((void**)&w, n * sizeof(float)));
    ChdContactTcNet tc = {};
    float* p = w;
    int rc = 0;
    for (int l = 0; l < 3 && !rc; ++l) {
      float *hi = p, *lo = p + (size_t)K[l] * N[l];
      p = lo + (size_t)K[l] * N[l];
      tc.w_hi[l] = hi, tc.w_lo[l] = lo;
      tc.bias[l] = net->dev.b[l], tc.scale[l] = net->dev.bn_scale[l], tc.mean[l] = net->dev.bn_mean[l], tc.beta[l] = net->dev.bn_beta[l];
      rc = chd_contact_tc_split(net->dev.W[l], K[l], N[l], hi, lo, net->stream);
      net->launches += 1;
    }
    if (!rc) {
      const cudaError_t e = cudaStreamSynchronize(net->stream);
      if (e != cudaSuccess) rc = -100 - (int)e;
    }
    if (rc) {
      cudaFree(w);
      return rc;
    }
    net->tc_w = w, net->tc = tc;
  }
  net->precision = precision;
  return 0;
}

}  // extern "C"
