// Internal interface of the 3xTF32 tensor-core layers of the contact classifier (chd_contact_tc.cu), used by
// chd_contact.cu when a net is switched to CHD_CONTACT_TF32X3.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstddef>

// The three large layers (352 -> 1024 -> 512 -> 128) in the fast mode.
struct ChdContactTcNet {
  const float* w_hi[3];   // [N][K] tf32-rounded weights (K-major: the only B layout wgmma takes for tf32)
  const float* w_lo[3];   // [N][K] tf32-rounded residuals W - w_hi
  const float* bias[3];
  const float* scale[3];  // gamma / sqrt(var + eps)
  const float* mean[3];
  const float* beta[3];
};

// Tensor maps and activation planes of one forward call (the workspace may be reallocated between calls).
struct ChdContactTcPlan {
  CUtensorMap a_hi[3], a_lo[3], w_hi[3], w_lo[3];
  float* act_hi[3];       // A0 [rows][352], A1 [rows][1024], A2 [rows][512]
  float* act_lo[3];
  float* a3;              // [rows][128] plain fp32, the input of chd_k_contact_tail
  const ChdContactTcNet* net;
};

// Floats of the fast mode's workspace for a slab of `rows` windows: hi and lo planes of A0..A2, then A3.
size_t chd_contact_tc_ws_floats(int rows);
// W [K][N] fp32 (the FFMA layout) -> hi, lo [N][K].  One launch on s.
int chd_contact_tc_split(const float* W, int K, int N, float* hi, float* lo, cudaStream_t s);
// Encodes the tensor maps of a workspace of `rows` windows (rows % 128 == 0).  0 or <= -100.
int chd_contact_tc_plan(const ChdContactTcNet* net, float* ws, int rows, ChdContactTcPlan* plan);
// Windows g0 .. g0+Mp-1 of frames [V][Fmax][25][3] -> plan.a3: the split gather and the three tensor-core layers,
// four launches on s.
int chd_contact_tc_layers(const ChdContactTcPlan& plan, const double* frames, int V, int Fmax, int g0, int Mp, cudaStream_t s);
