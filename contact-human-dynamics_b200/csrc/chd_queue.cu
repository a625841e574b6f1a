// sm_90a admission kernel of the physics solve queue (chd_phys_queue_create / chd_phys_queue_solve, chd_api.cu).
//
// A queue solves N clips through S <= N slots of one batch.  When a slot's clip has finished its schedule the host
// stages the next clips' records (every per-sequence row of the layout tables, built once over all N clips so that
// every clip fits every slot) and launches chd_k_admit over the slots being refilled.
#include <cuda_runtime.h>

#include "chd_dev.h"

// grid (CTAs per slot, admitted slots), 256 threads.  For admitted slot j = blockIdx.y:
//  - copies its staged record into the slot's rows of the layout tables, of the working copies of the tables stage 3
//    rewrites (and of their pristine and trial copies) and of the iterate;
//  - zeroes the slot's rows of every array batch creation zeroes: the iterate's companions and the multipliers, the
//    Jacobian values, row flags, KKT matrices, solution and right-hand sides, scratch, costs and SaveSolution rows;
//  - (CTA 0) resets the slot's interior-point state to that of a freshly created batch: all zero, at the start of the
//    schedule.
// A refilled slot is then, to every kernel, the same as that row of a freshly created batch.  The zeroing is needed
// because the previous clip may have been longer, had more feet or run stage 3: the kernels read the entries of a row
// beyond a shorter clip's n / m / Na and the padding of the KKT tiles as zeros (a fresh batch's allocations are
// zeroed), and the previous clip's values left there would reach the next clip's factorisation, sums and snapshots.
__global__ void chd_k_admit(ChdDev D, ChdAdmit A) {
  const int j = blockIdx.y;
  const int slot = A.slot[j];
  const char* rec = A.rec + (size_t)j * A.rec_bytes;
  const size_t t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nt = (size_t)gridDim.x * blockDim.x;
  for (int k = 0; k < A.nseg; ++k) {
    const ChdAdmitSeg sg = A.seg[k];
    char* dst = sg.dst + (size_t)slot * sg.slot_bytes;
    const char* src = sg.src >= 0 ? rec + sg.src : nullptr;
    const size_t align = (size_t)dst | sg.bytes | (src ? (size_t)src : 0);
    if ((align & 15) == 0) {
      uint4* d = (uint4*)dst;
      const uint4* s = (const uint4*)src;
      for (size_t i = t0; i < sg.bytes / 16; i += nt) d[i] = s ? s[i] : make_uint4(0, 0, 0, 0);
    } else if ((align & 3) == 0) {
      unsigned* d = (unsigned*)dst;
      const unsigned* s = (const unsigned*)src;
      for (size_t i = t0; i < sg.bytes / 4; i += nt) d[i] = s ? s[i] : 0u;
    } else {
      for (size_t i = t0; i < sg.bytes; i += nt) dst[i] = src ? src[i] : 0;
    }
  }
  if (blockIdx.x == 0) {
    unsigned* w = (unsigned*)(D.ipm + slot);
    for (int i = threadIdx.x; i < (int)(sizeof(ChdIpm) / 4); i += blockDim.x) w[i] = 0u;
    __syncthreads();
    if (threadIdx.x == 0) chd_sched_begin(D, D.ipm[slot]);
  }
}
