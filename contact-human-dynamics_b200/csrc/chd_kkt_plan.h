// Sizes of a batch's KKT systems (product code): the tile-format storage of a sequence's matrix (chd_kkt_tiles.cuh),
// which KKT kernel runs, its dynamic shared memory and the global scratch of chd_k_kkt_gwin.  Batch creation sizes the
// buffers and picks the kernel from it, and the layout builder checks a band with chd_kkt_gwin_status; the kernels
// carve their shared memory and scratch from the sizes it puts into ChdDev (chd_kkt_ctx_init).
#pragma once
#include <cstddef>

#include "chd_core.h"

#define CHD_KKT_THREADS 512
#define CHD_KKT_GROUPS_MAX 96          /* panel groups (band tiles below the diagonal + border tiles) chd_k_kkt_gwin's pair table holds */
#define CHD_SMEM_OPTIN 232448          /* shared memory per block an sm_90 kernel may opt in to (227 KB) */
#define CHD_KKT_GWIN_STATIC_MAX 16384  /* bound on chd_k_kkt_gwin's static shared memory (ptxas: 12144 B) */

enum ChdKktStatus {
  CHD_KKT_FITS = 0,
  CHD_KKT_TOO_WIDE_COMPACT = 1,   // chd_k_kkt: more than 64 panel groups for its compacted trailing-update loop
  CHD_KKT_TOO_WIDE_PAIRS = 2,     // chd_k_kkt_gwin: more than CHD_KKT_GROUPS_MAX panel groups for its pair table
  CHD_KKT_TOO_LARGE = 3,          // dynamic + static shared memory above the per-block opt-in limit
};

// chd_k_kkt_gwin, the kernel wide bands run in, for half bandwidth w_max and nb_max border unknowns: its dynamic shared
// memory (bytes), and whether its pair table and its dynamic + static shared memory fit.
CHD_HD size_t chd_kkt_gwin_smem(int Q, int nbt) {
  return (CHD_KKT_THREADS + 64 * (size_t)nbt * nbt + 2 * (size_t)(Q + nbt) * 64 + 16) * sizeof(double);
}
CHD_HD int chd_kkt_gwin_status(int w_max, int nb_max, size_t gwin_static, size_t smem_optin) {
  const int Q = (w_max + 7) / 8 + 1, nbt = (nb_max + 1 + 7) / 8;
  if (Q - 1 + nbt > CHD_KKT_GROUPS_MAX) return CHD_KKT_TOO_WIDE_PAIRS;
  if (chd_kkt_gwin_smem(Q, nbt) + gwin_static + 256 > smem_optin) return CHD_KKT_TOO_LARGE;
  return CHD_KKT_FITS;
}

// Sizes in doubles unless noted.  Dynamic shared memory (chd_kkt_ctx_init):
//   red[CHD_KKT_THREADS] | cc[nbp8^2] | ypan, xpan ... [pan_doubles] | dinv[16] | win[win_tiles*64] | bwin[Q*nbt*64]
// With win_smem (chd_k_kkt) the per-unknown vectors vecn[n_even] and xs[8*nbc_max + nbp8] alias the tail of win | bwin
// and the back-substitution stages two chunks of block rows in its front; otherwise (chd_k_kkt_gwin) the scratch holds
// vecn | xs | xs2[8*nbc_max] | win | bwin per sequence and shared memory ends after dinv.
struct ChdKktPlan {
  int status;                     // ChdKktStatus
  int win_smem;                   // 1: chd_k_kkt, window and vectors in shared memory; 0: chd_k_kkt_gwin, in the scratch
  int nbc_max, Q, Qfix, nbt;      // block columns, band tiles per block column (storage / fixed-duration stages), border tiles
  int win_tiles, pan_doubles;     // window slots; panel buffers (and with win_smem the back-substitution accumulator)
  size_t kstride;                 // storage per sequence: band | bord | corn
  size_t smem_bytes;              // dynamic shared memory of the KKT kernel (bytes)
  size_t scratch_stride;          // per sequence in the scratch (0: no scratch)
};

// Na_max / nb_max / w_max / w_fix_max / n_max: the batch's strides (chd_layout.h).  kkt_static / gwin_static: static
// shared memory of chd_k_kkt / chd_k_kkt_gwin; smem_optin: the per-block opt-in limit (bytes).
CHD_HD ChdKktPlan chd_kkt_plan(int Na_max, int nb_max, int w_max, int w_fix_max, int n_max, size_t kkt_static,
                               size_t gwin_static, size_t smem_optin) {
  ChdKktPlan P = {};
  P.nbc_max = (Na_max + 7) / 8;
  P.Q = (w_max + 7) / 8 + 1;
  P.Qfix = (w_fix_max + 7) / 8 + 1;
  P.nbt = (nb_max + 1 + 7) / 8;   // border unknowns + the right-hand-side row
  P.win_tiles = P.Q * (P.Q + 1) / 2 > 2 * P.Q ? P.Q * (P.Q + 1) / 2 : 2 * P.Q;
  const size_t nbc = P.nbc_max, Q = P.Q, nbt = P.nbt, nbp8 = 8 * nbt;
  P.kstride = nbc * Q * 64 + nbc * nbt * 64 + nbp8 * nbp8;
  const size_t win_region = (size_t)P.win_tiles * 64 + Q * nbt * 64;
  const size_t n_even = (size_t)((n_max + 1) & ~1), xs_len = 8 * nbc + nbp8;
  // the vectors alias the tail of the window, the back-substitution stages two block rows (Q tiles each) at least in
  // its front.  (+ 3072: chd_k_kkt's former distance-row curvature scratch; it guards nothing now, but dropping it
  // would move borderline batches from chd_k_kkt_gwin onto chd_k_kkt)
  const bool vectors_fit = win_region >= n_even + xs_len + 2 * Q * 64 + 3072;
  const size_t pan_ws = 2 * (Q + nbt) * 64 > 8 * nbc ? 2 * (Q + nbt) * 64 : 8 * nbc;
  const size_t ws_bytes = (CHD_KKT_THREADS + nbp8 * nbp8 + pan_ws + 16 + win_region) * sizeof(double);
  if (vectors_fit && ws_bytes + kkt_static + 256 <= smem_optin) {
    P.win_smem = 1;
    P.pan_doubles = (int)pan_ws;
    P.smem_bytes = ws_bytes;
    // any window that fits is well below 64 panel groups (Q + nbt <= 30 at 227 KB)
    P.status = Q - 1 + nbt > 64 ? CHD_KKT_TOO_WIDE_COMPACT : CHD_KKT_FITS;
  } else {
    // long horizons / wide bands: vectors and window in a global scratch area
    P.pan_doubles = (int)(2 * (Q + nbt) * 64);
    P.smem_bytes = chd_kkt_gwin_smem(P.Q, P.nbt);
    P.scratch_stride = n_even + xs_len + 8 * nbc + win_region;
    P.status = chd_kkt_gwin_status(w_max, nb_max, gwin_static, smem_optin);
  }
  return P;
}
