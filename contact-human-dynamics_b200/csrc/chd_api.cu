// C ABI of the phys-optim path (see include/chd.h).  Host driver: device memory, stage loops, launches.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>

#include "../../include/chd.h"
#include "chd_dev.h"

// kernels (chd_kernels.cu)
__global__ void chd_k_stage_begin(ChdDev D);
template <bool GLOBAL>
__global__ void chd_k_eval(ChdDev D);
__global__ void chd_k_init(ChdDev D);
__global__ void chd_k_kkt(ChdDev D);
__global__ void chd_k_kkt_gwin(ChdDev D);
__global__ void chd_k_kcopy(ChdDev D);
__global__ void chd_k_curv(ChdDev D);
__global__ void chd_k_asm(ChdDev D);
__global__ void chd_k_fp64_peak(int mode, int iters, double* sink);
__global__ void chd_k_hess_base(ChdDev D);
__global__ void chd_k_hess_dur(ChdDev D);
__global__ void chd_k_hess_zero(ChdDev D);
__global__ void chd_k_hess_fin(ChdDev D, int mode);
__global__ void chd_k_tables(ChdDev D);
__global__ void chd_k_clear_dyn(ChdDev D);
template <bool GLOBAL>
__global__ void chd_k_linesearch(ChdDev D);
__global__ void chd_k_sample(ChdDev D, double* out, int* frames_out);
__global__ void chd_k_snapshot(ChdDev D, int* frames_out);
__global__ void chd_k_sched_reset(ChdDev D);
__global__ void chd_k_admit(ChdDev D, ChdAdmit A);   // chd_queue.cu
__global__ void chd_k_cost_terms(ChdDev D, int finished_only, double* out);

#define CHD_CUDA(x)                                                                          \
  do {                                                                                       \
    cudaError_t e_ = (x);                                                                    \
    if (e_ != cudaSuccess) {                                                                 \
      fprintf(stderr, "libchd: CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      return -100 - (int)e_;                                                                 \
    }                                                                                        \
  } while (0)

enum { KT_EVAL = 0, KT_KKT = 1, KT_LS = 2, KT_INIT = 3, KT_SAMPLE = 4, KT_ADMIT = 5, KT_N = 8 };

// Form of the evaluation and line-search kernels for a batch: with the iterate (and the gradient) in shared memory
// when twice the longest sequence's iterate fits the opt-in limit, otherwise with both in global memory (D.x / D.grad /
// D.xt) and only the block-reduction buffer in shared memory.  The input size decides; batch creation picks it once.
struct ChdIterForm {
  void (*eval)(ChdDev);
  void (*linesearch)(ChdDev);
  size_t smem_eval, smem_ls;   // dynamic shared memory per CTA
};
static ChdIterForm chd_iter_form(int n_max, int smem_optin) {
  const size_t red = CHD_THREADS * sizeof(double);
  if ((2 * (size_t)n_max + CHD_THREADS) * sizeof(double) + 1024 <= (size_t)smem_optin)
    return {chd_k_eval<false>, chd_k_linesearch<false>, 2 * (size_t)n_max * sizeof(double) + red,
            (size_t)n_max * sizeof(double) + red};
  return {chd_k_eval<true>, chd_k_linesearch<true>, red, red};
}

// Queue of clips solved through the slots of a batch (chd_phys_queue_create): the layout rows of every clip packed
// into one record per clip, the admission kernel's segment table and the state of the running solve.
struct ChdQueue {
  int n = 0;                          // clips
  size_t rec_bytes = 0;               // bytes of one record (every row starts 16-byte aligned)
  char* store = nullptr;              // n records, page-locked (host-only handles: pageable)
  char* d_stage = nullptr;            // device staging area, one record per slot
  int *h_slot = nullptr, *d_slot = nullptr;   // slots being refilled (page-locked / device)
  ChdAdmit adm = {};
  int admit_blocks = 1;               // CTAs per admitted slot
  std::vector<int> clip;              // clip held by every slot, -1: none (harvested)
  int next = 0;                       // first clip not admitted yet
  // claim source (chd_phys_queue_set_claim), NULL: the queue's own order
  chd_phys_claim_fn* claim = nullptr;
  void* claim_ctx = nullptr;
  bool exhausted = false;             // the source returned fewer positions than asked during this solve
  std::vector<char> given;            // positions the source handed out during this solve
};

// Outputs of the running chd_phys_solve / chd_phys_queue_solve (NULL: not asked for), indexed by sequence (a queue: by
// clip) with n sequences (clips) per stage row.
struct ChdSolveOut {
  size_t n = 0;
  double *samples = nullptr, *stage_stats = nullptr, *terms = nullptr;
  int32_t *frames = nullptr, *success = nullptr, *stage_status = nullptr, *stage_iters = nullptr;
};

struct chd_phys_batch {
  ChdHostBatch hb;
  ChdDev D;
  std::vector<void*> allocs;
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  cudaEvent_t ev_kkt = nullptr, ev_ls = nullptr, ev_copy = nullptr;
  int64_t launches = 0;
  int timing = 0;
  bool host_only = false;
  double kt_ms[KT_N] = {0};
  int64_t kt_n[KT_N] = {0};
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int* d_frames = nullptr;
  double* d_samples = nullptr;
  ChdIterForm iter = {};   // evaluation / line-search kernels and their shared memory (chd_iter_form)
  size_t smem_kkt = 0;
  int kcopy_blocks = 1;
  ChdIpm* h_ipm = nullptr;  // host copy of the per-sequence solver state
  double* d_x0 = nullptr;
  int64_t h2d_bytes = 0;
  std::vector<ChdStageDev> stages;   // B x 6 rows of the stage table (a queue: of the slots; its records hold every clip's)
  std::vector<ChdStageEnd> ends;     // B records behind the stage rows on the device (a queue: as `stages`)
  std::vector<chd_phys_solver_options> opts;   // every sequence's (a queue: every clip's) options, defaults resolved
  ChdStageDev* d_stages = nullptr;
  double* terms_out = nullptr;        // chd_phys_set_cost_terms_out: [host] where a solve writes the final cost terms
  double* d_terms = nullptr;          // B x CHD_PHYS_N_TERMS (chd_k_cost_terms)
  int sched_max_iter = 0;
  bool sched_has_dur = false;   // the running schedule contains stage 3 (its cost Hessian is rebuilt every iteration)
  // pristine copies of the tables stage 3 rewrites (chd_phys_reset)
  double *poly_T0 = nullptr, *poly_tend0 = nullptr, *phase_tend0 = nullptr;
  int* ent_col0 = nullptr;
  ChdQueue* queue = nullptr;   // a queue handle: the batch's sequences are slots that clips pass through
  ChdSolveOut out;
};

namespace {

// the staged schedule of a full solve (phys_optim.cpp:554-749)
const int full_schedule[6] = {CHD_STAGE_11, CHD_STAGE_12, CHD_STAGE_21, CHD_STAGE_22, CHD_STAGE_3, CHD_STAGE_4};

// doubles of a SaveSolution sample row (chd.phys.sample_stride)
size_t sample_stride(const ChdHostBatch& hb) { return 6 + 7 * (size_t)hb.n_ee_max; }

// success flags, stage statuses, iterations and (when asked for) stage statistics of sequence (clip) c from its solver
// state
void write_status(const ChdSolveOut& o, size_t c, const ChdIpm& I) {
  // dynamics_succeed (:655); durations_succeed = stage 3 (:709), overwritten by stage 4 when that had to run (:746)
  if (o.success) o.success[2 * c] = I.st_status[CHD_STAGE_22] == 0, o.success[2 * c + 1] = I.st_status[CHD_STAGE_3] == 0 || I.st_status[CHD_STAGE_4] == 0;
  for (size_t s = 0; s < 6; ++s) {
    if (o.stage_status) o.stage_status[s * o.n + c] = I.st_status[s];
    if (o.stage_iters) o.stage_iters[s * o.n + c] = I.st_iters[s];
    if (o.stage_stats)
      for (int k = 0; k < 4; ++k) o.stage_stats[(s * o.n + c) * 4 + k] = I.st_stat[s][k];
  }
}

// the SaveSolution snapshots clip c does not take, those after its last stage, are NaN (row: doubles of one snapshot)
void write_untaken(const ChdSolveOut& o, size_t c, int last_stage, size_t row) {
  for (size_t s = last_stage + 1; o.samples && s < 3; ++s) std::fill_n(o.samples + (s * o.n + c) * row, row, NAN);
}

template <class T>
int dev_upload(chd_phys_batch* b, const std::vector<T>& v, const T** out) {
  void* p = nullptr;
  size_t bytes = std::max<size_t>(v.size(), 1) * sizeof(T);
  CHD_CUDA(cudaMallocAsync(&p, bytes, b->stream));      // stream-ordered pool: freed blocks are reused by the next batch
  b->allocs.push_back(p);
  if (!v.empty()) CHD_CUDA(cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, b->stream));
  b->h2d_bytes += (int64_t)(v.size() * sizeof(T));
  *out = (const T*)p;
  return 0;
}
template <class T>
int dev_alloc(chd_phys_batch* b, size_t count, T** out) {
  void* p = nullptr;
  CHD_CUDA(cudaMallocAsync(&p, std::max<size_t>(count, 1) * sizeof(T), b->stream));
  CHD_CUDA(cudaMemsetAsync(p, 0, std::max<size_t>(count, 1) * sizeof(T), b->stream));
  b->allocs.push_back(p);
  *out = (T*)p;
  return 0;
}

// the stage a last_stage option ends with (CHD_LAST_DURATIONS: none, the schedule's own end)
int last_stage_id(int last_stage) {
  return last_stage == CHD_LAST_NO_DYNAMICS ? CHD_STAGE_12 : (last_stage == CHD_LAST_DYNAMICS ? CHD_STAGE_22 : -1);
}

// row `stage` of a sequence's stage table: its layout's configuration with the cap of its solver options
ChdStageDev stage_dev(const ChdStageCfg& c, int stage, const chd_phys_solver_options& o) {
  ChdStageDev s;
  s.set_mask = c.set_mask;
  s.max_iter = o.max_iter[stage];
  s.snap_after = stage == CHD_STAGE_12 ? 0 : (stage == CHD_STAGE_22 ? 1 : ((stage == CHD_STAGE_4 || stage == CHD_STAGE_3) ? 2 : -1));
  s.opt_dur = stage == CHD_STAGE_3;
  for (int i = 0; i < 3; ++i) s.w_data[i] = c.w_data[i], s.w_vel[i] = c.w_vel[i], s.w_acc[i] = c.w_acc[i];
  s.w_dur = c.w_dur;
  return s;
}

ChdStageEnd stage_end(const chd_phys_solver_options& o) {
  return {o.tol, o.constr_viol_tol, o.dual_inf_tol, o.compl_inf_tol, last_stage_id(o.last_stage), 0};
}

// options of a clip as given (NULL: the defaults), with every cap of 0 resolved to the stage's own in `stages` (its six
// rows of the layout)
chd_phys_solver_options resolve_options(const chd_phys_solver_options* given, const ChdStageCfg* stages) {
  chd_phys_solver_options o = {CHD_TOL, CHD_CONSTR_VIOL_TOL, CHD_DUAL_INF_TOL, CHD_COMPL_INF_TOL, {0}, CHD_LAST_DURATIONS};
  if (given) o = *given;
  for (int s = 0; s < 6; ++s)
    if (o.max_iter[s] == 0) o.max_iter[s] = stages[s].max_iter;
  return o;
}

// a tolerance not finite or not > 0, a negative cap or an unknown last stage
bool bad_options(const chd_phys_solver_options& o) {
  for (double v : {o.tol, o.constr_viol_tol, o.dual_inf_tol, o.compl_inf_tol})
    if (!std::isfinite(v) || !(v > 0.0)) return true;
  for (int s = 0; s < 6; ++s)
    if (o.max_iter[s] < 0) return true;
  return o.last_stage < CHD_LAST_NO_DYNAMICS || o.last_stage > CHD_LAST_DURATIONS;
}

struct Timer {
  chd_phys_batch* b;
  int id;
  Timer(chd_phys_batch* bb, int i) : b(bb), id(i) {
    if (b->timing) cudaEventRecord(b->ev0, b->stream);
  }
  ~Timer() {
    b->launches++;
    b->kt_n[id]++;
    if (b->timing) {
      cudaEventRecord(b->ev1, b->stream);
      cudaEventSynchronize(b->ev1);
      float ms = 0;
      cudaEventElapsedTime(&ms, b->ev0, b->ev1);
      b->kt_ms[id] += ms;
    }
  }
};

void launch_eval(chd_phys_batch* b) {
  Timer t(b, KT_EVAL);
  b->iter.eval<<<b->hb.B, CHD_THREADS, b->iter.smem_eval, b->stream>>>(b->D);
}

// uploads the stage table (optionally with an iteration-cap override for one stage) and the schedule
int set_schedule(chd_phys_batch* b, const int* sched, int nsched, int override_stage, int override_max_iter) {
  std::vector<ChdStageDev> tab = b->stages;
  if (override_stage >= 0 && override_max_iter > 0)
    for (size_t i = 0; i < tab.size(); i += 6) tab[i + override_stage].max_iter = override_max_iter;
  CHD_CUDA(cudaMemcpyAsync(b->d_stages, tab.data(), tab.size() * sizeof(ChdStageDev), cudaMemcpyHostToDevice, b->stream));
  b->D.nsched = nsched;
  for (int i = 0; i < nsched; ++i) b->D.sched[i] = sched[i];
  b->sched_has_dur = false;
  for (int i = 0; i < nsched; ++i) b->sched_has_dur |= sched[i] == CHD_STAGE_3;
  // bound of the launch loop: the largest sum of a sequence's caps over the schedule (a queue: of any of its clips)
  b->sched_max_iter = 0;
  for (const chd_phys_solver_options& o : b->opts) {
    int sum = 0;
    for (int i = 0; i < nsched; ++i)
      sum += (sched[i] == override_stage && override_max_iter > 0 ? override_max_iter : o.max_iter[sched[i]]) + 2;
    b->sched_max_iter = std::max(b->sched_max_iter, sum);
  }
  chd_k_sched_reset<<<(b->hb.B + 127) / 128, 128, 0, b->stream>>>(b->D);
  b->launches++;
  return 0;
}

int queue_refill(chd_phys_batch* b, int it, int* last_it);

// the cost terms of every sequence (finished_only: of those whose schedule is over) into d_terms
void launch_cost_terms(chd_phys_batch* b, int finished_only) {
  chd_k_cost_terms<<<b->hb.B, CHD_TERMS_THREADS, 0, b->stream>>>(b->D, finished_only, b->d_terms);
  b->launches++;
}

// runs the uploaded schedule to completion: every sequence walks through its stages at its own pace (a queue refills
// the slots whose clip has finished at the check points, and the loop runs until the last admitted clip finishes)
int run_schedule(chd_phys_batch* b) {
  const int B = b->hb.B;
  const int check_every = 8;
  int last_it = b->sched_max_iter;
  for (int it = 0; it <= last_it; ++it) {
    {
      Timer t(b, KT_INIT);
      chd_k_stage_begin<<<B, CHD_THREADS, 0, b->stream>>>(b->D);
    }
    launch_eval(b);
    {
      Timer t(b, KT_INIT);
      chd_k_init<<<B, CHD_THREADS, 0, b->stream>>>(b->D);
    }
    {
      Timer t(b, KT_INIT);
      chd_k_hess_zero<<<dim3(8, B), 256, 0, b->stream>>>(b->D);
      chd_k_hess_base<<<dim3(16, B), 256, 0, b->stream>>>(b->D);
      chd_k_hess_fin<<<B, 128, 0, b->stream>>>(b->D, 0);
      b->launches += 2;
    }
    // Kwork refreshed by the side stream (iteration 0: the event has not been recorded yet and the wait is a no-op; the
    // sequences that begin a stage had Kwork prepared by the chd_k_hess_* kernels above)
    CHD_CUDA(cudaStreamWaitEvent(b->stream, b->ev_copy, 0));
    chd_k_asm<<<dim3(8, B), 256, 0, b->stream>>>(b->D);
    b->launches++;
    {
      Timer t(b, KT_KKT);
      if (b->D.win_smem) chd_k_kkt<<<B, CHD_KKT_THREADS, b->smem_kkt, b->stream>>>(b->D);
      else chd_k_kkt_gwin<<<B, CHD_KKT_THREADS, b->smem_kkt, b->stream>>>(b->D);
    }
    // Kwork <- Kbase for the next iteration, overlapped with the line search / evaluation kernels (sequences in stage 3
    // are skipped: their cost Hessian moves with the durations and is rebuilt into Kwork after the line search)
    CHD_CUDA(cudaEventRecord(b->ev_kkt, b->stream));
    CHD_CUDA(cudaStreamWaitEvent(b->copy_stream, b->ev_kkt, 0));
    chd_k_kcopy<<<dim3(b->kcopy_blocks, B), 256, 0, b->copy_stream>>>(b->D);
    b->launches++;
    {
      Timer t(b, KT_LS);
      b->iter.linesearch<<<B, CHD_THREADS, b->iter.smem_ls, b->stream>>>(b->D);
    }
    // distance-row curvature of the next iteration needs the accepted iterate: after the line search, on the side stream
    CHD_CUDA(cudaEventRecord(b->ev_ls, b->stream));
    CHD_CUDA(cudaStreamWaitEvent(b->copy_stream, b->ev_ls, 0));
    if (b->sched_has_dur) {
      chd_k_hess_dur<<<dim3(8, B), CHD_THREADS, 0, b->copy_stream>>>(b->D);
      chd_k_hess_fin<<<B, 128, 0, b->copy_stream>>>(b->D, 1);
      b->launches += 2;
    }
    chd_k_curv<<<dim3(8, B), 256, 0, b->copy_stream>>>(b->D);
    b->launches++;
    CHD_CUDA(cudaEventRecord(b->ev_copy, b->copy_stream));
    {
      Timer t(b, KT_SAMPLE);
      chd_k_snapshot<<<B, 128, 0, b->stream>>>(b->D, b->d_frames);
    }
    if ((it % check_every) == check_every - 1) {
      CHD_CUDA(cudaMemcpyAsync(b->h_ipm, b->D.ipm, B * sizeof(ChdIpm), cudaMemcpyDeviceToHost, b->stream));
      CHD_CUDA(cudaStreamSynchronize(b->stream));
      if (b->queue) {
        const int rc = queue_refill(b, it, &last_it);
        if (rc) return rc;
      }
      bool any = false;
      for (int i = 0; i < B; ++i) any |= (b->h_ipm[i].phase != CHD_PH_FINISHED);
      if (!any) break;
    }
  }
  CHD_CUDA(cudaMemcpyAsync(b->h_ipm, b->D.ipm, B * sizeof(ChdIpm), cudaMemcpyDeviceToHost, b->stream));
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  CHD_CUDA(cudaStreamSynchronize(b->copy_stream));
  CHD_CUDA(cudaGetLastError());
  return 0;
}

size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

// Every host layout table with one row per sequence, with the device arrays a clip's row goes to when it is admitted
// to a slot: the read-only tables; the iterate; the tables stage 3 rewrites with their pristine and trial copies.
template <class F>
void queue_tables(chd_phys_batch* b, F&& f) {
  ChdHostBatch& hb = b->hb;
  ChdDev& D = b->D;
  f(hb.seq, D.seq), f(hb.sets, D.sets), f(hb.node_var, D.node_var), f(hb.itab, D.itab), f(hb.ent_ptr, D.ent_ptr);
  f(hb.ent_col, D.ent_col, b->ent_col0), f(hb.ent_row, D.ent_row), f(hb.col_ptr, D.col_ptr), f(hb.col_ent, D.col_ent);
  f(hb.var_kkt, D.var_kkt), f(hb.row_kkt, D.row_kkt), f(hb.row_set, D.row_set), f(hb.poly_ph, D.poly_ph);
  f(hb.node_const, D.node_const), f(hb.par, D.par), f(hb.t_dyn, D.t_dyn), f(hb.t_rom, D.t_rom), f(hb.t_data, D.t_data);
  f(hb.row_lo, D.row_lo), f(hb.row_hi, D.row_hi), f(hb.dur0, D.dur0), f(hb.x0, D.x, b->d_x0);
  f(hb.poly_T, D.poly_T, b->poly_T0, D.poly_Tt), f(hb.poly_tend, D.poly_tend, b->poly_tend0, D.poly_tendt);
  f(hb.phase_tend, D.phase_tend, b->phase_tend0), f(b->stages, D.stages);
  f(b->ends, D.stages ? (const void*)(D.stages + b->stages.size()) : nullptr);
}

// Packs the layout of all hb.B clips into one record per clip and keeps the first `slots` rows of every table as the
// batch's own layout (the strides stay those of all clips).
int queue_pack(chd_phys_batch* b, int slots) {
  ChdQueue& q = *(b->queue = new ChdQueue());
  const size_t n = b->hb.B;
  q.n = (int)n;
  queue_tables(b, [&](auto& v, const void*, const void* = nullptr, const void* = nullptr) {
    q.rec_bytes = align16(q.rec_bytes) + v.size() / n * sizeof(v[0]);
  });
  q.rec_bytes = align16(q.rec_bytes);
  if (b->host_only) q.store = (char*)std::malloc(n * q.rec_bytes);
  else CHD_CUDA(cudaMallocHost((void**)&q.store, n * q.rec_bytes));
  if (!q.store) return -3;
  std::memset(q.store, 0, n * q.rec_bytes);
  size_t off = 0;
  queue_tables(b, [&](auto& v, const void*, const void* = nullptr, const void* = nullptr) {
    const size_t row = v.size() / n * sizeof(v[0]);
    off = align16(off);
    for (size_t i = 0; i < n; ++i) std::memcpy(q.store + i * q.rec_bytes + off, (const char*)v.data() + i * row, row);
    v.resize(v.size() / n * slots);
    off += row;
  });
  b->hb.B = slots;
  return 0;
}

// Segment table of the admission kernel over the batch's device arrays, staging area, slot list.
int queue_device(chd_phys_batch* b, int sms) {
  ChdQueue& q = *b->queue;
  const ChdHostBatch& hb = b->hb;
  const ChdDev& D = b->D;
  const size_t S = hb.B;
  ChdAdmit& A = q.adm;
  A.rec_bytes = q.rec_bytes;
  size_t off = 0, slot_bytes = 0;
  bool ok = true;
  auto seg = [&](const void* dst, size_t row, long long src) {
    if (A.nseg == CHD_ADMIT_SEGS) ok = false;
    else A.seg[A.nseg++] = {(char*)dst, row, row, src}, slot_bytes += row;
  };
  queue_tables(b, [&](auto& v, const void* d0, const void* d1 = nullptr, const void* d2 = nullptr) {
    const size_t row = v.size() / S * sizeof(v[0]);
    off = align16(off);
    for (const void* d : {d0, d1, d2})
      if (d) seg(d, row, (long long)off);
    off += row;
  });
  // zero fills: what dev_alloc zeroes at batch creation
  const size_t nb = hb.n_max * sizeof(double), mb = hb.m_max * sizeof(double), kb = (size_t)(hb.Na_max + hb.nb_max) * sizeof(double);
  for (const void* p : {(const void*)D.xt, (const void*)D.jty, (const void*)D.dx, (const void*)D.grad}) seg(p, nb, -1);
  seg(D.unobs, hb.n_max, -1);
  for (const double* p : {D.g, D.gt, D.sc, D.dL, D.dU, D.s, D.y, D.zL, D.zU, D.ds, D.dy, D.dzL, D.dzU}) seg(p, mb, -1);
  seg(D.rflag, hb.m_max * sizeof(int), -1);
  seg(D.Jv, hb.slots_max * sizeof(double), -1);
  seg(D.cost, 2 * sizeof(double), -1);
  seg(D.Kwork, D.kstride * sizeof(double), -1);
  seg(D.Kbase, D.kstride * sizeof(double), -1);
  for (const double* p : {D.sol, D.rhs0, D.rhs1}) seg(p, kb, -1);
  if (D.scratch) seg(D.scratch, D.scratch_stride * sizeof(double), -1);
  seg(b->d_frames, sizeof(int), -1);
  const size_t snap = hb.fo_max * sample_stride(hb) * sizeof(double);
  for (int s = 0; s < 3; ++s) {
    // the three SaveSolution snapshots are 3 x B x fo_max x stride: one row per slot in each
    if (A.nseg == CHD_ADMIT_SEGS) ok = false;
    else A.seg[A.nseg++] = {(char*)D.snapshots + s * S * snap, snap, snap, -1}, slot_bytes += snap;
  }
  if (!ok) {
    fprintf(stderr, "libchd: more than %d admission segments\n", CHD_ADMIT_SEGS);
    return -3;
  }
  // enough CTAs per slot that a single admitted slot spreads over the GPU, about 64 KB each
  q.admit_blocks = (int)std::min<size_t>(4 * (size_t)sms, std::max<size_t>(1, slot_bytes / 65536));
  CHD_CUDA(cudaMallocAsync((void**)&q.d_stage, S * q.rec_bytes, b->stream));
  b->allocs.push_back(q.d_stage);
  CHD_CUDA(cudaMallocAsync((void**)&q.d_slot, S * sizeof(int), b->stream));
  b->allocs.push_back(q.d_slot);
  CHD_CUDA(cudaMallocHost((void**)&q.h_slot, S * sizeof(int)));
  q.clip.assign(S, -1);
  return 0;
}

// admits the k clips at queue positions first, first + 1, ... into `slots` (in that order): one upload of their
// records, one launch
int queue_admit(chd_phys_batch* b, const int* slots, int k, int first) {
  ChdQueue& q = *b->queue;
  for (int j = 0; j < k; ++j) q.h_slot[j] = slots[j], q.clip[slots[j]] = first + j;
  Timer t(b, KT_ADMIT);
  CHD_CUDA(cudaMemcpyAsync(q.d_stage, q.store + (size_t)first * q.rec_bytes, k * q.rec_bytes, cudaMemcpyHostToDevice, b->stream));
  CHD_CUDA(cudaMemcpyAsync(q.d_slot, q.h_slot, k * sizeof(int), cudaMemcpyHostToDevice, b->stream));
  b->h2d_bytes += (int64_t)(k * (q.rec_bytes + sizeof(int)));
  q.adm.rec = q.d_stage, q.adm.slot = q.d_slot;
  chd_k_admit<<<dim3(q.admit_blocks, k), 256, 0, b->stream>>>(b->D, q.adm);
  return 0;
}

// asks the claim source for `want` positions: the k it hands out start at *first.  -1 if it fails, or hands out more
// than asked, a range outside [0, n) or a position it already handed out in this solve; the work in flight is drained
// first, so that nothing reaches the outputs after chd_phys_queue_solve has returned.
int queue_claim(chd_phys_batch* b, int want, int* first, int* k) {
  ChdQueue& q = *b->queue;
  int32_t f = 0;
  const int32_t got = q.claim(q.claim_ctx, want, &f);
  bool ok = got >= 0 && got <= want && (got == 0 || (f >= 0 && f <= q.n - got));
  for (int i = 0; ok && i < got; ++i) ok = !q.given[f + i];
  if (!ok) {
    cudaStreamSynchronize(b->stream);
    cudaStreamSynchronize(b->copy_stream);
    return -1;
  }
  for (int i = 0; i < got; ++i) q.given[f + i] = 1;
  q.exhausted = got < want;
  *first = f, *k = got;
  return 0;
}

// outputs of the clip in `slot` (its schedule is over, or the loop's bound was reached) into the clip's place
int queue_harvest(chd_phys_batch* b, int slot) {
  ChdQueue& q = *b->queue;
  const int c = q.clip[slot];
  if (c < 0) return 0;
  const ChdHostBatch& hb = b->hb;
  const ChdSolveOut& o = b->out;
  const size_t S = hb.B, row = hb.fo_max * sample_stride(hb);
  const int last = b->opts[c].last_stage;
  if (o.samples)
    for (size_t s = 0; s <= (size_t)last; ++s)
      CHD_CUDA(cudaMemcpyAsync(o.samples + (s * o.n + c) * row, b->D.snapshots + (s * S + slot) * row, row * sizeof(double),
                               cudaMemcpyDeviceToHost, b->stream));
  if (o.frames) CHD_CUDA(cudaMemcpyAsync(o.frames + c, b->d_frames + slot, sizeof(int), cudaMemcpyDeviceToHost, b->stream));
  if (o.terms)
    CHD_CUDA(cudaMemcpyAsync(o.terms + (size_t)c * CHD_PHYS_N_TERMS, b->d_terms + (size_t)slot * CHD_PHYS_N_TERMS,
                             CHD_PHYS_N_TERMS * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
  write_status(o, c, b->h_ipm[slot]);
  write_untaken(o, c, last, row);
  q.clip[slot] = -1;
  return 0;
}

// At a check point of run_schedule (h_ipm just copied): while clips are pending, the slots whose clip has finished are
// harvested and refilled with the next clips, in slot order.  With a claim source the next clips are the ones it hands
// out, and once it has run dry the finished slots are left to the final harvest.
int queue_refill(chd_phys_batch* b, int it, int* last_it) {
  ChdQueue& q = *b->queue;
  if (q.exhausted) return 0;
  const int pending = q.claim ? b->hb.B : q.n - q.next;
  std::vector<int> freed;
  for (int i = 0; i < b->hb.B && (int)freed.size() < pending; ++i)
    if (b->h_ipm[i].phase == CHD_PH_FINISHED) freed.push_back(i);
  if (freed.empty()) return 0;
  int rc, first = q.next, k = (int)freed.size();
  if (q.claim && (rc = queue_claim(b, k, &first, &k))) return rc;
  // this iteration's side-stream kernels (chd_k_kcopy, chd_k_curv, chd_k_hess_dur) may still read the slots' state
  CHD_CUDA(cudaStreamWaitEvent(b->stream, b->ev_copy, 0));
  if (b->out.terms) launch_cost_terms(b, 1);   // before admission overwrites the finished slots
  for (int s : freed)
    if ((rc = queue_harvest(b, s))) return rc;
  if (k == 0) return 0;
  if ((rc = queue_admit(b, freed.data(), k, first))) return rc;
  if (!q.claim) q.next += k;
  for (int j = 0; j < k; ++j) b->h_ipm[freed[j]].phase = CHD_PH_BEGIN;   // as the admission kernel left it
  *last_it = std::max(*last_it, it + 1 + b->sched_max_iter);
  return 0;
}

}  // namespace

extern "C" {

const char* chd_version(void) { return "libchd 0.1 (sm_90a)"; }

int chd_measure_fp64_peak(double* dfma_gflops, double* dmma_gflops) {
  int dev = 0, sms = 0;
  CHD_CUDA(cudaGetDevice(&dev));
  CHD_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  double* sink = nullptr;
  CHD_CUDA(cudaMalloc((void**)&sink, sizeof(double) * 1024));
  cudaEvent_t e0, e1;
  CHD_CUDA(cudaEventCreate(&e0));
  CHD_CUDA(cudaEventCreate(&e1));
  const int blocks = sms * 8, threads = 256, iters = 4096;
  for (int mode = 0; mode < 2; ++mode) {
    float best = 1e30f;
    for (int rep = 0; rep < 4; ++rep) {
      CHD_CUDA(cudaEventRecord(e0));
      chd_k_fp64_peak<<<blocks, threads>>>(mode, iters, sink);
      CHD_CUDA(cudaEventRecord(e1));
      CHD_CUDA(cudaEventSynchronize(e1));
      float ms = 0;
      CHD_CUDA(cudaEventElapsedTime(&ms, e0, e1));
      if (rep > 0 && ms < best) best = ms;
    }
    // mode 0: 8 independent FMA chains per thread; mode 1: 4 independent m16n8k8 accumulators per warp (2048 flop each)
    const double flop = mode == 0 ? (double)blocks * threads * iters * 8 * 2 : (double)blocks * (threads / 32) * iters * 4 * 2048;
    double* out = mode == 0 ? dfma_gflops : dmma_gflops;
    if (out) *out = flop / (best * 1e-3) / 1e9;
  }
  cudaEventDestroy(e0), cudaEventDestroy(e1), cudaFree(sink);
  return 0;
}

static int batch_create_impl(const chd_phys_problem* problems, int32_t batch, int32_t slots, const chd_phys_weights* weights,
                             int32_t device, const chd_phys_options& opt, chd_phys_batch* b);

// a batch (slots = 0) or a queue of `batch` clips through `slots` slots
static int create(const chd_phys_problem* problems, int32_t batch, int32_t slots, const chd_phys_weights* weights,
                  int32_t device, const chd_phys_options* opt, chd_phys_batch** out) {
  chd_phys_options o = {-1, nullptr, nullptr};
  if (opt) o = *opt;
  if (o.stage3_band_above < -1 || o.stage3_band_above > CHD_MAX_DUR) return -1;
  // a weight must be finite and not negative
  auto bad = [](const chd_phys_weights& w) {
    for (double v : {w.w_com_lin, w.w_com_ang, w.w_ee, w.w_smooth, w.w_dur})
      if (!std::isfinite(v) || v < 0.0) return true;
    return false;
  };
  if (o.clip_weights) {
    for (int i = 0; i < batch; ++i)
      if (bad(o.clip_weights[i])) return -1;
  } else if (weights && bad(*weights)) {
    return -1;
  }
  if (o.clip_options)
    for (int i = 0; i < batch; ++i)
      if (bad_options(o.clip_options[i])) return -1;
  chd_phys_batch* b = new chd_phys_batch();
  std::memset(&b->D, 0, sizeof(b->D));
  const int rc = batch_create_impl(problems, batch, slots, weights, device, o, b);
  if (rc) {
    chd_phys_batch_destroy(b);   // single cleanup path: streams, events, pooled allocations, host buffers
    return rc;
  }
  *out = b;
  return 0;
}

int chd_phys_batch_create(const chd_phys_problem* problems, int32_t batch, const chd_phys_weights* weights, int32_t device,
                          const chd_phys_options* opt, chd_phys_batch** out) {
  if (!problems || batch <= 0 || !out) return -1;
  return create(problems, batch, 0, weights, device, opt, out);
}

int chd_phys_queue_create(const chd_phys_problem* problems, int32_t n, int32_t slots, const chd_phys_weights* weights,
                          int32_t device, const chd_phys_options* opt, chd_phys_batch** out) {
  if (!problems || n <= 0 || slots <= 0 || !out) return -1;
  return create(problems, n, std::min(slots, n), weights, device, opt, out);
}

static int batch_create_impl(const chd_phys_problem* problems, int32_t batch, int32_t slots, const chd_phys_weights* weights,
                             int32_t device, const chd_phys_options& opt, chd_phys_batch* b) {
  const bool host_only = device == -2;  // layout tables only, no CUDA call (CPU-side tests of the host logic)
  if (device >= 0) CHD_CUDA(cudaSetDevice(device));
  chd_phys_weights w = {0.4, 1.7, 0.3, 0.1, 0.1};  // phys_optim.cpp:27-31
  if (weights) w = *weights;
  // one weight tuple per problem: the clip's own (chd_phys_options.clip_weights) or the batch's
  std::vector<chd_phys_weights> wv(batch, w);
  if (opt.clip_weights) wv.assign(opt.clip_weights, opt.clip_weights + batch);
  int rc = chd_build_layout(problems, batch, wv.data(), b->hb, opt.stage3_band_above);
  if (rc) return rc;
  ChdHostBatch& hb = b->hb;
  b->opts.resize(batch);
  b->ends.resize(batch);
  b->stages.resize(hb.stage.size());
  for (int i = 0; i < batch; ++i) {
    b->opts[i] = resolve_options(opt.clip_options ? opt.clip_options + i : nullptr, hb.stage.data() + (size_t)i * 6);
    b->ends[i] = stage_end(b->opts[i]);
    for (int s = 0; s < 6; ++s) b->stages[(size_t)i * 6 + s] = stage_dev(hb.stage[(size_t)i * 6 + s], s, b->opts[i]);
  }
  ChdDev& D = b->D;
  std::memset(&D, 0, sizeof(D));
  b->host_only = host_only;
  // a queue: the layout of all clips goes into the record store, the batch keeps `slots` rows of it
  if (slots && (rc = queue_pack(b, slots))) return rc;
  if (host_only) return 0;
  D.B = hb.B, D.S = hb.S, D.Pmax = hb.Pmax, D.n_max = hb.n_max, D.m_max = hb.m_max, D.slots_max = hb.slots_max;
  D.sets_max = hb.sets_max, D.tab_max = hb.tab_max, D.F_max = hb.F_max, D.Kd_max = hb.Kd_max, D.Kr_max = hb.Kr_max;
  D.Na_max = hb.Na_max, D.nb_max = hb.nb_max, D.w_max = hb.w_max, D.par_stride = hb.par_stride(), D.n_ee_max = hb.n_ee_max;
  D.fo_max = hb.fo_max, D.Ph_max = hb.Ph_max;
  CHD_CUDA(cudaStreamCreate(&b->stream));
  {
    // keep freed device memory in the default pool of this device (a batch object is created per solve by callers
    // that mirror the reference's one-process-per-clip flow)
    int dev_id = 0;
    cudaMemPool_t pool;
    CHD_CUDA(cudaGetDevice(&dev_id));
    CHD_CUDA(cudaDeviceGetDefaultMemPool(&pool, dev_id));
    unsigned long long keep = ~0ull;
    CHD_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
  }
  CHD_CUDA(cudaStreamCreateWithFlags(&b->copy_stream, cudaStreamNonBlocking));
  CHD_CUDA(cudaEventCreateWithFlags(&b->ev_kkt, cudaEventDisableTiming));
  CHD_CUDA(cudaEventCreateWithFlags(&b->ev_copy, cudaEventDisableTiming));
  CHD_CUDA(cudaEventCreateWithFlags(&b->ev_ls, cudaEventDisableTiming));
  CHD_CUDA(cudaEventCreate(&b->ev0));
  CHD_CUDA(cudaEventCreate(&b->ev1));
#define UP(field) if ((rc = dev_upload(b, hb.field, &D.field))) return rc;
#define UPM(field, T) if ((rc = dev_upload(b, hb.field, (const T**)&D.field))) return rc;
  UP(seq) UPM(poly_T, double) UPM(poly_tend, double) UP(node_const) UP(par) UP(t_dyn) UP(t_rom) UP(t_data) UP(row_lo) UP(row_hi) UP(node_var)
  UP(itab) UP(ent_ptr) UPM(ent_col, int) UP(ent_row) UP(col_ptr) UP(col_ent) UP(var_kkt) UP(row_kkt) UP(row_set) UP(sets) UPM(phase_tend, double)
  UP(dur0) UP(poly_ph)
  // pristine copies of what stage 3 rewrites + the line search's trial tables
  if ((rc = dev_upload(b, hb.poly_T, (const double**)&b->poly_T0))) return rc;
  if ((rc = dev_upload(b, hb.poly_tend, (const double**)&b->poly_tend0))) return rc;
  if ((rc = dev_upload(b, hb.phase_tend, (const double**)&b->phase_tend0))) return rc;
  if ((rc = dev_upload(b, hb.ent_col, (const int**)&b->ent_col0))) return rc;
  if ((rc = dev_upload(b, hb.poly_T, (const double**)&D.poly_Tt))) return rc;
  if ((rc = dev_upload(b, hb.poly_tend, (const double**)&D.poly_tendt))) return rc;
#undef UPM
#undef UP
  const size_t B = hb.B, nm = B * hb.n_max, mm = B * hb.m_max;
#define AL(field, cnt) if ((rc = dev_alloc(b, (cnt), &D.field))) return rc;
  AL(x, nm) AL(xt, nm) AL(jty, nm) AL(unobs, nm) AL(dx, nm) AL(grad, nm) AL(g, mm) AL(gt, mm) AL(Jv, B * hb.slots_max) AL(rflag, mm)
  AL(sc, mm) AL(dL, mm) AL(dU, mm) AL(s, mm) AL(y, mm) AL(zL, mm) AL(zU, mm) AL(ds, mm) AL(dy, mm) AL(dzL, mm) AL(dzU, mm)
  int dev = 0, sms = 0, smem_max = 0;
  CHD_CUDA(cudaGetDevice(&dev));
  CHD_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CHD_CUDA(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  cudaFuncAttributes fa_kkt, fa_gwin;
  CHD_CUDA(cudaFuncGetAttributes(&fa_kkt, chd_k_kkt));
  CHD_CUDA(cudaFuncGetAttributes(&fa_gwin, chd_k_kkt_gwin));
  const ChdKktPlan P = chd_kkt_plan(hb.Na_max, hb.nb_max, hb.w_max, hb.w_fix_max, hb.n_max, fa_kkt.sharedSizeBytes,
                                    fa_gwin.sharedSizeBytes, (size_t)smem_max);
  D.win_smem = P.win_smem, D.nbc_max = P.nbc_max, D.Q = P.Q, D.Qfix = P.Qfix, D.nbt = P.nbt, D.win_tiles = P.win_tiles;
  D.pan_doubles = P.pan_doubles, D.kstride = P.kstride, D.scratch_stride = P.scratch_stride;
  b->smem_kkt = P.smem_bytes;
  // CTAs per sequence: enough for four per SM over the whole batch, and at least one per 128 KB of band storage
  b->kcopy_blocks = (int)std::min<size_t>(512, std::max<size_t>(std::max<size_t>(1, 4 * (size_t)sms / B), P.kstride * sizeof(double) / 131072));
  AL(cost, B * 2) AL(Kwork, B * P.kstride) AL(Kbase, B * P.kstride) AL(sol, B * (size_t)(hb.Na_max + hb.nb_max)) AL(ipm, B)
  AL(rhs0, B * (size_t)(hb.Na_max + hb.nb_max)) AL(rhs1, B * (size_t)(hb.Na_max + hb.nb_max))
  if (P.scratch_stride) AL(scratch, B * P.scratch_stride)
#undef AL
  if ((rc = dev_upload(b, hb.x0, (const double**)&b->d_x0))) return rc;
  CHD_CUDA(cudaMemcpyAsync(D.x, b->d_x0, nm * sizeof(double), cudaMemcpyDeviceToDevice, b->stream));
  b->iter = chd_iter_form(hb.n_max, smem_max);
  if (P.status == CHD_KKT_TOO_WIDE_COMPACT || P.status == CHD_KKT_TOO_WIDE_PAIRS) {
    fprintf(stderr, "libchd: band + border too wide for the %s (Q=%d nbt=%d)\n",
            P.status == CHD_KKT_TOO_WIDE_COMPACT ? "compacted update loop" : "pair tables", P.Q, P.nbt);
    return -5;
  }
  if (P.status == CHD_KKT_TOO_LARGE) {
    fprintf(stderr, "libchd: KKT band + border too large for the shared memory of the factorisation (n_max=%d)\n", hb.n_max);
    return -5;
  }
  CHD_CUDA(cudaFuncSetAttribute(b->iter.eval, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)b->iter.smem_eval));
  CHD_CUDA(cudaFuncSetAttribute(P.win_smem ? chd_k_kkt : chd_k_kkt_gwin, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)b->smem_kkt));
  CHD_CUDA(cudaFuncSetAttribute(b->iter.linesearch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)b->iter.smem_ls));
  const size_t stride = sample_stride(hb);
  CHD_CUDA(cudaMallocAsync((void**)&b->d_samples, B * hb.fo_max * stride * sizeof(double), b->stream));
  CHD_CUDA(cudaMallocAsync((void**)&b->d_frames, B * sizeof(int), b->stream));
  b->allocs.push_back(b->d_samples);
  b->allocs.push_back(b->d_frames);
  b->h_ipm = (ChdIpm*)std::malloc(B * sizeof(ChdIpm));   // pageable: pinned allocation / release is slow per batch
  if (!b->h_ipm) return -3;
  // the stage rows (uploaded by every solve, set_schedule, and like them not counted in h2d_bytes) and behind them the
  // sequences' ChdStageEnd records
  const size_t rows_bytes = b->stages.size() * sizeof(ChdStageDev);
  CHD_CUDA(cudaMallocAsync((void**)&b->d_stages, rows_bytes + b->ends.size() * sizeof(ChdStageEnd), b->stream));
  b->allocs.push_back(b->d_stages);
  D.stages = b->d_stages;
  CHD_CUDA(cudaMemcpyAsync((char*)b->d_stages + rows_bytes, b->ends.data(), b->ends.size() * sizeof(ChdStageEnd),
                           cudaMemcpyHostToDevice, b->stream));
  if ((rc = dev_alloc(b, B * CHD_PHYS_N_TERMS, &b->d_terms))) return rc;
  if ((rc = dev_alloc(b, 3 * B * hb.fo_max * stride, &D.snapshots))) return rc;
  if (b->queue && (rc = queue_device(b, sms))) return rc;
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  return 0;
}

void chd_phys_batch_destroy(chd_phys_batch* b) {
  if (!b) return;
  if (b->stream) {
    for (void* p : b->allocs) cudaFreeAsync(p, b->stream);   // back to the pool, not to the driver (cudaFree synchronises the device)
    cudaStreamSynchronize(b->stream);
  }
  std::free(b->h_ipm);
  if (b->queue) {
    if (b->host_only) std::free(b->queue->store);
    else cudaFreeHost(b->queue->store), cudaFreeHost(b->queue->h_slot);
    delete b->queue;
  }
  if (b->ev0) cudaEventDestroy(b->ev0);
  if (b->ev1) cudaEventDestroy(b->ev1);
  if (b->ev_kkt) cudaEventDestroy(b->ev_kkt);
  if (b->ev_copy) cudaEventDestroy(b->ev_copy);
  if (b->ev_ls) cudaEventDestroy(b->ev_ls);
  if (b->copy_stream) cudaStreamDestroy(b->copy_stream);
  if (b->stream) cudaStreamDestroy(b->stream);
  delete b;
}

int chd_phys_get_dims(const chd_phys_batch* b, chd_phys_dims* d) {
  if (!b || !d) return -1;
  const ChdHostBatch& hb = b->hb;
  d->batch = hb.B, d->n_max = hb.n_max, d->m_max = hb.m_max, d->slots_max = hb.slots_max, d->n_splines = hb.S;
  d->p_max = hb.Pmax, d->sets_max = hb.sets_max, d->na_max = hb.Na_max, d->nb_max = hb.nb_max, d->w_max = hb.w_max;
  d->frames_out_max = hb.fo_max;
  return 0;
}
int chd_phys_get_sizes(const chd_phys_batch* b, int32_t* s) {
  if (!b || !s) return -1;
  for (int i = 0; i < b->hb.B; ++i) {
    const ChdSeq& h = b->hb.seq[i];
    s[6 * i + 0] = h.n, s[6 * i + 1] = h.m, s[6 * i + 2] = h.nslots, s[6 * i + 3] = h.Na, s[6 * i + 4] = h.nb, s[6 * i + 5] = h.w;
  }
  return 0;
}
int chd_phys_get_sizes_fixed(const chd_phys_batch* b, int32_t* s) {
  if (!b || !s) return -1;
  for (int i = 0; i < b->hb.B; ++i) s[3 * i] = b->hb.seq[i].nb_fix, s[3 * i + 1] = b->hb.seq[i].w_fix, s[3 * i + 2] = b->hb.seq[i].n_dur;
  return 0;
}
int chd_phys_get_x(const chd_phys_batch* b, double* x) {
  if (!b || !x || b->queue) return -1;
  if (b->host_only) {
    std::memcpy(x, b->hb.x0.data(), b->hb.x0.size() * sizeof(double));
    return 0;
  }
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  CHD_CUDA(cudaMemcpy(x, b->D.x, (size_t)b->hb.B * b->hb.n_max * sizeof(double), cudaMemcpyDeviceToHost));
  return 0;
}
int chd_phys_set_x(chd_phys_batch* b, const double* x) {
  if (!b || !x || b->host_only || b->queue) return -1;
  CHD_CUDA(cudaMemcpy(b->D.x, x, (size_t)b->hb.B * b->hb.n_max * sizeof(double), cudaMemcpyHostToDevice));
  chd_k_tables<<<b->hb.B, 64, 0, b->stream>>>(b->D);   // spline tables follow the durations held in x
  b->launches++;
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  return 0;
}

int chd_phys_eval(chd_phys_batch* b, int32_t stage, double* cost, double* grad, double* g, double* jac_vals) {
  if (!b || stage < 0 || stage > 5 || b->host_only || b->queue) return -1;
  const ChdHostBatch& hb = b->hb;
  int sched[1] = {stage};
  int rc = set_schedule(b, sched, 1, -1, 0);
  if (rc) return rc;
  {
    Timer t(b, KT_INIT);
    chd_k_stage_begin<<<hb.B, CHD_THREADS, 0, b->stream>>>(b->D);
  }
  launch_eval(b);
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  CHD_CUDA(cudaGetLastError());
  const size_t B = hb.B;
  if (cost) {
    std::vector<double> c2(2 * B);
    CHD_CUDA(cudaMemcpy(c2.data(), b->D.cost, 2 * B * sizeof(double), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < B; ++i) cost[i] = c2[2 * i];
  }
  if (grad) CHD_CUDA(cudaMemcpy(grad, b->D.grad, B * hb.n_max * sizeof(double), cudaMemcpyDeviceToHost));
  if (g) CHD_CUDA(cudaMemcpy(g, b->D.g, B * hb.m_max * sizeof(double), cudaMemcpyDeviceToHost));
  if (jac_vals) CHD_CUDA(cudaMemcpy(jac_vals, b->D.Jv, B * hb.slots_max * sizeof(double), cudaMemcpyDeviceToHost));
  return 0;
}

int chd_phys_get_layout(const chd_phys_batch* b, int32_t* ent_ptr, int32_t* ent_col, double* row_lo, double* row_hi,
                        int32_t* row_set, int32_t* var_kkt, int32_t* row_kkt) {
  if (!b) return -1;
  const ChdHostBatch& hb = b->hb;
  if (ent_ptr) std::memcpy(ent_ptr, hb.ent_ptr.data(), hb.ent_ptr.size() * sizeof(int));
  if (ent_col) std::memcpy(ent_col, hb.ent_col.data(), hb.ent_col.size() * sizeof(int));
  if (row_lo) std::memcpy(row_lo, hb.row_lo.data(), hb.row_lo.size() * sizeof(double));
  if (row_hi) std::memcpy(row_hi, hb.row_hi.data(), hb.row_hi.size() * sizeof(double));
  if (row_set) std::memcpy(row_set, hb.row_set.data(), hb.row_set.size() * sizeof(int));
  if (var_kkt) std::memcpy(var_kkt, hb.var_kkt.data(), hb.var_kkt.size() * sizeof(int));
  if (row_kkt) std::memcpy(row_kkt, hb.row_kkt.data(), hb.row_kkt.size() * sizeof(int));
  return 0;
}

int chd_phys_get_slot_index(const chd_phys_batch* b, int32_t* ent_row, int32_t* col_ptr, int32_t* col_ent) {
  if (!b) return -1;
  const ChdHostBatch& hb = b->hb;
  if (ent_row) std::memcpy(ent_row, hb.ent_row.data(), hb.ent_row.size() * sizeof(int));
  if (col_ptr) std::memcpy(col_ptr, hb.col_ptr.data(), hb.col_ptr.size() * sizeof(int));
  if (col_ent) std::memcpy(col_ent, hb.col_ent.data(), hb.col_ent.size() * sizeof(int));
  return 0;
}

int chd_phys_get_ent_col(const chd_phys_batch* b, int32_t* ent_col) {
  if (!b || !ent_col) return -1;
  if (b->host_only) {
    std::memcpy(ent_col, b->hb.ent_col.data(), b->hb.ent_col.size() * sizeof(int));
    return 0;
  }
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  CHD_CUDA(cudaMemcpy(ent_col, b->D.ent_col, b->hb.ent_col.size() * sizeof(int), cudaMemcpyDeviceToHost));
  return 0;
}

int chd_phys_get_duals(const chd_phys_batch* b, double* y, double* zL, double* zU, double* s, double* row_scale, double* obj_scale) {
  if (!b || b->host_only || b->queue) return -1;
  const size_t B = b->hb.B, mm = B * b->hb.m_max;
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  if (y) CHD_CUDA(cudaMemcpy(y, b->D.y, mm * sizeof(double), cudaMemcpyDeviceToHost));
  if (zL) CHD_CUDA(cudaMemcpy(zL, b->D.zL, mm * sizeof(double), cudaMemcpyDeviceToHost));
  if (zU) CHD_CUDA(cudaMemcpy(zU, b->D.zU, mm * sizeof(double), cudaMemcpyDeviceToHost));
  if (s) CHD_CUDA(cudaMemcpy(s, b->D.s, mm * sizeof(double), cudaMemcpyDeviceToHost));
  if (row_scale) CHD_CUDA(cudaMemcpy(row_scale, b->D.sc, mm * sizeof(double), cudaMemcpyDeviceToHost));
  if (obj_scale) {
    std::vector<ChdIpm> ipm(B);
    CHD_CUDA(cudaMemcpy(ipm.data(), b->D.ipm, B * sizeof(ChdIpm), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < B; ++i) obj_scale[i] = ipm[i].sf;
  }
  return 0;
}

int chd_phys_stage_stats(const chd_phys_batch* b, double* stats) {
  if (!b || !stats || b->host_only || !b->h_ipm) return -1;
  const int B = b->hb.B;
  for (int s = 0; s < 6; ++s)
    for (int i = 0; i < B; ++i)
      for (int q = 0; q < 4; ++q) stats[((size_t)s * B + i) * 4 + q] = b->h_ipm[i].st_stat[s][q];
  return 0;
}

int chd_phys_solve_stage(chd_phys_batch* b, int32_t stage, int32_t max_iter, int32_t* status, int32_t* iters, double* stats) {
  if (!b || stage < 0 || stage > 5 || b->host_only || b->queue) return -1;
  const int B = b->hb.B;
  int sched[1] = {stage};
  int rc = set_schedule(b, sched, 1, stage, max_iter);
  if (rc) return rc;
  if ((rc = run_schedule(b))) return rc;
  for (int i = 0; i < B; ++i) {
    const ChdIpm& I = b->h_ipm[i];
    if (status) status[i] = I.st_status[stage];
    if (iters) iters[i] = I.st_iters[stage];
    if (stats) {
      double* s = stats + 8 * i;
      s[0] = I.f, s[1] = I.E0, s[2] = I.viol_u, s[3] = I.dual_u, s[4] = I.compl_u, s[5] = I.mu, s[6] = I.delta_w, s[7] = I.ls_fail;
    }
    if (i == 0 && getenv("CHD_PROF")) fprintf(stderr, "chd prof (Mcycles) seq0 stage %d: err %.2f asm %.2f factor %.2f border %.2f back %.2f rec %.2f | factor (c): diag %.2f upd %.2f\n", stage, I.prof[0]/1e6, I.prof[1]/1e6, I.prof[2]/1e6, I.prof[3]/1e6, I.prof[4]/1e6, I.prof[5]/1e6, I.prof[6]/1e6, I.prof[7]/1e6);
  }
  return 0;
}

int chd_phys_sample_device(chd_phys_batch* b, double* out_device, void* stream) {
  if (!b || !out_device || b->host_only || b->queue) return -1;
  cudaStream_t st = stream ? (cudaStream_t)stream : b->stream;
  if (st == b->stream) {
    Timer t(b, KT_SAMPLE);
    chd_k_sample<<<b->hb.B, 128, 0, st>>>(b->D, out_device, b->d_frames);
    return 0;
  }
  // caller's stream: order the launch behind everything pending on the batch's own stream (reset / upload copies, the
  // solve) and make the batch's stream wait for it in turn (it writes d_frames and reads x)
  cudaEvent_t ev;
  CHD_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  CHD_CUDA(cudaEventRecord(ev, b->stream));
  CHD_CUDA(cudaStreamWaitEvent(st, ev, 0));
  chd_k_sample<<<b->hb.B, 128, 0, st>>>(b->D, out_device, b->d_frames);
  CHD_CUDA(cudaEventRecord(ev, st));
  CHD_CUDA(cudaStreamWaitEvent(b->stream, ev, 0));
  CHD_CUDA(cudaEventDestroy(ev));
  return 0;
}

int chd_phys_sample(chd_phys_batch* b, double* out, int32_t* frames_out) {
  if (!b || !out || b->host_only || b->queue) return -1;
  const ChdHostBatch& hb = b->hb;
  const size_t cnt = (size_t)hb.B * hb.fo_max * sample_stride(hb);
  CHD_CUDA(cudaMemsetAsync(b->d_samples, 0, cnt * sizeof(double), b->stream));
  int rc = chd_phys_sample_device(b, b->d_samples, nullptr);
  if (rc) return rc;
  CHD_CUDA(cudaMemcpyAsync(out, b->d_samples, cnt * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
  if (frames_out) CHD_CUDA(cudaMemcpyAsync(frames_out, b->d_frames, hb.B * sizeof(int), cudaMemcpyDeviceToHost, b->stream));
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  return 0;
}

// Staged schedule of phys_optim.cpp:554-749.  Every sequence walks through 1.1, 1.2, 2.1, 2.2, 3 and -- only when its
// stage 3 did not succeed (:713-749) -- 4 at its own pace (converged sequences do not wait for the slowest one of
// their stage).  Stage status -9 = stage not run (stage 4 after a successful stage 3), -3 = stage 3 not attempted
// (more phase durations than CHD_MAX_DUR with the switch times in the border, or a banded layout too wide).
int chd_phys_solve(chd_phys_batch* b, double* samples, int32_t* frames_out, int32_t* success, int32_t* stage_status,
                   int32_t* stage_iters) {
  if (!b || b->host_only || b->queue) return -1;
  const ChdHostBatch& hb = b->hb;
  const int B = hb.B;
  const size_t snap = (size_t)B * hb.fo_max * sample_stride(hb);
  int rc = set_schedule(b, full_schedule, 6, -1, 0);
  if (rc) return rc;
  b->out = {(size_t)B, samples, nullptr, b->terms_out, frames_out, success, stage_status, stage_iters};
  const ChdSolveOut& o = b->out;
  if (o.samples) CHD_CUDA(cudaMemsetAsync(b->D.snapshots, 0, 3 * snap * sizeof(double), b->stream));
  if ((rc = run_schedule(b))) return rc;
  for (int i = 0; i < B; ++i) write_status(o, i, b->h_ipm[i]);
  // one copy of every sequence's snapshots, frame counts and cost terms
  if (o.samples) CHD_CUDA(cudaMemcpyAsync(o.samples, b->D.snapshots, 3 * snap * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
  if (o.frames) CHD_CUDA(cudaMemcpyAsync(o.frames, b->d_frames, B * sizeof(int), cudaMemcpyDeviceToHost, b->stream));
  if (o.terms) {   // x is every sequence's final iterate, the one of the durations snapshot
    launch_cost_terms(b, 0);
    CHD_CUDA(cudaMemcpyAsync(o.terms, b->d_terms, (size_t)B * CHD_PHYS_N_TERMS * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
  }
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  for (int i = 0; i < B; ++i) write_untaken(o, i, b->opts[i].last_stage, hb.fo_max * sample_stride(hb));
  return 0;
}

// Queue of n clips through the batch's slots: every clip is admitted in queue order into the first free slot, and a
// slot is refilled at the check point after its clip finished.  Outputs as chd_phys_solve's, indexed by clip.  With a
// claim source only the clips it hands out are admitted and written.
int chd_phys_queue_solve(chd_phys_batch* b, double* samples, int32_t* frames_out, int32_t* success, int32_t* stage_status,
                         int32_t* stage_iters, double* stage_stats) {
  if (!b || b->host_only || !b->queue) return -1;
  ChdQueue& q = *b->queue;
  const int S = b->hb.B;
  int rc, first = 0, k = S;
  q.exhausted = false;
  if (q.claim) {
    q.given.assign(q.n, 0);
    if ((rc = queue_claim(b, S, &first, &k))) return rc;
    if (k == 0) return 0;   // nothing for this handle: no output is touched
  }
  if ((rc = set_schedule(b, full_schedule, 6, -1, 0))) return rc;
  b->out = {(size_t)q.n, samples, stage_stats, b->terms_out, frames_out, success, stage_status, stage_iters};
  q.clip.assign(S, -1);
  std::vector<int> slots(S);
  std::iota(slots.begin(), slots.end(), 0);
  if ((rc = queue_admit(b, slots.data(), k, first))) return rc;
  q.next = k;
  if (k < S) {
    // slots the claim source left empty: finished from the start, so every kernel passes over them
    std::vector<ChdIpm> idle(S - k);
    std::memset(idle.data(), 0, idle.size() * sizeof(ChdIpm));
    for (ChdIpm& I : idle) I.phase = CHD_PH_FINISHED, I.snap = -1;
    CHD_CUDA(cudaMemcpyAsync(b->D.ipm + k, idle.data(), idle.size() * sizeof(ChdIpm), cudaMemcpyHostToDevice, b->stream));
    b->h2d_bytes += (int64_t)(idle.size() * sizeof(ChdIpm));
  }
  if ((rc = run_schedule(b))) return rc;
  if (b->out.terms) launch_cost_terms(b, 0);
  for (int i = 0; i < S; ++i)
    if ((rc = queue_harvest(b, i))) return rc;
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  return 0;
}

int chd_phys_queue_set_claim(chd_phys_batch* b, chd_phys_claim_fn* claim, void* ctx) {
  if (!b || !b->queue) return -1;
  b->queue->claim = claim, b->queue->claim_ctx = claim ? ctx : nullptr;
  return 0;
}

int chd_phys_get_stage_weights(const chd_phys_batch* b, double* w) {
  if (!b || !w) return -1;
  for (const ChdStageDev& s : b->stages) {
    for (int q = 0; q < 3; ++q) w[q] = s.w_data[q], w[3 + q] = s.w_vel[q], w[6 + q] = s.w_acc[q];
    w[9] = s.w_dur;
    w += 10;
  }
  return 0;
}

int chd_phys_get_solver_options(const chd_phys_batch* b, chd_phys_solver_options* opts) {
  if (!b || !opts) return -1;
  std::copy(b->opts.begin(), b->opts.begin() + b->hb.B, opts);
  return 0;
}

int chd_phys_cost_terms(chd_phys_batch* b, double* terms) {
  if (!b || !terms || b->host_only || b->queue) return -1;
  launch_cost_terms(b, 0);
  CHD_CUDA(cudaMemcpyAsync(terms, b->d_terms, (size_t)b->hb.B * CHD_PHYS_N_TERMS * sizeof(double), cudaMemcpyDeviceToHost, b->stream));
  CHD_CUDA(cudaStreamSynchronize(b->stream));
  CHD_CUDA(cudaGetLastError());
  return 0;
}

int chd_phys_set_cost_terms_out(chd_phys_batch* b, double* terms) {
  if (!b || b->host_only) return -1;
  b->terms_out = terms;
  return 0;
}

int64_t chd_phys_launch_count(const chd_phys_batch* b) { return b ? b->launches : 0; }
int64_t chd_phys_h2d_bytes(const chd_phys_batch* b) { return b ? b->h2d_bytes : 0; }
int chd_phys_reset(chd_phys_batch* b) {
  if (!b || b->host_only || b->queue) return -1;
  CHD_CUDA(cudaMemcpyAsync(b->D.x, b->d_x0, (size_t)b->hb.B * b->hb.n_max * sizeof(double), cudaMemcpyDeviceToDevice, b->stream));
  // the input durations are back: host-built spline tables and Jacobian columns
  const ChdHostBatch& hb = b->hb;
  CHD_CUDA(cudaMemcpyAsync(b->D.poly_T, b->poly_T0, hb.poly_T.size() * sizeof(double), cudaMemcpyDeviceToDevice, b->stream));
  CHD_CUDA(cudaMemcpyAsync(b->D.poly_tend, b->poly_tend0, hb.poly_tend.size() * sizeof(double), cudaMemcpyDeviceToDevice, b->stream));
  CHD_CUDA(cudaMemcpyAsync(b->D.phase_tend, b->phase_tend0, hb.phase_tend.size() * sizeof(double), cudaMemcpyDeviceToDevice, b->stream));
  CHD_CUDA(cudaMemcpyAsync(b->D.ent_col, b->ent_col0, hb.ent_col.size() * sizeof(int), cudaMemcpyDeviceToDevice, b->stream));
  chd_k_clear_dyn<<<(hb.B + 127) / 128, 128, 0, b->stream>>>(b->D);
  b->launches++;
  return 0;
}
int chd_phys_set_timing(chd_phys_batch* b, int enable) {
  if (!b) return -1;
  b->timing = enable;
  return 0;
}
int chd_phys_kernel_times(chd_phys_batch* b, double* ms8, int64_t* launches8, int reset) {
  if (!b) return -1;
  for (int i = 0; i < KT_N; ++i) {
    if (ms8) ms8[i] = b->kt_ms[i];
    if (launches8) launches8[i] = b->kt_n[i];
    if (reset) b->kt_ms[i] = 0, b->kt_n[i] = 0;
  }
  return 0;
}

}  // extern "C"
