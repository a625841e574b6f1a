/* libchd -- C ABI of the H100-native batched physics-based trajectory optimiser and foot-contact
 * classifier (drop-in for the hot path of davrempe/contact-human-dynamics).
 *
 * Every entry point is plain C: pointers + sizes, int return (0 = ok, negative = error), no exceptions
 * cross the boundary, no ownership transfer unless stated.  Host pointers are marked [host], device
 * pointers [device].  All floating point is IEEE fp64 unless the name says otherwise.
 *
 * Reference interfaces replaced (paths relative to the reference repo):
 *   chd_phys_batch_create   <- towr_phys_optim/phys_optim.cpp:380-552  (Read*Info + NlpFormulation::
 *                              GetVariableSets / GetConstraints, src/nlp_formulation.cpp:79-360)
 *   chd_phys_solve          <- phys_optim.cpp:554-749  (the five/six staged ifopt::IpoptSolver::Solve calls)
 *   chd_phys_eval           <- ifopt ConstraintSet::GetValues / FillJacobianBlock and CostTerm::GetCost /
 *                              FillJacobianBlock as implemented in towr_phys_optim/src/{constraints,costs,models}
 *   chd_phys_sample         <- SaveSolution, phys_optim.cpp:63-143
 *   chd_contact_*           <- src/contact_learning/test.py:51-152 (val_full_video) +
 *                              src/contact_learning/models/openpose_only.py:29-78
 */
#ifndef CHD_H_
#define CHD_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* One sequence's inputs, i.e. what phys_optim reads from skel_info.txt, motion_info.txt,
 * terrain_info.txt and contact_info.txt (phys_optim.cpp:155-267).  End-effector order is the solver's:
 * L toe, R toe, L heel, R heel (phys_optim.cpp:491-513).  All pointers [host]. */
typedef struct chd_phys_problem {
  int32_t n_frames;            /* --nframes */
  int32_t n_ee;                /* 2 (toes only) or 4 (reference: always 4, phys_optim.cpp:432) */
  double dt;
  const double* hip_left;      /* n_frames x 3 */
  const double* hip_right;     /* n_frames x 3 */
  double max_leg_length, max_heel_length, heel_dist, body_mass;
  const double* inertia;       /* n_frames x 6: Ixx Iyy Izz Ixy Ixz Iyz */
  const double* base_lin;      /* n_frames x 3 */
  const double* base_ang;      /* n_frames x 3 */
  const double* ee_pos;        /* n_ee x n_frames x 3 */
  double floor_normal[3], floor_point[3];
  const int32_t* ee_start_contact; /* n_ee */
  const int32_t* ee_n_phases;      /* n_ee */
  const double* ee_durations;      /* concatenated, sum(ee_n_phases) */
} chd_phys_problem;

/* gflags of phys_optim.cpp:27-31 */
typedef struct chd_phys_weights {
  double w_com_lin, w_com_ang, w_ee, w_smooth, w_dur;
} chd_phys_weights;

typedef struct chd_phys_batch chd_phys_batch;

/* Stage ids (phys_optim.cpp:554-749): 0 = 1.1, 1 = 1.2, 2 = 2.1, 3 = 2.2, 4 = 3, 5 = 4. */
enum { CHD_ST_11 = 0, CHD_ST_12 = 1, CHD_ST_21 = 2, CHD_ST_22 = 3, CHD_ST_3 = 4, CHD_ST_4 = 5 };

/* Sizes of the padded batch (strides of every per-sequence array below). */
typedef struct chd_phys_dims {
  int32_t batch, n_max, m_max, slots_max, n_splines, p_max, sets_max, na_max, nb_max, w_max, frames_out_max;
} chd_phys_dims;

/* Layout options of chd_phys_batch_create.
 *   stage3_band_above: a sequence with more phase-duration variables than this carries its switch times as banded
 *   KKT unknowns (time ordered with the node values) instead of dense border unknowns, which lifts the limit of 96
 *   that stage 3 otherwise has.  -1: no sequence (the default); 0 .. 96 otherwise.  A banded sequence whose band would
 *   be too wide for the KKT kernels keeps stage 3 off (status -3).
 *   clip_weights: NULL (the default), or [host] one weight tuple per problem (`batch` entries for a batch, `n` for a
 *   queue), which overrides the `weights` argument: each sequence runs stages 2.1, 2.2, 3 and 4 with its own weights
 *   (stages 1.1 and 1.2 have fixed ones).  A sequence's results are those of a batch of the same problems that all use
 *   its tuple.  Read during creation only.
 *   clip_options: NULL (the defaults), or [host] one record of solver options per problem, indexed like clip_weights.
 *   Read during creation only. */

/* The last stage a clip runs (chd_phys_solver_options.last_stage), named after the SaveSolution snapshot it ends with. */
enum { CHD_LAST_NO_DYNAMICS = 0, CHD_LAST_DYNAMICS = 1, CHD_LAST_DURATIONS = 2 };
/* Solver options of one clip.
 *   tol, constr_viol_tol, dual_inf_tol, compl_inf_tol: IPOPT's termination tolerances, used by every stage of the clip
 *   (a stage has converged when the scaled NLP error <= tol and the unscaled constraint violation, dual infeasibility
 *   and complementarity are within the other three; the feasibility polish and mu_min = min(tol, compl_inf_tol) / 11
 *   use them too).  Defaults 1e-3 (phys_optim.cpp:578), 1e-4, 1.0, 1e-4.  Each must be finite and > 0.
 *   max_iter: iteration cap of stages 1.1, 1.2, 2.1, 2.2, 3, 4; 0 = the stage's cap in phys_optim.cpp (7000, 7000, 7000,
 *   2500, 2000, 7000).  Not negative.
 *   last_stage: CHD_LAST_NO_DYNAMICS stops the clip after stage 1.2, CHD_LAST_DYNAMICS after stage 2.2,
 *   CHD_LAST_DURATIONS (the default) runs the whole schedule (stage 4 when stage 3 did not succeed).  The stages a clip
 *   does not run report status -9 and 0 iterations, and the snapshots it does not take are NaN in `samples`. */
typedef struct chd_phys_solver_options {
  double tol, constr_viol_tol, dual_inf_tol, compl_inf_tol;
  int32_t max_iter[6];
  int32_t last_stage;
} chd_phys_solver_options;
typedef struct chd_phys_options {
  int32_t stage3_band_above;
  const chd_phys_weights* clip_weights;
  const chd_phys_solver_options* clip_options;
} chd_phys_options;
/* Builds the NLP layouts of `batch` sequences on the host and uploads them to the current CUDA device.
 * device < 0 keeps the current device.  weights and opt may be NULL: the defaults.  Returns -1 for a bad argument, an
 * option out of range, a weight that is negative or not finite or a bad solver option (a tolerance not finite or not
 * > 0, a negative cap, an unknown last_stage; all checked before any device work), -5 when the batch's
 * KKT band + border does not fit the factorisation kernels.  The length of a sequence is not limited otherwise:
 * iterates too long for shared memory are evaluated from global memory. */
int chd_phys_batch_create(const chd_phys_problem* problems, int32_t batch, const chd_phys_weights* weights,
                          int32_t device, const chd_phys_options* opt, chd_phys_batch** out);
void chd_phys_batch_destroy(chd_phys_batch* b);
int chd_phys_get_dims(const chd_phys_batch* b, chd_phys_dims* dims);
/* Per-sequence sizes: n (variables: node values, then the P-1 free phase durations of every foot), m (master rows),
 * nslots, Na, nb (border unknowns, incl. the switch times unless they are banded), w -- six int32 per sequence [host]. */
int chd_phys_get_sizes(const chd_phys_batch* b, int32_t* sizes6);
/* What the fixed-duration stages (all but stage 3) work with: border unknowns without the switch times, half bandwidth
 * of the static pattern, and the number of phase-duration variables (0: stage 3 not available) -- three int32 per
 * sequence [host].  With banded switch times (chd_phys_options) the first equals nb. */
int chd_phys_get_sizes_fixed(const chd_phys_batch* b, int32_t* sizes3);

/* Current iterate x: batch x n_max doubles.  [host] copies (synchronous). */
int chd_phys_get_x(const chd_phys_batch* b, double* x_host);
int chd_phys_set_x(chd_phys_batch* b, const double* x_host);

/* Function-level evaluation at the current x for `stage` (selects active rows and cost weights):
 *   cost[batch], grad[batch x n_max], g[batch x m_max] (master row order, inactive rows = 0),
 *   jac_vals[batch x slots_max] (block-row slots; columns via chd_phys_get_layout).  Any output may be NULL.
 * All outputs [host]. */
int chd_phys_eval(chd_phys_batch* b, int32_t stage, double* cost, double* grad, double* g, double* jac_vals);

/* Static layout tables, [host] outputs, any may be NULL:
 *   ent_ptr[batch x (m_max+1)], ent_col[batch x slots_max] (variable index or -1),
 *   row_lo / row_hi [batch x m_max], row_set[batch x m_max] (constraint-set type of each row),
 *   var_kkt[batch x n_max], row_kkt[batch x m_max] (KKT ordering; -1 = not an unknown). */
int chd_phys_get_layout(const chd_phys_batch* b, int32_t* ent_ptr, int32_t* ent_col, double* row_lo, double* row_hi,
                        int32_t* row_set, int32_t* var_kkt, int32_t* row_kkt);
/* Column-oriented view of the same Jacobian slots (what ifopt keeps as a column-compressed Eigen matrix,
 * ifopt::Composite::GetJacobian): ent_row[batch x slots_max] (row of every slot), col_ptr[batch x (n_max+1)],
 * col_ent[batch x slots_max] (slots grouped by variable).  [host] outputs, any may be NULL. */
int chd_phys_get_slot_index(const chd_phys_batch* b, int32_t* ent_row, int32_t* col_ptr, int32_t* col_ent);

/* Jacobian slot columns as they stand on the device: equal to chd_phys_get_layout's ent_col until stage 3 moves a
 * phase duration; from then on the polynomial active at a sample time is located at run time and the node / switch-time
 * columns of the time-located rows are rewritten by every evaluation.  Column index of a duration variable d_k = the
 * switch time tau_k = d_0 + ... + d_k the solver works with (derivatives are with respect to tau). [host] output. */
int chd_phys_get_ent_col(const chd_phys_batch* b, int32_t* ent_col);
/* Interior-point state of the last solved stage, master row order, batch x m_max each [host], any may be NULL:
 * constraint multipliers y, bound multipliers zL / zU of the slacks, slacks s (all of the scaled problem
 * min obj_scale * f  s.t.  row_scale * g(x) - s = 0), the row scaling and obj_scale[batch]
 * (what IpoptCalculatedQuantities reports as the scaled multipliers; unscaled y = y * row_scale / obj_scale). */
int chd_phys_get_duals(const chd_phys_batch* b, double* y, double* zL, double* zU, double* s, double* row_scale,
                       double* obj_scale);
/* Cost weights of every sequence's six stages as the solver uses them: [host] batch x 6 x 10 doubles, per stage
 * w_data (base lin, base ang, feet), w_vel (same order), w_acc (same order), w_dur.  A queue handle: of its first
 * `slots` clips, like the other layout queries.  Works on host-only layouts. */
int chd_phys_get_stage_weights(const chd_phys_batch* b, double* w);
/* Solver options of every sequence as the solver uses them, the defaults resolved (every cap the stage's own):
 * opts [host] batch records.  A queue handle: of its first `slots` clips, like the other layout queries.  Works on
 * host-only layouts. */
int chd_phys_get_solver_options(const chd_phys_batch* b, chd_phys_solver_options* opts);

/* The unweighted cost terms at the current x: terms [host] batch x CHD_PHYS_N_TERMS doubles, per sequence
 *   0-2 data fit (data_cost.cpp) of the base position, the base orientation, the feet (summed over end-effectors),
 *   3-5 velocity smoothing (vel_smooth_cost.cpp, position differences) in the same order,
 *   6-8 acceleration smoothing (velocity differences) in the same order,
 *   9   duration change (duration_cost.cpp; 0 for a sequence without free phase durations),
 * each with weight 1, all ten whatever the stage (after stage 3, on the spline tables of the moved durations).  So
 * the cost chd_phys_eval reports for a stage is the sum of these terms times that stage's weights
 * (chd_phys_get_stage_weights).  A sequence's terms are bitwise the same from call to call.  -1 on a queue handle. */
enum { CHD_PHYS_N_TERMS = 10 };
int chd_phys_cost_terms(chd_phys_batch* b, double* terms);
/* Opt-in: every later chd_phys_solve / chd_phys_queue_solve also writes each clip's cost terms (chd_phys_cost_terms) at
 * its final iterate, the one of the durations snapshot, to terms [host] batch (a queue: n) x CHD_PHYS_N_TERMS, indexed
 * like the other outputs (a queue takes them from a finished slot before its next clip is admitted).  NULL, the
 * default, turns it off; a solve then issues no extra launch or copy.  The buffer must stay valid while solves run. */
int chd_phys_set_cost_terms_out(chd_phys_batch* b, double* terms);

/* Residuals of every stage of the last chd_phys_solve / chd_phys_solve_stage: stats [host] 6 x batch x 4 =
 * objective, scaled NLP error E0 (IPOPT's overall error, tol 1e-3), unscaled max constraint violation
 * (constr_viol_tol 1e-4), unscaled dual infeasibility. */
int chd_phys_stage_stats(const chd_phys_batch* b, double* stats);

/* Runs the interior-point solve of one stage for every sequence (warm start from the current x).
 * status[batch] [host]: 0 = converged (IPOPT "Solve_Succeeded" test), -1 = iteration cap, -2 = numerical failure.
 * iters[batch] [host], stats[batch x 8] [host]: f, E0, unscaled constraint violation, unscaled dual inf,
 * unscaled complementarity, mu, delta_w, #line-search failures.  Outputs may be NULL. */
int chd_phys_solve_stage(chd_phys_batch* b, int32_t stage, int32_t max_iter, int32_t* status, int32_t* iters,
                         double* stats);

/* Whole staged schedule of phys_optim.cpp:554-749 for the batch.  `samples` [host]:
 * 3 x batch x frames_out_max x (6 + 7*n_ee_max) doubles = the three SaveSolution snapshots
 * (no_dynamics, dynamics, durations), frames_out[batch] [host] = frames per sequence,
 * success[batch x 2] [host] = (dynamics_succeed, durations_succeed) of success_log.txt.
 * stage_status [host, 6 x batch] / stage_iters [host, 6 x batch] may be NULL; status -9 = stage not run (stage 4 after a
 * successful stage 3, phys_optim.cpp:713, or a stage after the sequence's last_stage, whose snapshots are then NaN,
 * see chd_phys_solver_options), -3 = stage 3 not attempted (more than 96 phase durations and the switch
 * times not banded, see chd_phys_options, or a banded layout too wide for the KKT kernels). */
int chd_phys_solve(chd_phys_batch* b, double* samples, int32_t* frames_out, int32_t* success,
                   int32_t* stage_status, int32_t* stage_iters);

/* SaveSolution sampling of the current x: out [host] batch x frames_out_max x (6+7*n_ee_max). */
int chd_phys_sample(chd_phys_batch* b, double* out, int32_t* frames_out);

/* Device-resident variant of the sampler for the multi-GPU gather: writes into a caller-provided
 * [device] buffer (e.g. an NCCL send buffer) on the given stream (cudaStream_t passed as void*). */
int chd_phys_sample_device(chd_phys_batch* b, double* out_device, void* stream);

/* Physics solve queue: n clips solved through `slots` sequences of one batch (slots is clamped to n).  The layout is
 * built once over all n clips, so every clip fits every slot and chd_phys_get_dims reports the strides of a batch of
 * the n clips with batch = slots: outputs are sized n x frames_out_max x stride.  Device memory scales with slots.
 * Returns -1 for n <= 0, slots <= 0, problems or out NULL or an option out of range, -5 as chd_phys_batch_create.
 * On a queue handle the calls that address slots (get_x, set_x, eval, solve_stage, solve, sample, sample_device,
 * reset, get_duals) return -1; the layout queries describe the first `slots` clips; the instrumentation calls work,
 * chd_phys_h2d_bytes includes the uploads of every admission and chd_phys_kernel_times' entry 5 times them. */
int chd_phys_queue_create(const chd_phys_problem* problems, int32_t n, int32_t slots, const chd_phys_weights* weights,
                          int32_t device, const chd_phys_options* opt, chd_phys_batch** out);
/* The staged schedule of chd_phys_solve for every clip of the queue.  The first `slots` clips start in slots 0, 1, ...;
 * whenever a slot's clip has finished (checked every 8 iterations) the next clip in queue order takes it, a refilled
 * slot being the same to the solver as that row of a new batch.  Outputs [host] as chd_phys_solve's plus
 * stage_stats (chd_phys_stage_stats' 6 x n x 4 block), indexed by clip (n, not slots); any may be NULL.  A clip's
 * results are those of a chd_phys_batch_create batch of the same n clips.  Calling it again starts the queue over.
 * With a claim source set (chd_phys_queue_set_claim) the clips come from it instead: only the clips it hands out are
 * solved and written, the rows of the others are left as they were.  Returns -1 if the source fails or misbehaves. */
int chd_phys_queue_solve(chd_phys_batch* b, double* samples, int32_t* frames_out, int32_t* success, int32_t* stage_status,
                         int32_t* stage_iters, double* stage_stats);

/* Hands out queue positions: writes the first of k consecutive positions to *first and returns k (0 <= k <= want);
 * 0 = nothing left, negative = error.  Called on the host thread inside chd_phys_queue_solve. */
typedef int32_t(chd_phys_claim_fn)(void* ctx, int32_t want, int32_t* first);
/* Lets a claim source decide which clips of the queue this handle solves, e.g. a counter shared by several processes
 * that each hold a queue of the same n clips.  chd_phys_queue_solve then asks it for `slots` positions at the start
 * and, at every refill check point, for as many positions as there are finished slots; the k positions it returns
 * enter the first k of those slots as one upload.  Once it returns fewer than asked it is not asked again: finished
 * slots are still harvested but no longer refilled.  The solve returns -1, and the handle stays usable, if the source
 * returns a negative value, a range outside [0, n), or a position it already handed out in this solve (checked on the
 * host before any upload).  claim = NULL restores the queue's own order.  Returns -1 for NULL or a batch handle. */
int chd_phys_queue_set_claim(chd_phys_batch* b, chd_phys_claim_fn* claim, void* ctx);

/* Number of kernels launched by this batch so far. */
int64_t chd_phys_launch_count(const chd_phys_batch* b);
/* Bytes copied host -> device by chd_phys_batch_create (problem data + layout tables). */
int64_t chd_phys_h2d_bytes(const chd_phys_batch* b);
/* Restores the initial point of nlp_formulation.cpp:106-203 on the device (no host traffic). */
int chd_phys_reset(chd_phys_batch* b);

/* Per-kernel accumulated CUDA-event time (ms) and launch counts since the last reset:
 * names: 0 eval, 1 kkt (assemble+factor+solve), 2 linesearch, 3 init, 4 sample, 5 admission of a queue (upload +
 * chd_k_admit).  [host] arrays of 8. */
int chd_phys_kernel_times(chd_phys_batch* b, double* ms8, int64_t* launches8, int reset);
int chd_phys_set_timing(chd_phys_batch* b, int enable);

/* ---------------------------------------------------------------------------------------------------------
 * Foot-contact classifier (src/contact_learning/test.py:51-152 val_full_video + models/openpose_only.py:29-78).
 * weights: the five Linear weights in torch layout [out][in], concatenated in layer order
 *          (1024x351, 512x1024, 128x512, 32x128, 20x32); biases concatenated likewise;
 * bn: for each of the four BatchNorm1d layers gamma, beta, running_mean, running_var (4 x width floats), concatenated.
 * All [host].  Keys of the reference state_dict: model.{0,3,6,10,13}.{weight,bias}, model.{1,4,7,11}.*. */
typedef struct chd_contact_net chd_contact_net;
int chd_contact_create(const float* weights, const float* biases, const float* bn, float bn_eps, int32_t device,
                       chd_contact_net** out);
void chd_contact_destroy(chd_contact_net* net);
/* frames [host]: V x Fmax x 25 x 3 doubles = keypoints after the dataset's preprocessing (pad to the longest video,
 * scale to 1280 wide, low-confidence interpolation, division by 200.416..., real_video_dataset.py:132-163);
 * seq_lens [host] V; labels [host] V x Fmax x 4 int64 (columns L heel, L toe, R heel, R toe; rows >= seq_len are 0);
 * logits [host, optional] V x (Fmax-8) x 20; min_abs_logit [host, optional]: smallest |logit| that entered a vote. */
int chd_contact_forward(chd_contact_net* net, const double* frames, int32_t V, int32_t Fmax, const int32_t* seq_lens,
                        int64_t* labels, float* logits, float* min_abs_logit);
/* Same with every buffer already on the device (stream = cudaStream_t as void*, NULL = the net's own stream); all
 * device buffers, logits_dev and min_abs_dev included, are required (they are workspace of the vote kernel). */
int chd_contact_forward_device(chd_contact_net* net, const double* frames_dev, int32_t V, int32_t Fmax,
                               const int32_t* seq_lens_dev, int64_t* labels_dev, float* logits_dev, float* min_abs_dev,
                               void* stream);
/* Dataset preprocessing on the device (RealVideoDataset.__init__, real_video_dataset.py:132-163, OpenPoseDataset,
 * openpose_dataset.py:126-269, and process_openpose_data, openpose_dataset.py:49-121): raw [host] = concatenated
 * OpenPose keypoints (sum F) x 25 x 3 doubles [x, y, confidence] as load_keypoint_dir returns them, seq_offsets [host]
 * V+1 frame offsets.  Videos are padded to the longest one, xy is multiplied by `scale` before the low-confidence
 * interpolation and divided by `norm` after it.  Real videos use scale = 1280.0 / width of the source video (reference
 * default 1920) and norm = 200.4160302695367, both in double; the synthetic dataset uses scale = 1 (exact) and norm =
 * the median MidHip -> LBigToe distance of its raw keypoints.  frames_out [host] V x Fmax x 25 x 3 (Fmax = longest
 * video), seq_lens_out [host, optional] V.  Bit identical to the reference's numpy result.  Returns -1 for scale or
 * norm not > 0. */
int chd_contact_preprocess(chd_contact_net* net, const double* raw, const int32_t* seq_offsets, int32_t V, double scale,
                           double norm, double* frames_out, int32_t* seq_lens_out);
/* Scores the logits of chd_contact_forward_device against ground-truth contacts (test.py:51-152 val_full_video with
 * labels), one CTA per video, on `stream` after the forward.  logits_dev [device] V x (Fmax-8) x 20 as the forward leaves
 * them; truth_dev [device] int32 (sum of rows) x 4, video v owning rows truth_offsets_dev[v] .. [v+1]-1
 * (truth_offsets_dev [device] V+1, non-decreasing); a video's rows are padded with its last row or trimmed to Fmax
 * (fix_data_len, real_video_dataset.py:165-191), a nonzero entry is a contact, a video without rows has no labels and
 * gets zeros.  Outputs [device], per video:
 *   loss_sum_dev    V doubles: sum over windows x 5 frames x 4 contacts of BCE-with-logits (OpenPoseModel.loss), every
 *                   term in fp32, the sum in fp64;
 *   conf_frames_dev V x 5 x 4 int64: (tp, fp, fn, tn) of sigmoid(x) > classify_thresh (fp32) for predicted frame p of
 *                   every window w against truth row w + 2 + p (OpenPoseModel.accuracy, tgt_frame = p);
 *   conf_merged_dev V x 4 int64: (tp, fp, fn, tn) over all Fmax frames x 4 of the 0.5 vote before trimming to seq_len,
 *                   against truth row clamp(f, 2, Fmax - 3) (test.py:124-140).
 * Windows over the padding of shorter videos are counted, as in the reference.  Each video's outputs are bitwise the
 * same whatever else is in the batch (given the same Fmax).  Returns 0, -1 bad argument, <= -100 CUDA error. */
int chd_contact_score_device(chd_contact_net* net, const float* logits_dev, int32_t V, int32_t Fmax, const int32_t* truth_dev,
                             const int32_t* truth_offsets_dev, float classify_thresh, double* loss_sum_dev,
                             int64_t* conf_frames_dev, int64_t* conf_merged_dev, void* stream);
/* test.py --full-video in one call: raw keypoints in, foot_contacts rows out, and with ground truth also the scores.
 * One upload of the raw keypoints (and the truth), then preprocessing (chd_contact_preprocess's scale / norm), forward,
 * vote, (score) and pack on the net's stream, then one download.  raw may be page-locked: the copies are asynchronous.
 * labels_out [host] (sum F) x 4 int64 (columns L heel, L toe, R heel, R toe; the rows every video's foot_contacts.npy
 * holds, concatenated); min_abs_logit [host, optional].
 *   Unlabelled (test.py --save-contacts --real-data): truth_offsets = NULL.  Nothing is scored; truth, classify_thresh,
 *   loss_sum, conf_frames and conf_merged are ignored and may be NULL.
 *   Labelled: truth [host] int32 (sum of rows) x 4 (may be NULL when there are no rows), truth_offsets [host] V+1
 *   starting at 0, non-decreasing; loss_sum [host] V, conf_frames [host] V x 5 x 4, conf_merged [host] V x 4 as
 *   chd_contact_score_device writes them for classify_thresh.
 * Either precision mode.  Returns 0, -1 bad argument, <= -100 CUDA error. */
int chd_contact_detect(chd_contact_net* net, const double* raw, const int32_t* seq_offsets, int32_t V, double scale, double norm,
                       const int32_t* truth, const int32_t* truth_offsets, float classify_thresh, int64_t* labels_out,
                       double* loss_sum, int64_t* conf_frames, int64_t* conf_merged, float* min_abs_logit);
int64_t chd_contact_launch_count(const chd_contact_net* net);
/* Numerical mode of every later chd_contact_forward / _forward_device / _detect call on this net.
 * FP32 (default): FFMA, labels match the reference's fp32 forward.  TF32X3: the 352-1024-512-128 layers on the
 * tensor core (wgmma) with every operand split into two TF32 parts, three products per term; logits within 5e-5
 * absolute of an fp64 forward (measured on an H100: 8.3e-6 on the golden clips, fp32 mode 8.5e-7; at most 1.1e-5 from
 * the fp32 mode over 100k windows), so labels can differ from FP32 only where a logit is within about 1e-5 of zero.
 * The slab workspace grows from 7.9 KB to 15.3 KB per window (132 MB -> 256 MB for a full slab of 16384 windows) and
 * the split weights take 7.6 MB.  Switching back to FP32 frees the fast mode's buffers; results are then bitwise
 * those of a net that never left FP32.
 * Returns 0, -1 bad argument, <= -100 CUDA error. */
enum { CHD_CONTACT_FP32 = 0, CHD_CONTACT_TF32X3 = 1 };
int chd_contact_set_precision(chd_contact_net* net, int32_t precision);

/* OpenPose keypoint ingestion on the host threads (replaces the serial per-file json.load of
 * src/utils/openpose_utils.py:48-76 load_keypoint_file / load_keypoint_dir): n_files `*_keypoints.json` files ->
 * out [host] n_files x num_joints x 3 fp64 (x, y, confidence of the FIRST person's "pose_keypoints_2d"; zeros for a frame
 * without people), bit-identical to the reference's arrays (strtod).  n_threads <= 0: all hardware threads.
 * Returns 0, -1 bad argument, -2 unreadable file, -3 malformed file / keypoint count != 3 * num_joints. */
int chd_openpose_load(const char* const* paths, int32_t n_files, int32_t num_joints, double* out, int32_t n_threads);

/* ---------------------------------------------------------------------------------------------------------
 * Kinematic initialisation: the linear solves inside least_squares(tr_solver='lsmr') of optimize_trajectory.py:660-670
 * and :779-789, for K clips in one launch.  Clip k owns frames seg[k] .. seg[k+1]-1 of the concatenated frame axis;
 * every system is the damped Gauss-Newton system of the clip,
 *     (H + lam[k] * diag(max(diag H, 1e-12))) s = g,
 * with H symmetric block-pentadiagonal in 87 x 87 blocks: D [device] (F_total x 87 x 87) diagonal blocks,
 * B1 [device] ((F_total-1) x 87 x 87) with B1[f] = block (f+1, f), B2 [device] ((F_total-2) x 87 x 87) with
 * B2[f] = block (f+2, f), all row major; blocks that would couple two clips are not read.  g, s [device] F_total x 87.
 * seg [device] K+1 frame offsets, lam [device] K.  sel [device, may be NULL]: the n_sel clips to solve (NULL: all K);
 * the others' s and status are not touched.  work [device]: chd_kin_work_bytes(F_total) bytes.
 * status [device] K: 0 solved, f + 1 when block f of the clip (clip-local frame) has a pivot that is not positive and
 * finite (s of that clip unspecified), -1 when the clip's frame range is not inside [0, F_total).  Each clip's s is
 * bitwise the same whatever else is in the launch.  Asynchronous on `stream` (cudaStream_t as void*).
 * Returns 0, -1 bad argument, <= -100 CUDA error. */
int chd_kin_solve(const double* D, const double* B1, const double* B2, const double* g, const int32_t* seg,
                  const double* lam, const int32_t* sel, int32_t n_sel, int32_t K, int32_t F_total, double* work,
                  double* s, int32_t* status, void* stream);
/* Bytes of `work` chd_kin_solve needs for F_total frames (three padded 88 x 88 fp64 blocks per frame); -1 if F_total < 0. */
int64_t chd_kin_work_bytes(int32_t F_total);

/* ---------------------------------------------------------------------------------------------------------
 * Full-body IK: JacobianInverseKinematicsCK (InverseKinematics.py:326-540; unit weights, gamma 1, no angle limits) for
 * K clips of one skeleton, `iterations` damped least-squares steps with damping lambda = damping / 1.001 and the
 * smoothing term smoothness * (x_{f-1} + x_{f+1} - 2 x_f) (a clip's first / last frame stands in for its missing
 * neighbour); x = [Euler angles; local translations] with `translate`, the Euler angles alone otherwise.
 * parents [host] J, parents[0] = -1, -1 <= parents[j] < j;  targets [host] T joint indices;
 * seg [host] K+1 frame offsets (0 .. F_total, non-decreasing): clip k owns frames seg[k] .. seg[k+1]-1;
 * R [device] F_total x J x 3 x 3 and P [device] F_total x J x 3 local rotations / translations, updated in place;
 * goal [device] F_total x T x 3 world positions of the targets;  work [device] chd_ik_work_bytes(F_total, J, T) bytes.
 * Returns 0, -1 bad argument (J outside 1..128, T outside 1..64, parents not ordered, a target out of range, bad seg;
 * nothing is launched), <= -100 CUDA error.  Asynchronous on `stream`, except that the upload of the ancestor tables
 * from pageable host memory may wait for earlier work on the stream.  Each clip's result is bitwise independent of the
 * rest of the batch. */
int chd_ik_solve(int32_t J, const int32_t* parents, int32_t T, const int32_t* targets, const int32_t* seg, int32_t K,
                 int32_t F_total, double* R, double* P, const double* goal, int32_t iterations, double damping,
                 double smoothness, int32_t translate, double* work, void* stream);
/* Bytes of `work` chd_ik_solve needs (ancestor tables and two copies of the state); -1 outside the limits above. */
int64_t chd_ik_work_bytes(int32_t F_total, int32_t J, int32_t T);

const char* chd_version(void);

/* Measurement helper (no reference counterpart): sustained fp64 throughput of the current device in GFLOP/s, for the
 * scalar FMA pipe (DFMA) and for the fp64 tensor-core instruction the KKT kernel uses (mma.sync m16n8k8, DMMA);
 * MEASURED_PEAKS.json carries no fp64 figure (SURVEY 8(d)).  Either output may be NULL. */
int chd_measure_fp64_peak(double* dfma_gflops, double* dmma_gflops);

#ifdef __cplusplus
}
#endif
#endif /* CHD_H_ */
