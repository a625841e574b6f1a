// Host-side NLP layout of a batch of phys-optim sequences (product code).
// Replaces, per sequence, NlpFormulation::GetVariableSets / GetConstraints
// (towr_phys_optim/src/nlp_formulation.cpp:79-360) and the ifopt Problem assembly of
// phys_optim.cpp:544-552: instead of objects it emits flat, padded tables the kernels index directly.
#pragma once
#include <vector>

#include "../../include/chd.h"
#include "chd_core.h"

struct ChdStageCfg {
  unsigned set_mask;                 // active constraint-set types
  double w_data[3];                  // lin, ang, ee
  double w_vel[3];                   // "velocity smoothing" (deriv = pos)
  double w_acc[3];                   // "acceleration smoothing" (deriv = vel)
  int max_iter;
  double w_dur;                      // duration_cost.cpp (stage 3 only)
};

struct ChdHostBatch {
  int B = 0;
  // padded strides
  int S = 0, Pmax = 0, n_max = 0, m_max = 0, slots_max = 0, sets_max = 0, tab_max = 0, F_max = 0, Kd_max = 0, Kr_max = 0;
  int Na_max = 0, nb_max = 0, w_max = 0, w_fix_max = 0, n_ee_max = 0, fo_max = 0, Ph_max = 0;
  std::vector<ChdSeq> seq;
  std::vector<double> poly_T, poly_tend, node_const, par, t_dyn, t_rom, t_data, row_lo, row_hi, x0, phase_tend;
  std::vector<double> dur0;          // B x n_ee_max x Ph_max initial phase durations (DurationCost target, table rebuilds)
  std::vector<int> node_var, itab, ent_ptr, ent_col, var_kkt, row_kkt, row_set;
  std::vector<int> poly_ph;          // B x S x Pmax: phase | poly-in-phase << 12 | polys-in-phase << 20 (phase based splines)
  std::vector<int> ent_row, col_ptr, col_ent;   // row of every Jacobian slot; slots grouped by column (gathers instead of atomics)
  std::vector<ChdSet> sets;
  std::vector<ChdStageCfg> stage;    // B x 6: the stages of every sequence (its weights), [b * 6 + stage id]
  int par_stride() const { return (18 + 3 * n_ee_max) * F_max; }
};

// returns 0 on success; negative on malformed input.  w: the weights of every problem (batch entries).
// stage3_band_above: see chd_phys_options (-1: switch times are border unknowns, stage 3 limited to CHD_MAX_DUR of them)
int chd_build_layout(const chd_phys_problem* problems, int batch, const chd_phys_weights* w, ChdHostBatch& out,
                     int stage3_band_above = -1);
// the same weights for every problem
inline int chd_build_layout(const chd_phys_problem* problems, int batch, const chd_phys_weights& w, ChdHostBatch& out,
                            int stage3_band_above = -1) {
  return chd_build_layout(problems, batch, std::vector<chd_phys_weights>(batch, w).data(), out, stage3_band_above);
}
