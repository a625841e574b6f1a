// Host-side layout builder (product code).  See chd_layout.h.
#include "chd_layout.h"
#include "chd_dev.h"

#include <algorithm>
#include <atomic>
#include <thread>
#include <cmath>
#include <cstring>
#include <numeric>

namespace {

struct PolyInfo {
  int phase, poly_in_phase, n_polys;
  bool constant;
};

struct SplineBuild {
  std::vector<double> T;        // polynomial durations
  std::vector<int> var;         // (npoly+1)*6 -> sequence-local x index or -1, [px,py,pz,vx,vy,vz]
  std::vector<double> cval;     // value used where var == -1 (and initial value otherwise)
  std::vector<PolyInfo> info;   // phase based splines only
  std::vector<char> const_node; // phase based: node adjacent to a constant polynomial
  int xoff = 0, nvar = 0;
  int npoly() const { return (int)T.size(); }
  int nnodes() const { return (int)T.size() + 1; }
};

// phys_optim.cpp:289-312 (GetPolyChangingPhase)
std::vector<int> polys_changing(bool start_constant, const double* dur, int P, double max_dur, int per_change) {
  std::vector<int> out;
  bool constant = start_constant;
  const double per_s = per_change / max_dur;
  for (int i = 0; i < P; ++i) {
    if (!constant) {
      int np = per_change;
      if (dur[i] > max_dur) np += (int)std::ceil((dur[i] - max_dur) * per_s);
      out.push_back(np);
    }
    constant = !constant;
  }
  return out;
}

// nodes_variables_dynamic_phase_based.cpp:10-34 + towr NodesVariablesPhaseBased::IsConstantNode
void build_phase_spline(SplineBuild& s, const double* dur, int P, bool first_constant, const std::vector<int>& n_change) {
  bool constant = first_constant;
  int cc = 0;
  for (int i = 0; i < P; ++i) {
    if (constant) {
      s.info.push_back({i, 0, 1, true});
    } else {
      int np = n_change[cc++];
      for (int j = 0; j < np; ++j) s.info.push_back({i, j, np, false});
    }
    constant = !constant;
  }
  for (auto& pi : s.info) s.T.push_back(dur[pi.phase] / pi.n_polys);
  int nn = s.nnodes();
  s.const_node.assign(nn, 0);
  for (int node = 0; node < nn; ++node) {
    bool c = false;
    if (node > 0 && s.info[node - 1].constant) c = true;
    if (node < nn - 1 && s.info[node].constant) c = true;
    s.const_node[node] = c;
  }
  s.var.assign((size_t)nn * 6, -1);
  s.cval.assign((size_t)nn * 6, 0.0);
}

struct SeqBuild {
  ChdSeq h;
  std::vector<SplineBuild> sp;
  std::vector<double> x0, t_dyn, t_rom, t_data, row_lo, row_hi, var_t0, var_t1, row_t;
  std::vector<char> var_fixed, var_stance, var_dur;
  std::vector<ChdSet> sets;
  std::vector<int> itab, ent_ptr, ent_col, var_kkt, row_kkt, row_set;
};

// towr TimeDiscretizationConstraint: 0, dt, 2dt (accumulated) ..., T
std::vector<double> discretize(double T, double dt) {
  std::vector<double> d = {0.0};
  double t = 0.0;
  for (int i = 0; i < std::floor(T / dt); ++i) {
    t += dt;
    d.push_back(t);
  }
  d.push_back(T);
  return d;
}

// Whether a KKT system of half bandwidth w_max and nb_max border unknowns fits chd_k_kkt_gwin, the kernel bands this
// wide run in: its pair table (panel groups) and its shared memory.  Checked for the whole batch, whose strides come
// from the widest band and the largest border of possibly different sequences.
bool kkt_fits(int w_max, int nb_max) {
  return chd_kkt_gwin_status(w_max, nb_max, CHD_KKT_GWIN_STATIC_MAX, CHD_SMEM_OPTIN) == CHD_KKT_FITS;
}

// Returns 0, a negative code for malformed input, or 1 when banded switch times would make the band too wide for the
// KKT kernels (the caller then builds the sequence again without them).
int build_sequence(const chd_phys_problem& p, SeqBuild& sb, int band_above) {
  if (p.n_ee != 2 && p.n_ee != 4) return -2;
  if (p.n_frames < 12) return -3;
  const int F = p.n_frames, n_ee = p.n_ee;
  ChdSeq& h = sb.h;
  std::memset(&h, 0, sizeof(h));
  h.n_ee = n_ee;
  h.F = F;
  h.n_splines = 2 + 2 * n_ee;
  h.dt = p.dt;
  h.mass = p.body_mass;
  h.grav = 9.80665;      // towr DynamicModel gravity
  h.mu = 0.5;            // towr HeightMap default friction coefficient
  h.force_limit = 1000;  // parameters.cpp:56
  h.max_leg = p.max_leg_length;
  h.max_heel = p.max_heel_length;
  h.heel_dist = p.heel_dist;
  for (int d = 0; d < 3; ++d) h.normal[d] = p.floor_normal[d], h.point[d] = p.floor_point[d];
  const double nn = std::sqrt(h.normal[0] * h.normal[0] + h.normal[1] * h.normal[1] + h.normal[2] * h.normal[2]);
  for (int d = 0; d < 3; ++d) h.gvec[d] = -h.normal[d] / nn;  // gravity = -floor normal (phys_optim.cpp:437)
  h.dhdx = -h.normal[0] / h.normal[2];                        // ground_plane.cpp:28-40
  h.dhdy = -h.normal[1] / h.normal[2];
  {  // towr HeightMap basis of a plane
    double n[3] = {-h.dhdx, -h.dhdy, 1.0}, t1[3] = {1.0, 0.0, h.dhdx}, t2[3] = {0.0, 1.0, h.dhdy};
    double a = std::sqrt(chd_dot(n, n)), b = std::sqrt(chd_dot(t1, t1)), c = std::sqrt(chd_dot(t2, t2));
    for (int d = 0; d < 3; ++d) h.nrm[d] = n[d] / a, h.tan1[d] = t1[d] / b, h.tan2[d] = t2[d] / c;
  }
  // contact schedule
  std::vector<const double*> dur(n_ee);
  std::vector<int> P(n_ee);
  {
    const double* d = p.ee_durations;
    for (int ee = 0; ee < n_ee; ++ee) {
      dur[ee] = d;
      P[ee] = p.ee_n_phases[ee];
      if (P[ee] < 1) return -4;
      d += P[ee];
    }
  }
  double T = 0.0;  // Parameters::GetTotalTime: the first foot is the reference (parameters.cpp:138-153)
  for (int i = 0; i < P[0]; ++i) T += dur[0][i];
  h.T = T;
  for (int ee = 0; ee < n_ee; ++ee) h.start_contact[ee] = p.ee_start_contact[ee] != 0, h.n_phases[ee] = P[ee];
  // base polynomials (parameters.cpp:109-125)
  std::vector<double> base_T;
  {
    double t_left = T;
    const double eps = 1e-10, dtb = 0.1;
    while (t_left > eps) {
      base_T.push_back(t_left > dtb ? dtb : t_left);
      t_left -= dtb;
    }
  }
  sb.sp.assign(h.n_splines, SplineBuild());
  auto height = [&](double x, double y) {  // ground_plane.cpp:18-26
    double z = -h.normal[1] * (y - h.point[1]) - h.normal[0] * (x - h.point[0]);
    z /= h.normal[2];
    return z + h.point[2];
  };
  auto V = [&](const double* a, int i, int d) { return a[3 * i + d]; };
  // initial / final base velocity: mean of the first / last five finite differences (phys_optim.cpp:442-481)
  double v0[3] = {0, 0, 0}, vf[3] = {0, 0, 0};
  for (int d = 0; d < 3; ++d) {
    for (int i = 0; i < 5; ++i) {
      v0[d] += (V(p.base_lin, i + 1, d) - V(p.base_lin, i, d)) / p.dt;
      vf[d] += (V(p.base_lin, F - 1 - i, d) - V(p.base_lin, F - 2 - i, d)) / p.dt;
    }
    v0[d] /= 5;
    vf[d] /= 5;
  }
  int xoff = 0;
  sb.x0.clear();
  sb.var_fixed.clear();
  sb.var_stance.clear();
  // base splines: towr NodesVariablesAll, [px,py,pz,vx,vy,vz] per node, linear interpolation init
  for (int s = 0; s < 2; ++s) {
    SplineBuild& S = sb.sp[s];
    S.T = base_T;
    const int nn_ = S.nnodes();
    S.var.resize((size_t)nn_ * 6);
    S.cval.resize((size_t)nn_ * 6);
    const double* data = s == 0 ? p.base_lin : p.base_ang;
    for (int node = 0; node < nn_; ++node)
      for (int k = 0; k < 6; ++k) {
        const int d = k % 3;
        const double a = V(data, 0, d), b = V(data, F - 1, d);
        double val = k < 3 ? a + node / static_cast<double>(nn_ - 1) * (b - a) : (b - a) / T;
        bool fixed = false;
        if (s == 0 && k >= 3 && node == 0) val = v0[d], fixed = true;        // AddStartBound (nlp_formulation.cpp:121)
        if (s == 0 && k >= 3 && node == nn_ - 1) val = vf[d], fixed = true;  // AddFinalBound (nlp_formulation.cpp:122)
        S.var[node * 6 + k] = xoff + node * 6 + k;
        S.cval[node * 6 + k] = val;
        sb.x0.push_back(val);
        sb.var_fixed.push_back(fixed);
        sb.var_stance.push_back(0);
      }
    S.xoff = xoff;
    S.nvar = nn_ * 6;
    xoff += S.nvar;
  }
  // ee motion splines (nlp_formulation.cpp:133-162, nodes_variables_dynamic_phase_based.cpp:58-106)
  const double fx = V(p.base_lin, F - 1, 0), fy = V(p.base_lin, F - 1, 1);
  const double fin[3] = {fx, fy, height(fx, fy)};
  for (int ee = 0; ee < n_ee; ++ee) {
    SplineBuild& S = sb.sp[chd_sp_motion(ee)];
    build_phase_spline(S, dur[ee], P[ee], p.ee_start_contact[ee] != 0,
                       polys_changing(p.ee_start_contact[ee] != 0, dur[ee], P[ee], 2.0, 6));
    const int nn_ = S.nnodes();
    const double* e0 = p.ee_pos + (size_t)ee * F * 3;
    S.xoff = xoff;
    auto interp = [&](int node, int d) { return e0[d] + node / static_cast<double>(nn_ - 1) * (fin[d] - e0[d]); };
    for (int node = 0; node < nn_; ++node) {
      if (!S.const_node[node]) {
        for (int d = 0; d < 3; ++d) {
          S.var[node * 6 + d] = xoff, S.cval[node * 6 + d] = interp(node, d);
          sb.x0.push_back(interp(node, d)), sb.var_fixed.push_back(0), sb.var_stance.push_back(0), xoff++;
          const double vel = (fin[d] - e0[d]) / T;
          S.var[node * 6 + 3 + d] = xoff, S.cval[node * 6 + 3 + d] = vel;
          sb.x0.push_back(vel), sb.var_fixed.push_back(0), sb.var_stance.push_back(0), xoff++;
        }
      } else {
        // one xyz variable shared by the two nodes of the stance polynomial; ifopt starts from the value of
        // the last NodeValueInfo (node + 1); velocities are constants 0
        for (int d = 0; d < 3; ++d) {
          const double val = interp(node + 1, d);
          S.var[node * 6 + d] = xoff, S.var[(node + 1) * 6 + d] = xoff;
          S.cval[node * 6 + d] = val, S.cval[(node + 1) * 6 + d] = val;
          sb.x0.push_back(val), sb.var_fixed.push_back(0), sb.var_stance.push_back(1), xoff++;
        }
        node += 1;
      }
    }
    S.nvar = xoff - S.xoff;
  }
  // ee force splines (nlp_formulation.cpp:164-186, nodes_variables_dynamic_phase_based.cpp:108-151)
  for (int ee = 0; ee < n_ee; ++ee) {
    SplineBuild& S = sb.sp[chd_sp_force(n_ee, ee)];
    build_phase_spline(S, dur[ee], P[ee], p.ee_start_contact[ee] == 0,
                       polys_changing(p.ee_start_contact[ee] == 0, dur[ee], P[ee], 2.0, 6));
    const int nn_ = S.nnodes();
    S.xoff = xoff;
    const double fz = h.mass * h.grav / n_ee;
    for (int node = 0; node < nn_; ++node) {
      if (!S.const_node[node]) {
        for (int d = 0; d < 3; ++d) {
          const double val = d == 2 ? fz : 0.0;
          S.var[node * 6 + d] = xoff, S.cval[node * 6 + d] = val;
          sb.x0.push_back(val), sb.var_fixed.push_back(0), sb.var_stance.push_back(0), xoff++;
          S.var[node * 6 + 3 + d] = xoff, S.cval[node * 6 + 3 + d] = 0.0;
          sb.x0.push_back(0.0), sb.var_fixed.push_back(0), sb.var_stance.push_back(0), xoff++;
        }
      } else {
        node += 1;  // swing polynomial: both nodes pinned to zero force
      }
    }
    S.nvar = xoff - S.xoff;
  }
  // phase durations (nlp_formulation.cpp:188-203; stacked after the node sets, phys_optim.cpp:680-681): P - 1 free
  // durations per foot.  They are variables of stage 3 only; the other stages keep them fixed.
  sb.var_dur.assign(sb.x0.size(), 0);
  {
    int nd = 0;
    for (int ee = 0; ee < n_ee; ++ee) nd += P[ee] - 1;
    h.dur_band = band_above >= 0 && nd > band_above;
    h.n_dur = nd <= CHD_MAX_DUR || h.dur_band ? nd : 0;
    for (int ee = 0; ee < n_ee; ++ee) {
      h.dur_xoff[ee] = xoff;
      if (!h.n_dur) continue;
      for (int k = 0; k < P[ee] - 1; ++k)
        sb.x0.push_back(dur[ee][k]), sb.var_fixed.push_back(0), sb.var_stance.push_back(0), sb.var_dur.push_back(1), xoff++;
    }
  }
  h.n = xoff;
  for (int s = 0; s < h.n_splines; ++s) h.sp_npoly[s] = sb.sp[s].npoly(), h.sp_xoff[s] = sb.sp[s].xoff, h.sp_nvar[s] = sb.sp[s].nvar;

  // node times -> variable time spans
  sb.var_t0.assign(h.n, 1e300);
  sb.var_t1.assign(h.n, -1e300);
  std::vector<std::vector<double>> tend(h.n_splines);
  for (int s = 0; s < h.n_splines; ++s) {
    double t = 0;
    for (int k = 0; k <= sb.sp[s].npoly(); ++k) {
      for (int q = 0; q < 6; ++q) {
        int v = sb.sp[s].var[k * 6 + q];
        if (v >= 0) sb.var_t0[v] = std::min(sb.var_t0[v], t), sb.var_t1[v] = std::max(sb.var_t1[v], t);
      }
      if (k < sb.sp[s].npoly()) {
        t += sb.sp[s].T[k];
        tend[s].push_back(t);
      }
    }
  }
  // input switch times: ph_end[ee][k] = end of phase k of foot ee
  std::vector<std::vector<double>> ph_end(n_ee);
  for (int ee = 0; ee < n_ee; ++ee) {
    double t = 0.0;
    for (int k = 0; k < P[ee]; ++k) t += dur[ee][k], ph_end[ee].push_back(t);
  }
  const double margin = CHD_TAU_TRUST;   // [s] how far stage 3 may move a switch time (and with it a polynomial boundary)
  for (int v = 0; v < h.n; ++v)
    if (sb.var_dur[v]) sb.var_t0[v] = 0.0, sb.var_t1[v] = T;
  // banded switch times: tau_k bounds phases k and k+1, whose rows and cost samples are all it touches
  if (h.dur_band)
    for (int ee = 0; ee < n_ee; ++ee)
      for (int k = 0; k < P[ee] - 1; ++k) {
        const int v = h.dur_xoff[ee] + k;
        sb.var_t0[v] = (k > 0 ? ph_end[ee][k - 1] : 0.0) - margin;
        sb.var_t1[v] = (k + 1 < P[ee] - 1 ? ph_end[ee][k + 1] : T) + margin;
      }
  // Switch times a sample at time t can depend on in stage 3: a sample in phase j of foot ee depends on tau_{j-1} and
  // tau_j, and once every switch time has moved by up to the trust margin t may lie in a neighbouring phase instead.
  // One option (pair of variables, -1 for the fixed ends 0 and T) per phase t can lie in, appended to `opts`.
  auto tau_reach = [&](int ee, double t, std::vector<std::vector<int>>& opts) {
    if (!h.dur_band) return;
    std::vector<int> o;
    for (int j = 0; j < P[ee]; ++j) {   // (the last phase runs to T whatever the input durations of the foot add up to)
      const double a = j > 0 ? ph_end[ee][j - 1] : -1e300, b = j < P[ee] - 1 ? ph_end[ee][j] : 1e300;
      if (t < a - margin || t > b + margin) continue;
      o.push_back(j >= 1 ? h.dur_xoff[ee] + j - 1 : -1);
      o.push_back(j <= P[ee] - 2 ? h.dur_xoff[ee] + j : -1);
    }
    opts.push_back(o);
  };
  // calls fn(cols) with `base` plus one option of every entry of `opts` for each combination (fn(base) when empty)
  auto for_options = [](const std::vector<int>& base, const std::vector<std::vector<int>>& opts, auto&& fn) {
    size_t total = 1;
    for (const auto& o : opts) total *= o.size() / 2;
    std::vector<int> cols;
    for (size_t c = 0; c < total; ++c) {
      cols = base;
      size_t rem = c;
      for (const auto& o : opts) {
        const size_t k = rem % (o.size() / 2);
        rem /= o.size() / 2;
        cols.push_back(o[2 * k]), cols.push_back(o[2 * k + 1]);
      }
      fn(cols);
    }
  };
  // time tables
  sb.t_dyn = discretize(T, 0.1);   // parameters.cpp:58-59 (dynamic and height share dt = 0.1)
  sb.t_rom = discretize(T, 0.08);  // parameters.cpp:57
  sb.t_data.resize(F);
  {
    double t = 0.0;  // data_cost.cpp:45-49
    for (int i = 0; i < F; ++i) sb.t_data[i] = t, t += 1 * p.dt;
    int ns = 0;      // vel_smooth_cost.cpp:41: for (t = 0; t < T_spline - dt; t += dt)
    const double Tsp = std::accumulate(base_T.begin(), base_T.end(), 0.0);
    for (double tt = 0.0; tt < (Tsp - p.dt); tt += p.dt) ns++;
    h.n_smooth = std::min(ns, F);
  }
  h.n_dyn = (int)sb.t_dyn.size();
  h.n_rom = (int)sb.t_rom.size();

  // ---- master constraint rows ----
  int row = 0;
  auto add_set = [&](int type, int a, int b, int nitems, int tab) {
    ChdSet st{type, a, b, row, nitems, tab};
    sb.sets.push_back(st);
    row += nitems * chd_rows_per_item(type);
  };
  add_set(CHD_SET_ACC, 0, 0, (int)base_T.size() - 1, 0);
  add_set(CHD_SET_ACC, 1, 0, (int)base_T.size() - 1, 0);
  for (int ee = 0; ee < n_ee; ++ee) add_set(CHD_SET_TERRAIN, ee, 0, sb.sp[chd_sp_motion(ee)].nnodes() - 1, 0);
  for (int ee = 0; ee < n_ee; ++ee) add_set(CHD_SET_ROM, ee, 0, h.n_rom, 0);
  add_set(CHD_SET_DYN, 0, 0, h.n_dyn, 0);
  for (int ee = 0; ee < n_ee; ++ee) {
    const SplineBuild& S = sb.sp[chd_sp_force(n_ee, ee)];
    int tab = (int)sb.itab.size(), cnt = 0;
    for (int node = 0; node < S.nnodes(); ++node)
      if (!S.const_node[node]) sb.itab.push_back(node), cnt++;
    add_set(CHD_SET_FORCE, ee, 0, cnt, tab);
  }
  if (n_ee >= 4) {  // nlp_formulation.cpp:243-262
    add_set(CHD_SET_HEEL, 0, 2, h.n_rom, 0);
    add_set(CHD_SET_HEEL, 1, 3, h.n_rom, 0);
  }
  for (int ee = 0; ee < n_ee; ++ee) add_set(CHD_SET_HEIGHT, ee, 0, h.n_dyn, 0);
  if (h.n_dur) {  // stage 3 only (phys_optim.cpp:667-679): total-duration rows, duration bounds as rows
    for (int ee = 0; ee < n_ee; ++ee) add_set(CHD_SET_TOTTIME, ee, 0, 1, 0);
    for (int ee = 0; ee < n_ee; ++ee) add_set(CHD_SET_DURPOS, ee, 0, P[ee] - 1, 0);
  }
  h.m = row;
  h.nsets = (int)sb.sets.size();

  // ---- rows: bounds, time stamps, Jacobian slot columns ----
  sb.row_lo.assign(h.m, 0.0);
  sb.row_hi.assign(h.m, 0.0);
  sb.row_t.assign(h.m, 0.0);
  sb.row_set.assign(h.m, 0);
  sb.ent_ptr.assign(h.m + 1, 0);
  sb.ent_col.clear();
  // In stage 3 the polynomial boundaries of the phase-based splines move with the durations, so the polynomial active
  // at a fixed sample time can change: the node columns of those blocks are re-assigned at run time (chd_k_eval), and
  // the bandwidth below is sized for the neighbouring polynomials too (row_ext = their extra nodes).
  // With banded switch times, row_tau holds the switch-time options of the feet the row touches (tau_reach).
  std::vector<std::vector<int>> row_ext(h.m);
  std::vector<std::vector<std::vector<int>>> row_tau(h.m);
  int cur_row = 0;
  auto ext_nodes = [&](int s, int poly, double t, std::vector<int>& out) {
    if (s < 2 || !h.n_dur) return;
    auto put = [&](int node) {
      for (int q = 0; q < 6; ++q) out.push_back(sb.sp[s].var[node * 6 + q]);
    };
    for (int pp = poly - 1; pp >= 0 && tend[s][pp] > t - margin; --pp) put(pp);                                  // earlier polynomials that end within the margin
    for (int pp = poly + 1; pp < sb.sp[s].npoly() && tend[s][pp - 1] < t + margin; ++pp) put(pp + 1);            // later ones that start within it
  };
  auto block = [&](int s, double t) {  // 12 slots: side x (pos,vel) x dim of the polynomial active at t
    double tl;
    int poly = chd_locate(tend[s].data(), sb.sp[s].npoly(), t, &tl);
    for (int side = 0; side < 2; ++side)
      for (int q = 0; q < 6; ++q) sb.ent_col.push_back(sb.sp[s].var[(poly + side) * 6 + q]);
    ext_nodes(s, poly, t, row_ext[cur_row]);
  };
  // switch-time slots of the feet a time-located row touches: two per foot, columns assigned at run time in stage 3
  auto tau_slots = [&](int feet) {
    for (int q = 0; q < 2 * feet; ++q) sb.ent_col.push_back(-1);
  };
  for (const ChdSet& st : sb.sets) {
    const int rpi = chd_rows_per_item(st.type);
    for (int it = 0; it < st.nitems; ++it)
      for (int r = 0; r < rpi; ++r) {
        const int R = st.row0 + it * rpi + r;
        cur_row = R;
        sb.row_set[R] = st.type;
        sb.ent_ptr[R] = (int)sb.ent_col.size();
        switch (st.type) {
          case CHD_SET_ACC: {
            sb.row_t[R] = tend[st.a][it];
            for (int a = 0; a < 3; ++a)
              for (int dv = 0; dv < 2; ++dv) sb.ent_col.push_back(sb.sp[st.a].var[(it + a) * 6 + dv * 3 + r]);
            break;
          }
          case CHD_SET_TERRAIN: {
            const SplineBuild& S = sb.sp[chd_sp_motion(st.a)];
            const int node = it + 1;  // node 0 is skipped
            sb.row_t[R] = tend[chd_sp_motion(st.a)][node - 1];
            for (int d = 0; d < 3; ++d) sb.ent_col.push_back(S.var[node * 6 + d]);
            sb.row_lo[R] = 0.0;
            sb.row_hi[R] = S.const_node[node] ? 0.0 : 1e20;
            break;
          }
          case CHD_SET_ROM: {
            const double t = sb.t_rom[it];
            sb.row_t[R] = t;
            block(0, t), block(1, t), block(chd_sp_motion(st.a), t);
            tau_slots(1);
            tau_reach(st.a, t, row_tau[R]);
            const double L = st.a < 2 ? h.max_leg : h.max_heel;  // leg_length_constraint.cpp:21-27
            sb.row_lo[R] = 0.0, sb.row_hi[R] = 0.5 * L * L;
            break;
          }
          case CHD_SET_DYN: {
            const double t = sb.t_dyn[it];
            sb.row_t[R] = t;
            block(0, t), block(1, t);
            for (int ee = 0; ee < n_ee; ++ee) block(chd_sp_motion(ee), t), block(chd_sp_force(n_ee, ee), t);
            tau_slots(n_ee);
            for (int ee = 0; ee < n_ee; ++ee) tau_reach(ee, t, row_tau[R]);
            break;
          }
          case CHD_SET_FORCE: {
            const int s = chd_sp_force(n_ee, st.a);
            const int node = sb.itab[st.tab + it];
            sb.row_t[R] = node > 0 ? tend[s][node - 1] : 0.0;
            for (int d = 0; d < 3; ++d) sb.ent_col.push_back(sb.sp[s].var[node * 6 + d]);
            if (r == 0) sb.row_lo[R] = 0.0, sb.row_hi[R] = h.force_limit;
            else if (r == 1 || r == 3) sb.row_lo[R] = -1e20, sb.row_hi[R] = 0.0;
            else sb.row_lo[R] = 0.0, sb.row_hi[R] = 1e20;
            break;
          }
          case CHD_SET_HEEL: {
            const double t = sb.t_rom[it];
            sb.row_t[R] = t;
            block(chd_sp_motion(st.a), t), block(chd_sp_motion(st.b), t);
            tau_slots(2);
            tau_reach(st.a, t, row_tau[R]), tau_reach(st.b, t, row_tau[R]);
            sb.row_lo[R] = sb.row_hi[R] = 0.5 * h.heel_dist * h.heel_dist;
            break;
          }
          case CHD_SET_HEIGHT: {
            const double t = sb.t_dyn[it];
            sb.row_t[R] = t;
            block(chd_sp_motion(st.a), t);
            tau_slots(1);
            tau_reach(st.a, t, row_tau[R]);
            sb.row_lo[R] = 0.0, sb.row_hi[R] = 1e20;
            break;
          }
          case CHD_SET_TOTTIME: {  // sum of the free durations = last switch time (total_duration_constraint.cpp:60-82)
            sb.row_t[R] = T;
            sb.ent_col.push_back(h.dur_xoff[st.a] + P[st.a] - 2);
            sb.row_lo[R] = std::max(0.0, T - 500.0), sb.row_hi[R] = T - 0.0;   // parameters.cpp:60 bounds (0, 500)
            break;
          }
          case CHD_SET_DURPOS: {   // d_k = tau_k - tau_{k-1} >= 0
            sb.row_t[R] = T;
            sb.ent_col.push_back(h.dur_xoff[st.a] + it);
            sb.ent_col.push_back(it > 0 ? h.dur_xoff[st.a] + it - 1 : -1);
            sb.row_lo[R] = 0.0, sb.row_hi[R] = 1e20;
            break;
          }
        }
      }
  }
  sb.ent_ptr[h.m] = (int)sb.ent_col.size();
  h.nslots = (int)sb.ent_col.size();

  // ---- KKT ordering: time-sorted band + border of long-lived (stance) variables ----
  // Stance variables living longer than `span_max` go to the dense border, the others into the band.  The best
  // threshold depends on the gait: long stances (walking, ~0.6 s) belong in the border, the 0.13-0.33 s stances of
  // densely switching contacts fit inside the band's natural width.  Candidates are scored by the tile work of one
  // factorisation, block columns x (band groups + border groups)^2.
  auto order_kkt = [&](double span_max) -> double {
    struct Key {
      double t;
      int kind, id;
    };
    std::vector<Key> keys;
    std::vector<int> border;
    sb.var_kkt.assign(h.n, -1);
    sb.row_kkt.assign(h.m, -1);
    for (int v = 0; v < h.n; ++v) {
      if (sb.var_fixed[v] || (sb.var_dur[v] && !h.dur_band)) continue;
      if (sb.var_stance[v] && sb.var_t1[v] - sb.var_t0[v] > span_max) border.push_back(v);
      else keys.push_back({0.5 * (sb.var_t0[v] + sb.var_t1[v]), 0, v});
    }
    // rows that keep their multiplier as a KKT unknown: equalities, and inequalities with more than 12 slots
    // (leg length); the others (terrain, friction pyramid, height -- the latter is degenerate with the terrain
    // equality during stance and is numerically safer condensed) are condensed into the primal block
    auto explicit_row = [&](int r) { return sb.row_lo[r] == sb.row_hi[r] || sb.ent_ptr[r + 1] - sb.ent_ptr[r] > 16; };
    for (int r = 0; r < h.m; ++r)
      if (explicit_row(r)) keys.push_back({sb.row_t[r] + 1e-6, 1, r});
    std::stable_sort(keys.begin(), keys.end(), [](const Key& a, const Key& b) { return a.t < b.t; });
    for (size_t i = 0; i < keys.size(); ++i) (keys[i].kind == 0 ? sb.var_kkt[keys[i].id] : sb.row_kkt[keys[i].id]) = (int)i;
    h.Na = (int)keys.size();
    h.nb_fix = (int)border.size();
    // the switch times of stage 3 influence every row of two whole phases: dense border unknowns, placed last so that
    // the fixed-duration stages simply work with the first nb_fix border unknowns (unless they are banded, above)
    if (!h.dur_band)
      for (int v = 0; v < h.n; ++v)
        if (sb.var_dur[v]) border.push_back(v);
    h.nb = (int)border.size();
    for (int j = 0; j < h.nb; ++j) sb.var_kkt[border[j]] = h.Na + j;
    // half bandwidth from the coupling cliques: w_fix of the fixed-duration stages (the static pattern), w with the
    // neighbouring polynomials stage 3 may move onto a sample time
    int w = 0, w_fix = 0;
    bool with_ext = true;
    auto span = [&](const int* cols, int cnt, int rowpos) {
      int lo = 1 << 30, hi = -1;
      for (int i = 0; i < cnt; ++i) {
        if (cols[i] < 0) continue;
        if (!with_ext && sb.var_dur[cols[i]]) continue;   // the fixed-duration stages never couple a switch time
        int k = sb.var_kkt[cols[i]];
        if (k < 0 || k >= h.Na) continue;
        lo = std::min(lo, k), hi = std::max(hi, k);
      }
      if (rowpos >= 0) lo = std::min(lo, rowpos), hi = std::max(hi, rowpos);
      if (hi >= 0) (with_ext ? w : w_fix) = std::max(with_ext ? w : w_fix, hi - lo);
    };
    auto clique = [&](const std::vector<int>& cols) { span(cols.data(), (int)cols.size(), -1); };
    // (banded switch times, stage 3: a clique holds the switch times of one phase per foot at a time -- the options of
    // row_tau / tau_reach are alternatives, not one clique)
    const std::vector<std::vector<int>> no_opts;
    std::vector<int> merged;
    for (int pass = 0; pass < 2; ++pass)
    for (int r = 0; r < h.m; ++r) {
      with_ext = pass == 1;
      merged.assign(sb.ent_col.begin() + sb.ent_ptr[r], sb.ent_col.begin() + sb.ent_ptr[r + 1]);
      if (with_ext) merged.insert(merged.end(), row_ext[r].begin(), row_ext[r].end());
      const std::vector<std::vector<int>>& opts = with_ext ? row_tau[r] : no_opts;
      const int* c = merged.data();
      const int cnt = (int)merged.size();
      if (sb.row_kkt[r] >= 0) {  // explicit row: couples the row with each of its variables
        for (int i = 0; i < cnt; ++i) span(c + i, 1, sb.row_kkt[r]);
        for (const auto& o : opts)
          for (size_t i = 0; i < o.size(); ++i) span(&o[i], 1, sb.row_kkt[r]);
        if (sb.row_set[r] == CHD_SET_ROM || sb.row_set[r] == CHD_SET_HEEL) for_options(merged, opts, clique);  // curvature term y+ Jd^T Jd
      } else {
        for_options(merged, opts, clique);        // condensed inequality row: J^T Sigma J clique
      }
    }
    // cost cliques: data samples (one polynomial) and smoothing samples (polynomials at t and t + dt); stage 3 adds the
    // switch times of the foot splines' positions (the duration cost w D^T D couples the same pairs as the DURPOS rows)
    for (int pass = 0; pass < 2; ++pass)
    for (int s = 0; s < 2 + n_ee; ++s) {
      with_ext = pass == 1;
      for (int i = 0; i < F; ++i) {
        std::vector<int> cols;
        std::vector<std::vector<int>> opts;
        double tl;
        int poly = chd_locate(tend[s].data(), sb.sp[s].npoly(), sb.t_data[i], &tl);
        for (int q = 0; q < 12; ++q) cols.push_back(sb.sp[s].var[poly * 6 + q]);
        if (with_ext) ext_nodes(s, poly, sb.t_data[i], cols);
        if (with_ext && s >= 2) tau_reach(s - 2, sb.t_data[i], opts);
        if (i < h.n_smooth) {
          int poly2 = chd_locate(tend[s].data(), sb.sp[s].npoly(), sb.t_data[i] + p.dt, &tl);
          for (int q = 0; q < 12; ++q) cols.push_back(sb.sp[s].var[poly2 * 6 + q]);
          if (with_ext) ext_nodes(s, poly2, sb.t_data[i] + p.dt, cols);
          if (with_ext && s >= 2) tau_reach(s - 2, sb.t_data[i] + p.dt, opts);
        }
        for_options(cols, opts, clique);
      }
    }
    w = std::max(w, w_fix);
    h.w = w;
    h.w_fix = w_fix;
    // scored by the fixed-duration stages (most of the iterations)
    const double grp = (w_fix + 7) / 8 + 1 + (h.nb_fix + 1 + 7) / 8;
    return (double)((h.Na + 7) / 8) * grp * grp;
  };
  const double cand[4] = {0.15, 0.35, 0.5, 1e30};
  int best = 0;
  double best_cost = 0;
  for (int ci = 0; ci < 4; ++ci) {
    const double cst = order_kkt(cand[ci]);
    if (ci == 0 || cst < 0.9 * best_cost) best = ci, best_cost = cst;   // leave the default unless clearly better
  }
  order_kkt(cand[best]);
  if (h.dur_band && !kkt_fits(h.w, h.nb)) return 1;
  return 0;
}

}  // namespace

int chd_build_layout(const chd_phys_problem* problems, int batch, const chd_phys_weights* w, ChdHostBatch& hb,
                     int stage3_band_above) {
  std::vector<SeqBuild> sbs(batch);
  {
    // sequences are independent: build their tables on the host cores in parallel (end-to-end latency of a batch)
    const int nth = std::max(1, std::min<int>({batch, 16, (int)std::thread::hardware_concurrency()}));
    std::vector<int> rcs(batch, 0);
    std::atomic<int> next(0);
    auto work = [&]() {
      for (int i = next.fetch_add(1); i < batch; i = next.fetch_add(1)) {
        rcs[i] = build_sequence(problems[i], sbs[i], stage3_band_above);
        if (rcs[i] == 1) {   // banded switch times too wide for the kernels: the layout without them
          sbs[i] = SeqBuild();
          rcs[i] = build_sequence(problems[i], sbs[i], -1);
        }
      }
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < nth; ++t) pool.emplace_back(work);
    work();
    for (auto& t : pool) t.join();
    for (int i = 0; i < batch; ++i)
      if (rcs[i]) return rcs[i];
  }
  // The kernels' limits hold for the batch (band strides from the widest band, border from the largest one): while it
  // does not fit, the banded sequence with the widest band is built again without banded switch times.  A batch that
  // does not fit without any banded sequence is left to batch creation's own checks, as without the option.
  while (true) {
    int w_max = 0, nb_max = 0, widest = -1;
    for (int i = 0; i < batch; ++i) {
      w_max = std::max(w_max, sbs[i].h.w), nb_max = std::max(nb_max, sbs[i].h.nb);
      if (sbs[i].h.dur_band && (widest < 0 || sbs[i].h.w > sbs[widest].h.w)) widest = i;
    }
    if (widest < 0 || kkt_fits(w_max, nb_max)) break;
    sbs[widest] = SeqBuild();
    const int rc = build_sequence(problems[widest], sbs[widest], -1);
    if (rc) return rc;
  }
  hb.B = batch;
  auto up = [](int& a, int b) { a = std::max(a, b); };
  for (auto& sb : sbs) {
    up(hb.S, sb.h.n_splines), up(hb.n_max, sb.h.n), up(hb.m_max, sb.h.m), up(hb.slots_max, sb.h.nslots);
    up(hb.sets_max, sb.h.nsets), up(hb.tab_max, (int)sb.itab.size()), up(hb.F_max, sb.h.F), up(hb.Kd_max, sb.h.n_dyn);
    up(hb.Kr_max, sb.h.n_rom), up(hb.Na_max, sb.h.Na), up(hb.nb_max, sb.h.nb), up(hb.w_max, sb.h.w), up(hb.w_fix_max, sb.h.w_fix), up(hb.n_ee_max, sb.h.n_ee);
    for (auto& s : sb.sp) up(hb.Pmax, s.npoly());
    up(hb.fo_max, (int)((sb.h.T + 1e-5) / sb.h.dt) + 1);
    for (int ee = 0; ee < sb.h.n_ee; ++ee) up(hb.Ph_max, sb.h.n_phases[ee]);
  }
  hb.tab_max = std::max(hb.tab_max, 1);
  const int B = batch, S = hb.S, Pm = hb.Pmax, Fm = hb.F_max;
  hb.seq.resize(B);
  hb.poly_T.assign((size_t)B * S * Pm, 1.0);
  hb.poly_tend.assign((size_t)B * S * Pm, 1e300);
  hb.node_var.assign((size_t)B * S * (Pm + 1) * 6, -1);
  hb.node_const.assign((size_t)B * S * (Pm + 1) * 6, 0.0);
  hb.par.assign((size_t)B * hb.par_stride(), 0.0);
  hb.t_dyn.assign((size_t)B * hb.Kd_max, 0.0);
  hb.t_rom.assign((size_t)B * hb.Kr_max, 0.0);
  hb.t_data.assign((size_t)B * Fm, 0.0);
  hb.row_lo.assign((size_t)B * hb.m_max, 0.0);
  hb.row_hi.assign((size_t)B * hb.m_max, 0.0);
  hb.row_set.assign((size_t)B * hb.m_max, -1);
  hb.x0.assign((size_t)B * hb.n_max, 0.0);
  hb.itab.assign((size_t)B * hb.tab_max, 0);
  hb.ent_ptr.assign((size_t)B * (hb.m_max + 1), 0);
  hb.ent_col.assign((size_t)B * hb.slots_max, -1);
  hb.ent_row.assign((size_t)B * hb.slots_max, 0);
  hb.col_ptr.assign((size_t)B * (hb.n_max + 1), 0);
  hb.col_ent.assign((size_t)B * hb.slots_max, 0);
  hb.var_kkt.assign((size_t)B * hb.n_max, -1);
  hb.row_kkt.assign((size_t)B * hb.m_max, -1);
  hb.sets.assign((size_t)B * hb.sets_max, ChdSet{-1, 0, 0, 0, 0, 0});
  hb.phase_tend.assign((size_t)B * hb.n_ee_max * hb.Ph_max, 1e300);
  hb.dur0.assign((size_t)B * hb.n_ee_max * hb.Ph_max, 0.0);
  hb.poly_ph.assign((size_t)B * S * Pm, 0);
  for (int i = 0; i < B; ++i) {
    SeqBuild& sb = sbs[i];
    const chd_phys_problem& p = problems[i];
    hb.seq[i] = sb.h;
    for (int s = 0; s < sb.h.n_splines; ++s) {
      const SplineBuild& sp = sb.sp[s];
      double t = 0;
      for (int k = 0; k < sp.npoly(); ++k) {
        t += sp.T[k];
        hb.poly_T[((size_t)i * S + s) * Pm + k] = sp.T[k];
        hb.poly_tend[((size_t)i * S + s) * Pm + k] = t;
      }
      for (int k = 0; k < (int)sp.info.size(); ++k)
        hb.poly_ph[((size_t)i * S + s) * Pm + k] = sp.info[k].phase | (sp.info[k].poly_in_phase << 12) | (sp.info[k].n_polys << 20);
      std::copy(sp.var.begin(), sp.var.end(), hb.node_var.begin() + ((size_t)i * S + s) * (Pm + 1) * 6);
      std::copy(sp.cval.begin(), sp.cval.end(), hb.node_const.begin() + ((size_t)i * S + s) * (Pm + 1) * 6);
    }
    {
      const double* d = p.ee_durations;
      for (int ee = 0; ee < sb.h.n_ee; ++ee) {
        double t = 0;
        for (int k = 0; k < p.ee_n_phases[ee]; ++k) {
          t += d[k];
          hb.phase_tend[((size_t)i * hb.n_ee_max + ee) * hb.Ph_max + k] = t;
          hb.dur0[((size_t)i * hb.n_ee_max + ee) * hb.Ph_max + k] = d[k];
        }
        d += p.ee_n_phases[ee];
      }
    }
    double* par = hb.par.data() + (size_t)i * hb.par_stride();
    const int F = sb.h.F;
    std::copy(p.hip_left, p.hip_left + 3 * F, par + 0);
    std::copy(p.hip_right, p.hip_right + 3 * F, par + 3 * Fm);
    std::copy(p.inertia, p.inertia + 6 * F, par + 6 * Fm);
    std::copy(p.base_lin, p.base_lin + 3 * F, par + 12 * Fm);
    std::copy(p.base_ang, p.base_ang + 3 * F, par + 15 * Fm);
    for (int ee = 0; ee < sb.h.n_ee; ++ee)
      std::copy(p.ee_pos + (size_t)ee * 3 * F, p.ee_pos + (size_t)(ee + 1) * 3 * F, par + (18 + 3 * ee) * Fm);
    std::copy(sb.t_dyn.begin(), sb.t_dyn.end(), hb.t_dyn.begin() + (size_t)i * hb.Kd_max);
    std::copy(sb.t_rom.begin(), sb.t_rom.end(), hb.t_rom.begin() + (size_t)i * hb.Kr_max);
    std::copy(sb.t_data.begin(), sb.t_data.end(), hb.t_data.begin() + (size_t)i * Fm);
    std::copy(sb.row_lo.begin(), sb.row_lo.end(), hb.row_lo.begin() + (size_t)i * hb.m_max);
    std::copy(sb.row_hi.begin(), sb.row_hi.end(), hb.row_hi.begin() + (size_t)i * hb.m_max);
    std::copy(sb.row_set.begin(), sb.row_set.end(), hb.row_set.begin() + (size_t)i * hb.m_max);
    std::copy(sb.x0.begin(), sb.x0.end(), hb.x0.begin() + (size_t)i * hb.n_max);
    std::copy(sb.itab.begin(), sb.itab.end(), hb.itab.begin() + (size_t)i * hb.tab_max);
    std::copy(sb.ent_ptr.begin(), sb.ent_ptr.end(), hb.ent_ptr.begin() + (size_t)i * (hb.m_max + 1));
    for (int r = sb.h.m + 1; r <= hb.m_max; ++r) hb.ent_ptr[(size_t)i * (hb.m_max + 1) + r] = sb.h.nslots;
    std::copy(sb.ent_col.begin(), sb.ent_col.end(), hb.ent_col.begin() + (size_t)i * hb.slots_max);
    {
      // column-oriented view of the same slots: J^T y and the right-hand side are gathered per variable on the device
      int* erow = hb.ent_row.data() + (size_t)i * hb.slots_max;
      int* cptr = hb.col_ptr.data() + (size_t)i * (hb.n_max + 1);
      int* cent = hb.col_ent.data() + (size_t)i * hb.slots_max;
      for (int r = 0; r < sb.h.m; ++r)
        for (int e = sb.ent_ptr[r]; e < sb.ent_ptr[r + 1]; ++e) erow[e] = r;
      std::vector<int> cnt(hb.n_max + 1, 0);
      for (int e = 0; e < sb.h.nslots; ++e)
        if (sb.ent_col[e] >= 0) cnt[sb.ent_col[e] + 1]++;
      for (int v = 0; v < hb.n_max; ++v) cnt[v + 1] += cnt[v];
      std::copy(cnt.begin(), cnt.end(), cptr);
      for (int e = 0; e < sb.h.nslots; ++e)
        if (sb.ent_col[e] >= 0) cent[cnt[sb.ent_col[e]]++] = e;
    }
    std::copy(sb.var_kkt.begin(), sb.var_kkt.end(), hb.var_kkt.begin() + (size_t)i * hb.n_max);
    std::copy(sb.row_kkt.begin(), sb.row_kkt.end(), hb.row_kkt.begin() + (size_t)i * hb.m_max);
    std::copy(sb.sets.begin(), sb.sets.end(), hb.sets.begin() + (size_t)i * hb.sets_max);
  }
  // staged schedule (phys_optim.cpp:554-749, SURVEY Appendix B): six stage rows per sequence, which differ only in the
  // user weights (stages 2.1, 2.2, 3 and 4); stages 1.1 and 1.2 keep their fixed weights
  const unsigned ACC = CHD_MASK(CHD_SET_ACC), LEG = CHD_MASK(CHD_SET_TERRAIN) | CHD_MASK(CHD_SET_ROM),
                 HEEL = CHD_MASK(CHD_SET_HEEL), DYN = CHD_MASK(CHD_SET_DYN) | CHD_MASK(CHD_SET_FORCE),
                 HGT = CHD_MASK(CHD_SET_HEIGHT);
  hb.stage.resize((size_t)B * 6);
  for (int i = 0; i < B; ++i) {
    const chd_phys_weights& wt = w[i];
    ChdStageCfg* st = hb.stage.data() + (size_t)i * 6;
    ChdStageCfg s1 = {ACC, {1.0, 1.0, 1.0}, {0.1, 0.1, 0.1}, {0, 0, 0}, 7000, 0.0};
    ChdStageCfg s2 = {ACC | LEG | DYN | HEEL, {wt.w_com_lin, wt.w_com_ang, wt.w_ee}, {0.001, 0.001, wt.w_smooth},
                      {0.0001, 0.0001, 0.0001}, 7000, 0.0};
    st[CHD_STAGE_11] = s1;
    st[CHD_STAGE_12] = s1;
    st[CHD_STAGE_12].set_mask = ACC | LEG | HEEL;
    st[CHD_STAGE_21] = s2;
    st[CHD_STAGE_22] = s2;
    st[CHD_STAGE_22].set_mask |= HGT;
    st[CHD_STAGE_22].max_iter = 2500;
    // stage 3 (phys_optim.cpp:663-711): every set of 2.2 + TotalTime (+ the duration bounds as rows), no acceleration
    // smoothing (:693, vel_smooth_cost.cpp:72-79), DurationCost (:696-703)
    st[CHD_STAGE_3] = st[CHD_STAGE_22];
    st[CHD_STAGE_3].set_mask |= CHD_MASK(CHD_SET_TOTTIME) | CHD_MASK(CHD_SET_DURPOS);
    for (int q = 0; q < 3; ++q) st[CHD_STAGE_3].w_acc[q] = 0.0;
    st[CHD_STAGE_3].w_dur = wt.w_dur;
    st[CHD_STAGE_3].max_iter = 2000;
    st[CHD_STAGE_4] = st[CHD_STAGE_22];
    st[CHD_STAGE_4].max_iter = 7000;
  }
  return 0;
}
