// TEST INFRASTRUCTURE ONLY -- CPU oracle of the interior-point loop ("chd-ipm", DESIGN.md section IPM).
//
// Single-threaded C++ statement of the interior-point algorithm the CUDA solver runs: IPOPT's primal-dual barrier framework (slack
// reformulation, fraction-to-the-boundary, monotone barrier update, scaled optimality error and
// termination test of phys_optim.cpp:568-578's options, gradient-based scaling) with a Gauss-Newton
// Hessian model, Levenberg-Marquardt regularisation and a filter line search without restoration.
// It is generic over the NLP callbacks of towr_problem.cpp (the role ifopt plays for IPOPT) and solves
// the condensed KKT system with an unpivoted banded LDL^T plus dense border -- written independently of
// the CUDA implementation (row-oriented storage, scalar loops).
//
// PARITY UNPINNED: the reference's own solver stack (IPOPT + MA57 + L-BFGS) cannot be built offline; this
// oracle pins the CUDA solver to the same algorithm run on the CPU, not to IPOPT iterates.
// Experimental switches (environment variables, all off by default; the parity tests use the defaults):
//   CHD_EXACT=1      exact bilinear momentum curvature of the dynamics rows + inertia control (negative pivots of the
//                    band LDL^T must equal the number of equality rows, otherwise delta_w *= CHD_DW_INERTIA (8))
//   CHD_DW_MIN, CHD_DW_DEC   floor / decay factor of the Levenberg-Marquardt regularisation (1e-8, 3)
//   CHD_MU_RESCUE=1  lower the barrier floor (x1/5, >= 1e-9) only when every test but the unscaled complementarity passes
//   CHD_MU_MIN, CHD_MU_SF    barrier floor (default min(tol, compl_inf_tol) / 11; IPOPT's own default is 1e-11)
//   CHD_NDUR, CHD_DREG       proximal term on the last CHD_NDUR variables (stage-3 duration variables)
// They document the convergence studies summarised in DESIGN.md section 4.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

extern "C" {
void chdo_set_stage(void* h, int st);
int chdo_n(void* h);
int chdo_m(void* h);
void chdo_get_x(void* h, double* x);
void chdo_set_x(void* h, const double* x);
void chdo_var_bounds(void* h, double* lo, double* hi);
int chdo_num_constraint_sets(void* h);
int chdo_constraint_set_rows(void* h, int i);
const char* chdo_constraint_set_name(void* h, int i);
void chdo_con_bounds(void* h, double* lo, double* hi);
double chdo_cost(void* h);
void chdo_grad(void* h, double* g);
void chdo_cons(void* h, double* g);
int chdo_jac(void* h, int* ri, int* ci, double* vals);
int chdo_cost_hessian(void* h, int* ri, int* ci, double* vals);
int chdo_lag_hessian(void* h, const double* y, int* ri, int* ci, double* vals);
void chdo_row_times(void* h, double* t);
void chdo_var_times(void* h, double* t0, double* t1);
int chdo_dur_blocks(void* h, int* off, int* cnt);
void chdo_var_set_sizes(void* h, int* out);
int chdo_n_ee(void* h);
void chdo_init_durations(void* h, double* d);   // the free durations (first P-1 of every foot) of the input contact schedule
}

namespace {

const double kInf = 1e19;
struct Opts {
  double tol = 1e-3, constr_viol_tol = 1e-4, dual_inf_tol = 1.0, compl_inf_tol = 1e-4;
  double mu_init = 0.1, kappa_eps = 10.0, kappa_mu = 0.2, theta_mu = 1.5, tau_min = 0.99;
  double kappa1 = 1e-2, kappa2 = 1e-2, kappa_sigma = 1e10, s_max = 100.0, scal_max_grad = 100.0, bound_relax = 1e-8;
  double delta_w0 = 1e-4, delta_c = 1e-8, dw_min = 1e-8, dw_max = 1e4, dw_inc = 4.0, dw_dec = 3.0;
  int max_backtrack = 25;
  double gamma_theta = 1e-5, gamma_phi = 1e-5, s_phi = 2.3, s_theta = 1.1, eta_phi = 1e-8;
  int filt_max = 24;
};

struct Triplets {
  std::vector<int> r, c;
  std::vector<double> v;
};

// symmetric arrowhead matrix: band part (row-major, row i holds columns i-w..i) + dense border rows
struct Arrow {
  int Na = 0, nb = 0, w = 0, n_neg = 0;   // n_neg: negative pivots of the last factorisation (band part)
  std::vector<double> band, bord, corn, rhs;  // band[i*(w+1) + (w-(i-j))], bord[b*Na + j], corn[b*nb + b2] (lower), rhs[Na+nb]
  void init(int Na_, int nb_, int w_) {
    Na = Na_, nb = nb_, w = w_;
    band.assign((size_t)Na * (w + 1), 0.0);
    bord.assign((size_t)nb * Na, 0.0);
    corn.assign((size_t)nb * nb, 0.0);
    rhs.assign(Na + nb, 0.0);
  }
  void add(int i, int j, double v) {
    if (i < j) std::swap(i, j);
    if (i < Na) band[(size_t)i * (w + 1) + (w - (i - j))] += v;
    else if (j < Na) bord[(size_t)(i - Na) * Na + j] += v;
    else corn[(size_t)(i - Na) * nb + (j - Na)] += v;
  }
  // in-place LDL^T without pivoting and solve; returns false on a zero / non-finite pivot
  bool solve(std::vector<double>& x) {
    const int W = w + 1;
    auto A = [&](int i, int j) -> double& { return band[(size_t)i * W + (w - (i - j))]; };
    std::vector<double> z(rhs);
    n_neg = 0;
    for (int k = 0; k < Na; ++k) {
      const double d = A(k, k);
      n_neg += d < 0.0;
      if (!(std::fabs(d) > 1e-300) || !std::isfinite(d)) { if (getenv("CHDO_DEBUG")) fprintf(stderr, "band pivot %d = %g\n", k, d); return false; }
      const int lim = std::min(w, Na - 1 - k);
      // column k of L in the band
      for (int i = k + 1; i <= k + lim; ++i) {
        const double aik = A(i, k);
        if (aik == 0.0) continue;
        const double l = aik / d;
        for (int j = k + 1; j <= i; ++j) A(i, j) -= l * A(j, k);
        z[i] -= l * z[k];
      }
      for (int b = 0; b < nb; ++b) {
        const double abk = bord[(size_t)b * Na + k];
        if (abk == 0.0) continue;
        const double l = abk / d;
        for (int j = k + 1; j <= k + lim; ++j) bord[(size_t)b * Na + j] -= l * A(j, k);
        for (int b2 = 0; b2 <= b; ++b2) corn[(size_t)b * nb + b2] -= l * bord[(size_t)b2 * Na + k];
        z[Na + b] -= l * z[k];
      }
      // store scaled column (after all updates that use the unscaled values)
      for (int i = k + 1; i <= k + lim; ++i) A(i, k) /= d;
      for (int b = 0; b < nb; ++b) bord[(size_t)b * Na + k] /= d;
    }
    // border Schur complement: LDL^T of corn
    for (int k = 0; k < nb; ++k) {
      const double d = corn[(size_t)k * nb + k];
      if (!(d > 0.0) || !std::isfinite(d)) { if (getenv("CHDO_DEBUG")) fprintf(stderr, "border pivot %d = %g\n", k, d); return false; }
      for (int i = k + 1; i < nb; ++i) {
        const double l = corn[(size_t)i * nb + k] / d;
        for (int j = k + 1; j <= i; ++j) corn[(size_t)i * nb + j] -= l * corn[(size_t)j * nb + k];
        z[Na + i] -= l * z[Na + k];
      }
      for (int i = k + 1; i < nb; ++i) corn[(size_t)i * nb + k] /= d;  // scale after the unscaled column was used
    }
    x.assign(Na + nb, 0.0);
    for (int k = nb - 1; k >= 0; --k) {
      double v = z[Na + k] / corn[(size_t)k * nb + k];
      for (int i = k + 1; i < nb; ++i) v -= corn[(size_t)i * nb + k] * x[Na + i];
      x[Na + k] = v;
    }
    for (int k = Na - 1; k >= 0; --k) {
      double v = z[k] / A(k, k);
      const int lim = std::min(w, Na - 1 - k);
      for (int i = k + 1; i <= k + lim; ++i) v -= A(i, k) * x[i];
      for (int b = 0; b < nb; ++b) v -= bord[(size_t)b * Na + k] * x[Na + b];
      x[k] = v;
    }
    return true;
  }
};

// primal-dual state a stage leaves behind, keyed by constraint-set name (the stages stack their sets in different orders)
struct WarmState {
  bool valid = false;
  std::vector<std::string> names;
  std::vector<int> off, rows;
  std::vector<double> y, s, zL, zU, sc;
  double sf = 1.0, mu = 0.1, delta_w = 1e-4;
};

struct Solver {
  WarmState* ws = nullptr;   // state of the previous stage of the same problem (nullptr / !valid: cold start)
  bool warm = false;
  void* h;
  Opts o;
  int n = 0, m = 0;
  int m0 = 0;                 // rows of the NLP's own constraint sets; rows m0..m-1 are the duration lower bounds d_k >= 0
  std::vector<int> durk;      // per variable: -1, or k = index of the phase duration inside its PhaseDurations set
  std::vector<int> dur_vars;  // duration variables in stacking order
  std::vector<double> xlo, xhi, cl, cu;
  std::vector<char> fixed, eq, hasL, hasU, dist_row, dyn_row;
  std::vector<int> vk, rk;  // KKT ordering
  int Na = 0, nb = 0, w = 0;
  // CSR Jacobian
  std::vector<int> jp, jc;
  std::vector<double> jv;

  void eval_jac() {
    int nnz = chdo_jac(h, nullptr, nullptr, nullptr);
    std::vector<int> ri(nnz), ci(nnz);
    jv.assign(nnz, 0.0);
    chdo_jac(h, ri.data(), ci.data(), jv.data());
    jp.assign(m + 1, 0);
    for (int k = 0; k < nnz; ++k) jp[ri[k] + 1]++;
    for (int r = 0; r < m0; ++r) jp[r + 1] += jp[r];
    jc = ci;  // triplets are row sorted
    if (dur_vars.empty()) return;
    // duration lower bounds as rows, then the change of variables d = D tau (switch times): column tau_k of a row is
    // (column d_k) - (column d_{k+1}); the dense "all earlier phases" columns of towr's GetJacobianOfPos cancel exactly
    for (size_t i = 0; i < dur_vars.size(); ++i) jc.push_back(dur_vars[i]), jv.push_back(1.0), jp[m0 + i + 1] = (int)jc.size();
    std::vector<int> njp(m + 1, 0), njc;
    std::vector<double> njv, acc(n, 0.0);
    std::vector<int> touched;
    std::vector<char> mark(n, 0);
    for (int r = 0; r < m; ++r) {
      touched.clear();
      auto put = [&](int c, double v) {
        if (!mark[c]) mark[c] = 1, touched.push_back(c);
        acc[c] += v;
      };
      for (int e = jp[r]; e < jp[r + 1]; ++e) {
        const int c = jc[e];
        put(c, jv[e]);
        if (durk[c] > 0) put(c - 1, -jv[e]);
      }
      std::sort(touched.begin(), touched.end());
      for (int c : touched) {
        if (acc[c] != 0.0) njc.push_back(c), njv.push_back(acc[c]);
        acc[c] = 0.0, mark[c] = 0;
      }
      njp[r + 1] = (int)njc.size();
    }
    jp.swap(njp), jc.swap(njc), jv.swap(njv);
  }
  void to_tau_grad(std::vector<double>& g) const {   // g_tau_k = g_d_k - g_d_{k+1}
    for (size_t i = 0; i + 1 < dur_vars.size(); ++i) {
      const int j = dur_vars[i];
      if (durk[j + 1] == durk[j] + 1) g[j] -= g[j + 1];
    }
  }
  void to_tau_hess(Triplets& t) const {
    if (dur_vars.empty()) return;
    Triplets o;
    auto img = [&](int v, int (&id)[2], double (&sg)[2]) {
      id[0] = v, sg[0] = 1.0;
      if (durk[v] > 0) { id[1] = v - 1, sg[1] = -1.0; return 2; }
      return 1;
    };
    for (size_t k = 0; k < t.v.size(); ++k) {
      int ir[2], ic[2];
      double sr[2], scv[2];
      const int nr = img(t.r[k], ir, sr), nc = img(t.c[k], ic, scv);
      for (int a = 0; a < nr; ++a)
        for (int b = 0; b < nc; ++b) o.r.push_back(ir[a]), o.c.push_back(ic[b]), o.v.push_back(sr[a] * scv[b] * t.v[k]);
    }
    t = o;
  }
  Triplets hess(bool cost, const double* y) {
    Triplets t;
    int nnz = cost ? chdo_cost_hessian(h, nullptr, nullptr, nullptr) : chdo_lag_hessian(h, y, nullptr, nullptr, nullptr);
    t.r.resize(nnz), t.c.resize(nnz), t.v.resize(nnz);
    if (cost) chdo_cost_hessian(h, t.r.data(), t.c.data(), t.v.data());
    else chdo_lag_hessian(h, y, t.r.data(), t.c.data(), t.v.data());
    to_tau_hess(t);
    return t;
  }

  void ordering() {
    // time-sorted band; variables that live longer than 0.15 s (stance positions) go to the border
    std::vector<double> t0(n), t1(n), rt(m);
    chdo_var_times(h, t0.data(), t1.data());
    chdo_row_times(h, rt.data());
    struct Key {
      double t;
      int kind, id;
    };
    std::vector<Key> keys;
    std::vector<int> border;
    vk.assign(n, -1);
    rk.assign(m, -1);
    for (int v = 0; v < n; ++v) {
      if (fixed[v]) continue;
      if (t1[v] - t0[v] > 0.15) border.push_back(v);
      else keys.push_back({0.5 * (t0[v] + t1[v]), 0, v});
    }
    for (int r = 0; r < m; ++r)
      if (eq[r]) keys.push_back({rt[r] + 1e-6, 1, r});
    std::stable_sort(keys.begin(), keys.end(), [](const Key& a, const Key& b) { return a.t < b.t; });
    for (size_t i = 0; i < keys.size(); ++i) (keys[i].kind == 0 ? vk[keys[i].id] : rk[keys[i].id]) = (int)i;
    Na = (int)keys.size();
    nb = (int)border.size();
    for (int j = 0; j < nb; ++j) vk[border[j]] = Na + j;
  }
  // half bandwidth needed by the current patterns
  int bandwidth(const Triplets& W1, const Triplets& W2) {
    int bw = 0;
    auto upd = [&](int a, int b) {
      if (a < 0 || b < 0 || a >= Na || b >= Na) return;
      bw = std::max(bw, std::abs(a - b));
    };
    for (int r = 0; r < m; ++r) {
      if (eq[r]) {
        for (int e = jp[r]; e < jp[r + 1]; ++e) upd(rk[r], vk[jc[e]]);
      } else {
        int lo = 1 << 30, hi = -1;
        for (int e = jp[r]; e < jp[r + 1]; ++e) {
          int k = vk[jc[e]];
          if (k >= 0 && k < Na) lo = std::min(lo, k), hi = std::max(hi, k);
        }
        if (hi >= 0) bw = std::max(bw, hi - lo);
      }
    }
    for (size_t k = 0; k < W1.v.size(); ++k) upd(vk[W1.r[k]], vk[W1.c[k]]);
    for (size_t k = 0; k < W2.v.size(); ++k) upd(vk[W2.r[k]], vk[W2.c[k]]);
    return bw;
  }

  int run(int stage, int max_iter, double* stats, int verbose) {
    chdo_set_stage(h, stage);
    n = chdo_n(h), m0 = chdo_m(h);
    durk.assign(n, -1);
    dur_vars.clear();
    {
      int off[8], cnt[8];
      const int nblk = chdo_dur_blocks(h, off, cnt);
      for (int b = 0; b < nblk; ++b)
        for (int k = 0; k < cnt[b]; ++k) durk[off[b] + k] = k, dur_vars.push_back(off[b] + k);
    }
    m = m0 + (int)dur_vars.size();
    std::vector<double> x(n);
    chdo_get_x(h, x.data());
    xlo.assign(n, 0), xhi.assign(n, 0);
    chdo_var_bounds(h, xlo.data(), xhi.data());
    fixed.assign(n, 0);
    for (int i = 0; i < n; ++i)
      if (xlo[i] == xhi[i]) fixed[i] = 1, x[i] = xlo[i];
    cl.assign(m, 0), cu.assign(m, 0);
    chdo_con_bounds(h, cl.data(), cu.data());
    for (int r = m0; r < m; ++r) cl[r] = 0.0, cu[r] = 1e20;   // PhaseDurations bounds (0, 500) of parameters.cpp:60: the upper one is implied by the TotalTime rows
    eq.assign(m, 0), hasL.assign(m, 0), hasU.assign(m, 0), dist_row.assign(m, 0), dyn_row.assign(m, 0);
    for (int r = 0; r < m; ++r) {
      eq[r] = cl[r] == cu[r];
      hasL[r] = !eq[r] && cl[r] > -kInf;
      hasU[r] = !eq[r] && cu[r] < kInf;
    }
    {
      int off = 0;
      for (int i = 0; i < chdo_num_constraint_sets(h); ++i) {
        std::string nm = chdo_constraint_set_name(h, i);
        int rows = chdo_constraint_set_rows(h, i);
        if (nm.rfind("leg-length", 0) == 0 || nm.rfind("ee-dist", 0) == 0)
          for (int r = off; r < off + rows; ++r) dist_row[r] = 1;
        if (nm == "dynamic")
          for (int r = off; r < off + rows; ++r) dyn_row[r] = 1;
        off += rows;
      }
    }
    ordering();
    auto evaluate = [&](const std::vector<double>& xx, double& f, std::vector<double>& c) {
      chdo_set_x(h, xx.data());
      f = chdo_cost(h);
      c.resize(m);
      chdo_cons(h, c.data());
      for (size_t i = 0; i < dur_vars.size(); ++i) c[m0 + i] = xx[dur_vars[i]];
    };
    double f;
    std::vector<double> c, g(n);
    evaluate(x, f, c);
    chdo_grad(h, g.data());
    to_tau_grad(g);
    eval_jac();
    // gradient based scaling
    double gmax = 0;
    for (int i = 0; i < n; ++i)
      if (!fixed[i]) gmax = std::max(gmax, std::fabs(g[i]));
    const bool use_warm = warm && ws && ws->valid;
    const double sf = use_warm ? ws->sf : (gmax > o.scal_max_grad ? o.scal_max_grad / gmax : 1.0);
    std::vector<double> sc(m, 1.0), dL(m), dU(m), s(m), y(m, 0.0), zL(m, 0.0), zU(m, 0.0);
    // warm start: rows of constraint sets the previous stage also had inherit scaling, slack and multipliers
    std::vector<int> wsrc(m, -1);
    std::vector<std::string> set_names;
    std::vector<int> set_off, set_rows;
    {
      int off = 0;
      for (int i = 0; i < chdo_num_constraint_sets(h); ++i) {
        set_names.push_back(chdo_constraint_set_name(h, i));
        set_off.push_back(off), set_rows.push_back(chdo_constraint_set_rows(h, i));
        if (use_warm)
          for (size_t q = 0; q < ws->names.size(); ++q)
            if (ws->names[q] == set_names.back() && ws->rows[q] == set_rows.back())
              for (int r = 0; r < set_rows.back(); ++r) wsrc[off + r] = ws->off[q] + r;
        off += set_rows.back();
      }
    }
    const double mu_start = use_warm ? std::max(ws->mu, getenv("CHD_WARM_MU") ? atof(getenv("CHD_WARM_MU")) : 0.0) : o.mu_init;
    int n_bounds = 0;
    for (int r = 0; r < m; ++r) {
      double rm = 0;
      for (int e = jp[r]; e < jp[r + 1]; ++e)
        if (!fixed[jc[e]]) rm = std::max(rm, std::fabs(jv[e]));
      sc[r] = std::max(rm > o.scal_max_grad ? o.scal_max_grad / rm : 1.0, 1e-8);
      if (wsrc[r] >= 0) sc[r] = ws->sc[wsrc[r]];
      const double lo = cl[r] * sc[r], hi = cu[r] * sc[r], d = sc[r] * c[r];
      if (eq[r]) {
        dL[r] = lo, dU[r] = hi, s[r] = d;
        continue;
      }
      dL[r] = hasL[r] ? lo - o.bound_relax * std::max(1.0, std::fabs(lo)) : -INFINITY;
      dU[r] = hasU[r] ? hi + o.bound_relax * std::max(1.0, std::fabs(hi)) : INFINITY;
      double sv = d;
      if (hasL[r]) {
        double pL = o.kappa1 * std::max(1.0, std::fabs(dL[r]));
        if (hasU[r]) pL = std::min(pL, o.kappa2 * (dU[r] - dL[r]));
        sv = std::max(sv, dL[r] + pL);
      }
      if (hasU[r]) {
        double pU = o.kappa1 * std::max(1.0, std::fabs(dU[r]));
        if (hasL[r]) pU = std::min(pU, o.kappa2 * (dU[r] - dL[r]));
        sv = std::min(sv, dU[r] - pU);
      }
      s[r] = sv;
      zL[r] = hasL[r] ? 1.0 : 0.0;
      zU[r] = hasU[r] ? 1.0 : 0.0;
      if (use_warm) {   // new rows of a warm-started stage start on the central path of the inherited barrier parameter
        if (hasL[r]) zL[r] = mu_start / (sv - dL[r]);
        if (hasU[r]) zU[r] = mu_start / (dU[r] - sv);
      }
      n_bounds += hasL[r] + hasU[r];
    }
    if (use_warm)
      for (int r = 0; r < m; ++r) {
        const int q = wsrc[r];
        if (q < 0) continue;
        y[r] = ws->y[q];
        if (!eq[r]) s[r] = ws->s[q], zL[r] = ws->zL[q], zU[r] = ws->zU[q];
      }
    double mu = mu_start, delta_w = use_warm ? std::max(ws->delta_w, o.delta_w0) : o.delta_w0, mu_filter = -1.0, theta_max = 0, theta_min = 0;
    double mu_min = getenv("CHD_MU_MIN") ? atof(getenv("CHD_MU_MIN")) : std::min(o.tol, o.compl_inf_tol) / (o.kappa_eps + 1.0);
    if (getenv("CHD_MU_SF")) mu_min = std::min(o.tol, o.compl_inf_tol * sf) / (o.kappa_eps + 1.0);   // the unscaled complementarity test must be reachable
    if (verbose) printf("sf %.4f mu_min %.3e\n", sf, mu_min);
    std::vector<std::pair<double, double>> filt;
    int status = -1, it = 0, ls_fail = 0;
    double E0 = 0, violu = 0, dual_u = 0, compl_u = 0;
    std::vector<double> rx(n), dx(n), ds(m), dy(m), dzL(m), dzU(m), sol, ypos(m), xt(n), ct;
    Arrow K;
    const bool exact_curv = getenv("CHD_EXACT") != nullptr;
    const double dw_inertia = getenv("CHD_DW_INERTIA") ? atof(getenv("CHD_DW_INERTIA")) : 8.0;
    int n_eq_rows = 0, n_inertia = 0;
    for (int r = 0; r < m; ++r) n_eq_rows += eq[r] && rk[r] >= 0 && rk[r] < Na;
    if (getenv("CHD_DW_MIN")) o.dw_min = atof(getenv("CHD_DW_MIN"));
    if (getenv("CHD_DW_DEC")) o.dw_dec = atof(getenv("CHD_DW_DEC"));
    const double nl_ke = dur_vars.empty() ? 0.0 : (getenv("CHD_NL_KE") ? atof(getenv("CHD_NL_KE")) : 1.0);   // stage 3 only (CHD_NL_GUARD in chd_dev.h)
    const double nl_fl = getenv("CHD_NL_FL") ? atof(getenv("CHD_NL_FL")) : 1e-4;
    double theta_ref = 0.0;
    const int af_n = getenv("CHD_AF_N") ? atoi(getenv("CHD_AF_N")) : 10;   // CHD_AF_N / CHD_AF_MIN of the product (csrc/chd_dev.h)
    const double af_min = getenv("CHD_AF_MIN") ? atof(getenv("CHD_AF_MIN")) : 1e-10;
    double dw_floor = o.dw_min, af_E = 0.0;
    int af_cnt = 0, af_it = 0;
    bool af_off = false;
    const double polish_dw = getenv("CHD_POLISH") ? atof(getenv("CHD_POLISH")) : 1.0;   // CHD_DW_POLISH of the product (csrc/chd_dev.h)
    int n_polish = 0;
    const double du_unobs = getenv("CHD_DU") ? atof(getenv("CHD_DU")) : 1e-4;   // CHD_DW_UNOBS of the product (csrc/chd_dev.h)
    int mot_lo = 0, mot_hi = 0;
    {
      const int ne = chdo_n_ee(h);
      std::vector<int> szs(2 + 3 * ne);
      chdo_var_set_sizes(h, szs.data());
      mot_lo = szs[0] + szs[1];
      mot_hi = mot_lo;
      for (int e = 0; e < ne; ++e) mot_hi += szs[2 + e];
    }
    const double tau_trust = getenv("CHD_TAU_TRUST") ? atof(getenv("CHD_TAU_TRUST")) : 0.04;
    std::vector<double> x_init_dur(dur_vars.size());
    if (!dur_vars.empty()) chdo_init_durations(h, x_init_dur.data());
    const double rt0 = getenv("CHD_RT0") ? atof(getenv("CHD_RT0")) : 0.0, rt_dec = getenv("CHD_RT_DEC") ? atof(getenv("CHD_RT_DEC")) : 3.0;
    const double rt_min = getenv("CHD_RT_MIN") ? atof(getenv("CHD_RT_MIN")) : 0.0;
    double rho_tau = dur_vars.empty() ? 0.0 : rt0;
    const int exp_ndur = getenv("CHD_NDUR") ? atoi(getenv("CHD_NDUR")) : 0;
    const double exp_dreg = getenv("CHD_DREG") ? atof(getenv("CHD_DREG")) : 0.0;
    for (it = 0;; ++it) {
      // ---- error measures ----
      for (int i = 0; i < n; ++i) rx[i] = sf * g[i];
      double ysum = 0, zsum = 0, cviol = 0, theta = 0, rs = 0, cmax = -INFINITY, cmin = INFINITY;
      violu = 0;
      for (int r = 0; r < m; ++r) {
        const double d = sc[r] * c[r];
        ysum += std::fabs(y[r]);
        violu = std::max(violu, std::max(cl[r] - c[r], c[r] - cu[r]));
        const double ys = sc[r] * y[r];
        for (int e = jp[r]; e < jp[r + 1]; ++e) rx[jc[e]] += ys * jv[e];
        if (eq[r]) {
          const double re = d - dL[r];
          cviol = std::max(cviol, std::fabs(re)), theta += std::fabs(re);
        } else {
          const double ri = d - s[r];
          cviol = std::max(cviol, std::fabs(ri)), theta += std::fabs(ri);
          rs = std::max(rs, std::fabs(-y[r] - zL[r] + zU[r]));
          zsum += zL[r] + zU[r];
          if (hasL[r]) { double cp = (s[r] - dL[r]) * zL[r]; cmax = std::max(cmax, cp), cmin = std::min(cmin, cp); }
          if (hasU[r]) { double cp = (dU[r] - s[r]) * zU[r]; cmax = std::max(cmax, cp), cmin = std::min(cmin, cp); }
        }
      }
      violu = std::max(violu, 0.0);
      double dual_inf = rs;
      for (int i = 0; i < n; ++i)
        if (!fixed[i]) dual_inf = std::max(dual_inf, std::fabs(rx[i]));
      const double s_d = std::max(o.s_max, (ysum + zsum) / std::max((double)(m + n_bounds), 1.0)) / o.s_max;
      const double s_c = std::max(o.s_max, zsum / std::max((double)n_bounds, 1.0)) / o.s_max;
      auto compl_err = [&](double mm) { return n_bounds > 0 ? std::max(std::fabs(cmax - mm), std::fabs(cmin - mm)) : 0.0; };
      E0 = std::max(std::max(dual_inf / s_d, cviol), compl_err(0.0) / s_c);
      dual_u = dual_inf / sf, compl_u = compl_err(0.0) / sf;
      if (verbose) printf("it %3d f %.6e E0 %.2e viol %.2e dual %.2e mu %.1e dw %.1e rt %.1e\n", it, f, E0, violu, dual_inf, mu, delta_w, rho_tau);
      if (verbose > 2) {
        int im = 0; double nrm = 0; int cnt = 0;
        for (int i = 0; i < n; ++i) if (!fixed[i]) { if (std::fabs(rx[i]) > std::fabs(rx[im]) || fixed[im]) im = i; nrm += rx[i] * rx[i]; cnt += std::fabs(rx[i]) > 0.1 * dual_inf; }
        double ymax = 0; int iy = 0; for (int r = 0; r < m; ++r) if (std::fabs(y[r]) > ymax) ymax = std::fabs(y[r]), iy = r;
{ int iv = 0; double vm = -1; for (int r = 0; r < m; ++r) { double v = std::max(cl[r] - c[r], c[r] - cu[r]); if (v > vm) vm = v, iv = r; }
          int off = 0; std::string nm = "durpos"; for (int q = 0; q < chdo_num_constraint_sets(h); ++q) { int rows = chdo_constraint_set_rows(h, q); if (iv >= off && iv < off + rows) { nm = chdo_constraint_set_name(h, q); nm += "[" + std::to_string(iv - off) + "/" + std::to_string(rows) + "]"; } off += rows; }
          printf("      max viol row %d %s (%.3e) sc %.3e s-d %.3e y %.3e\n", iv, nm.c_str(), vm, sc[iv], s[iv] - sc[iv] * c[iv], y[iv]); }
        printf("      argmax rx %d (%.3e) l2 %.3e count>10%% %d | ymax %.3e at row %d | s_d %.3e\n", im, rx[im], std::sqrt(nrm), cnt, ymax, iy, s_d);
      }
      if (E0 <= o.tol && violu <= o.constr_viol_tol && dual_u <= o.dual_inf_tol && compl_u <= o.compl_inf_tol) {
        status = 0;
        break;
      }
      if (it >= max_iter) {
        status = -1;
        break;
      }
      while (true) {
        const double Emu = std::max(std::max(dual_inf / s_d, cviol), compl_err(mu) / s_c);
        if (Emu <= o.kappa_eps * mu && mu > mu_min) mu = std::max(mu_min, std::min(o.kappa_mu * mu, std::pow(mu, o.theta_mu)));
        else break;
      }
      // experimental (CHD_MU_RESCUE): the scaled error passes but the unscaled complementarity test cannot be met at
      // the barrier floor (large multipliers make s_c > 11): let the barrier parameter go below the floor, gently
      if (getenv("CHD_MU_RESCUE") && E0 <= o.tol && violu <= o.constr_viol_tol && dual_u <= o.dual_inf_tol && compl_u > o.compl_inf_tol &&
          mu <= mu_min * 1.0000001)
        mu_min = std::max(mu_min / 5.0, 1e-9), mu = mu_min;
      // feasibility polish: every test but the unscaled constraint violation passes -> this step only restores
      // feasibility (a large Levenberg-Marquardt weight makes it the least-norm Newton correction of the constraints)
      const bool polish = polish_dw > 0.0 && E0 <= o.tol && dual_u <= o.dual_inf_tol && compl_u <= o.compl_inf_tol && violu > o.constr_viol_tol;
      const double delta_w_state = delta_w;
      if (polish) delta_w = std::max(delta_w, polish_dw), n_polish++;
      const double tau = std::max(o.tau_min, 1.0 - mu);
      if (it == 0) theta_max = 1e4 * std::max(1.0, theta), theta_min = 1e-4 * std::max(1.0, theta), theta_ref = theta;
      if (mu != mu_filter) filt.clear(), mu_filter = mu;
      // ---- condensed KKT ----
      for (int r = 0; r < m; ++r) ypos[r] = (dist_row[r] && sc[r] * y[r] > 1e-8) ? sc[r] * y[r] : 0.0;  // CHD_CURV_MIN
      if (exact_curv)
        for (int r = 0; r < m; ++r)
          if (dyn_row[r]) ypos[r] = sc[r] * y[r];   // exact bilinear momentum terms (indefinite: inertia control below)
      Triplets W1 = hess(true, nullptr), W2 = hess(false, ypos.data());
      w = bandwidth(W1, W2);
      K.init(Na, nb, w);
      for (int i = 0; i < n; ++i)
        if (vk[i] >= 0) K.add(vk[i], vk[i], delta_w + (i >= n - exp_ndur ? exp_dreg : 0.0) + (durk[i] >= 0 ? rho_tau : 0.0)), K.rhs[vk[i]] += -sf * g[i];
      for (size_t k = 0; k < W1.v.size(); ++k) {
        int a = vk[W1.r[k]], b = vk[W1.c[k]];
        if (a >= 0 && b >= 0 && a >= b) K.add(a, b, sf * W1.v[k]);
      }
      if (du_unobs > 0.0) {
        // foot-motion node values no cost sample sees (polynomials shorter than a frame): without curvature of their
        // own the Newton step uses them as free slack and they drift by orders of magnitude; they get a fixed
        // Levenberg-Marquardt weight instead of the adaptive one (what L-BFGS's initial scaling does for IPOPT)
        std::vector<char> seen(n, 0);
        for (size_t k = 0; k < W1.v.size(); ++k)
          if (W1.r[k] == W1.c[k] && sf * W1.v[k] > 1e-14) seen[W1.r[k]] = 1;   // CHD_UNOBS_EPS
        for (int i = mot_lo; i < mot_hi; ++i)
          if (vk[i] >= 0 && !seen[i]) K.add(vk[i], vk[i], du_unobs);
      }
      for (size_t k = 0; k < W2.v.size(); ++k) {
        int a = vk[W2.r[k]], b = vk[W2.c[k]];
        if (a >= 0 && b >= 0 && a >= b) K.add(a, b, W2.v[k]);
      }
      for (int r = 0; r < m; ++r) {
        if (eq[r]) {
          K.add(rk[r], rk[r], -o.delta_c);
          K.rhs[rk[r]] += -(sc[r] * c[r] - dL[r]);
          for (int e = jp[r]; e < jp[r + 1]; ++e) {
            int kc = vk[jc[e]];
            if (kc < 0) continue;
            K.add(rk[r], kc, sc[r] * jv[e]);
            K.rhs[kc] += -sc[r] * y[r] * jv[e];
          }
        } else {
          const double gapL = hasL[r] ? s[r] - dL[r] : 1.0, gapU = hasU[r] ? dU[r] - s[r] : 1.0;
          const double Sig = (hasL[r] ? zL[r] / gapL : 0.0) + (hasU[r] ? zU[r] / gapU : 0.0);
          const double bvec = (hasL[r] ? mu / gapL : 0.0) - (hasU[r] ? mu / gapU : 0.0);
          const double coef = Sig * (sc[r] * c[r] - s[r]) - bvec;
          for (int ea = jp[r]; ea < jp[r + 1]; ++ea) {
            int ka = vk[jc[ea]];
            if (ka < 0) continue;
            const double va = sc[r] * jv[ea];
            K.rhs[ka] += -va * coef;
            for (int eb = jp[r]; eb < jp[r + 1]; ++eb) {
              int kb = vk[jc[eb]];
              if (kb < 0 || ka < kb) continue;
              K.add(ka, kb, Sig * va * sc[r] * jv[eb]);
            }
          }
        }
      }
      const bool ok = K.solve(sol);
      if (ok && exact_curv && K.n_neg != n_eq_rows) {
        // wrong inertia: the step would not be a descent direction for the barrier problem; stiffen and retry
        delta_w = std::min(std::max(delta_w * dw_inertia, 1e-8), o.dw_max * 10);
        n_inertia++;
        if (verbose > 1) printf("      inertia %d != %d -> dw %.1e\n", K.n_neg, n_eq_rows, delta_w);
        if (delta_w > o.dw_max) { status = -2; break; }
        continue;
      }
      if (!ok) {
        if (polish) delta_w = delta_w_state;
        delta_w = std::min(std::max(delta_w * 100.0, 1e-4), o.dw_max * 10);
        ls_fail++;
        if (delta_w > o.dw_max) {
          status = -2;
          break;
        }
        continue;
      }
      // ---- step recovery ----
      for (int i = 0; i < n; ++i) dx[i] = vk[i] >= 0 ? sol[vk[i]] : 0.0;   // step in (nodes, switch times)
      double a_pr = 1.0, a_du = 1.0, dphi = 0, phib = 0;
      for (int i = 0; i < n; ++i) dphi += sf * g[i] * dx[i];
      for (int r = 0; r < m; ++r) {
        if (eq[r]) {
          dy[r] = sol[rk[r]], ds[r] = 0;
          continue;
        }
        double Jdx = 0;
        for (int e = jp[r]; e < jp[r + 1]; ++e) Jdx += jv[e] * dx[jc[e]];
        const double dsr = sc[r] * Jdx + (sc[r] * c[r] - s[r]);
        const double gapL = hasL[r] ? s[r] - dL[r] : 1.0, gapU = hasU[r] ? dU[r] - s[r] : 1.0;
        const double sigL = hasL[r] ? zL[r] / gapL : 0.0, sigU = hasU[r] ? zU[r] / gapU : 0.0;
        const double bvec = (hasL[r] ? mu / gapL : 0.0) - (hasU[r] ? mu / gapU : 0.0);
        ds[r] = dsr;
        dy[r] = (sigL + sigU) * dsr - y[r] - bvec;
        dzL[r] = hasL[r] ? mu / gapL - zL[r] - sigL * dsr : 0.0;
        dzU[r] = hasU[r] ? mu / gapU - zU[r] + sigU * dsr : 0.0;
        if (hasL[r] && dsr < 0) a_pr = std::min(a_pr, -tau * gapL / dsr);
        if (hasU[r] && dsr > 0) a_pr = std::min(a_pr, tau * gapU / dsr);
        if (hasL[r] && dzL[r] < 0) a_du = std::min(a_du, -tau * zL[r] / dzL[r]);
        if (hasU[r] && dzU[r] < 0) a_du = std::min(a_du, -tau * zU[r] / dzU[r]);
        if (hasL[r]) dphi -= mu * dsr / gapL, phib -= mu * std::log(gapL);
        if (hasU[r]) dphi += mu * dsr / gapU, phib -= mu * std::log(gapU);
      }
      const double phi0 = sf * f + phib;
      for (int i = (int)dur_vars.size() - 1; i >= 0; --i) {   // back to phase durations: dd_k = dtau_k - dtau_{k-1}
        const int j = dur_vars[i];
        if (durk[j] > 0) dx[j] -= dx[j - 1];
      }
      // ---- filter line search ----
      double alpha = a_pr, ft = f;
      if (verbose > 1) printf("      a_pr %.3e a_du %.3e dphi %.3e\n", a_pr, a_du, dphi);
      bool accepted = false, ftype = false;
      int ls = 0, nl_rej = 0;
      for (ls = 0; ls < o.max_backtrack; ++ls) {
        for (int i = 0; i < n; ++i) xt[i] = x[i] + alpha * dx[i];
        evaluate(xt, ft, ct);
        double theta_t = 0, bar = 0;
        for (int r = 0; r < m; ++r) {
          const double d = sc[r] * ct[r];
          if (eq[r]) theta_t += std::fabs(d - dL[r]);
          else {
            const double st = s[r] + alpha * ds[r];
            theta_t += std::fabs(d - st);
            if (hasL[r]) bar -= mu * std::log(st - dL[r]);
            if (hasU[r]) bar -= mu * std::log(dU[r] - st);
          }
        }
        const double phit = sf * ft + bar;
        if (verbose > 1) printf("        trial %d alpha %.6e theta_t %.6e phi_t %.9e\n", ls, alpha, theta_t, phit);
        bool okp = std::isfinite(phit) && std::isfinite(theta_t) && theta_t <= theta_max;
        // nonlinearity guard: the linearised constraints predict theta(alpha) = (1 - alpha) theta; the trial point is
        // refused while the second-order error exceeds nl_ke x the predicted decrease (or a small absolute level)
        if (!dur_vars.empty() && okp) {   // trust region of stage 3 (CHD_TAU_TRUST in csrc/chd_core.h): switch times within 0.04 s of the input
          double t = 0, t0 = 0;
          for (size_t i = 0; i < dur_vars.size(); ++i) {
            const int j = dur_vars[i];
            if (durk[j] == 0) t = 0, t0 = 0;
            t += xt[j], t0 += x_init_dur[i];
            if (std::fabs(t - t0) > tau_trust) okp = false;
          }
        }
        if (nl_ke > 0.0 && okp && theta_t - (1.0 - alpha) * theta > nl_ke * std::max(alpha * theta, nl_fl * std::max(1.0, theta_ref))) okp = false, nl_rej++;
        for (auto& e : filt)
          if (okp && theta_t >= e.first && phit >= e.second) okp = false;
        if (okp) {
          const bool switching = dphi < 0 && alpha * std::pow(-dphi, o.s_phi) > std::pow(theta, o.s_theta);
          const bool armijo = phit <= phi0 + o.eta_phi * alpha * dphi;
          if (theta <= theta_min && switching) {
            if (armijo) accepted = true, ftype = true;
          } else if (theta_t <= (1 - o.gamma_theta) * theta || phit <= phi0 - o.gamma_phi * theta) {
            accepted = true;
            ftype = switching && armijo;
          }
        }
        if (accepted) break;
        alpha *= 0.5;
      }
      if (!accepted) {
        alpha *= 2.0;
        ls = o.max_backtrack;
        ls_fail++;
      }
      if (accepted && !ftype && (int)filt.size() < o.filt_max) filt.emplace_back((1 - o.gamma_theta) * theta, phi0 - o.gamma_phi * theta);
      if (polish) delta_w = delta_w_state;
      {
        const int ls_f = rt0 > 0.0 ? ls - nl_rej : ls;   // trials refused by the filter itself
        const double dec3 = (!dur_vars.empty() && getenv("CHD_DW_DEC3")) ? atof(getenv("CHD_DW_DEC3")) : o.dw_dec;
        const double inc3 = (!dur_vars.empty() && getenv("CHD_DW_INC3")) ? atof(getenv("CHD_DW_INC3")) : o.dw_inc;
        const int cap3 = (!dur_vars.empty() && getenv("CHD_LS_CAP3")) ? atoi(getenv("CHD_LS_CAP3")) : 3;
        // Adaptive floor of the Levenberg-Marquardt weight.  Sequences that take full steps at the floor converge linearly
        // at a rate set by the floor (the reduced Hessian along force directions is ~1e-10): after `af_n` such steps in a
        // row the floor drops by 10x (not below af_min).  The lower floor is a gamble (the Gauss-Newton model misses
        // constraint curvature: some sequences start to oscillate or crawl), so it is taken back for the rest of the
        // stage at the first backtrack, or when the scaled error has not halved 30 iterations after the first drop.
        if (af_n > 0 && !af_off) {
          const bool at_floor = ls == 0 && delta_w <= dw_floor * 1.0000001;
          if (dw_floor < o.dw_min) {
            if (ls > 0 || (it - af_it >= 30 && E0 > 0.5 * af_E)) dw_floor = o.dw_min, af_off = true;
            else if (at_floor && ++af_cnt >= af_n) dw_floor = std::max(dw_floor * 0.1, af_min), af_cnt = 0;
          } else if (at_floor) {
            if (++af_cnt >= af_n) dw_floor = std::max(dw_floor * 0.1, af_min), af_cnt = 0, af_E = E0, af_it = it;
          } else if (ls > 0) {
            af_cnt = 0;
          }
        }
        const double fl = af_n > 0 ? dw_floor : o.dw_min;
        if (ls_f == 0) delta_w = std::max(delta_w / dec3, fl);
        else delta_w = std::min(delta_w * std::pow(inc3, (double)std::min(ls_f, cap3)), o.dw_max);
        if (rt0 > 0.0) {
          if (nl_rej == 0) rho_tau = std::max(rho_tau / rt_dec, rt_min);
          else rho_tau = std::min(std::max(rho_tau, 1e-6) * std::pow(o.dw_inc, (double)std::min(nl_rej, 3)), 1e6);
        }
      }
      x = xt;
      for (int r = 0; r < m; ++r) {
        y[r] += alpha * dy[r];
        if (eq[r]) continue;
        s[r] += alpha * ds[r];
        if (hasL[r]) {
          const double gap = s[r] - dL[r];
          zL[r] = std::min(std::max(zL[r] + a_du * dzL[r], mu / (o.kappa_sigma * gap)), o.kappa_sigma * mu / gap);
        }
        if (hasU[r]) {
          const double gap = dU[r] - s[r];
          zU[r] = std::min(std::max(zU[r] + a_du * dzU[r], mu / (o.kappa_sigma * gap)), o.kappa_sigma * mu / gap);
        }
      }
      evaluate(x, f, c);
      chdo_grad(h, g.data());
      to_tau_grad(g);
      eval_jac();
    }
    chdo_set_x(h, x.data());
    if (ws) {
      ws->valid = true;
      ws->names = set_names, ws->off = set_off, ws->rows = set_rows;
      ws->y = y, ws->s = s, ws->zL = zL, ws->zU = zU, ws->sc = sc;
      ws->sf = sf, ws->mu = mu, ws->delta_w = delta_w;
    }
    if (stats) {
      stats[0] = f, stats[1] = E0, stats[2] = violu, stats[3] = dual_u, stats[4] = compl_u, stats[5] = mu, stats[6] = delta_w, stats[7] = ls_fail;
      stats[8] = it, stats[9] = Na, stats[10] = nb, stats[11] = w;
    }
    return status;
  }
};

}  // namespace

extern "C" {
// Solves one stage in place (warm start from the problem's current variables).  stats: 12 doubles
// (f, E0, unscaled violation, unscaled dual inf, unscaled complementarity, mu, delta_w, ls failures, iterations, Na, nb, w).
static std::map<void*, WarmState> g_warm;
int chdo_solve_stage(void* h, int stage, int max_iter, double* stats, int verbose) {
  Solver S;
  S.h = h;
  S.ws = &g_warm[h];
  // stage 3 (id 4) continues from the primal-dual point of stage 2.2; every other stage starts cold like IPOPT
  S.warm = stage == 4 && !(getenv("CHD_WARM") && atoi(getenv("CHD_WARM")) == 0);
  return S.run(stage, max_iter, stats, verbose);
}
void chdo_forget(void* h) { g_warm.erase(h); }
}
