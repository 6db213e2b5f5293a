// highs_b200/csrc/host_prep_hipdlp.cpp -- host prologue of the engine's SECOND algorithm mode (HiPDLP: reflected
// Halpern PDHG, `solver=hipdlp`; SURVEY.md 8(a) a20, 8(f) rank 2).  Product code (C++), no CUDA.
//
// HiPDLP prepares the LP differently from cuPDLP-C, so it gets its own formulate / scale (the layouts and the device
// side are shared):
//   PDLPSolver::preprocessLp   /root/reference/highs/pdlp/hipdlp/pdhg.cc:152-358
//       rows are classified with +-infinity (not +-1e20), free rows are a class of their own, the objective is NOT
//       multiplied by the sense, a column's entries are sorted by (new row, value), rows keep a lower AND an upper
//       bound (GEQ: [b, inf], EQ: [b, b], BOUND/FREE: [0, 0] with a slack column, LEQ negated into GEQ);
//   Scaling::scaleProblem      hipdlp/scaling.cc:23-263
//       Ruiz (inf-norm) x pdlp_ruiz_iterations, then Pock-Chambolle (alpha = 1), then optionally L2, each applied as
//       a_ij /= (r_i * c_j) -- ONE division by the product -- with only FINITE bounds scaled;
//   PDLPSolver::powerMethod    hipdlp/pdhg.cc:1529-1671 (the cuPDLP-C variant: 20 iterations on A A' from the ones vector).
// The arithmetic follows the reference expression by expression (tests/test_hipdlp_host.py compares with the oracle
// bit for bit); the loop structure is ours.
#include <algorithm>
#include <cmath>
#include <limits>
#include <utility>

#include "host_prep.hpp"

namespace b200 {

void formulate_hipdlp(const b200pdlp_lp& lp, StdForm& f) {
  const int n0 = lp.num_col, m = lp.num_row;
  const double inf = std::numeric_limits<double>::infinity();
  f = StdForm();
  f.hipdlp = true;
  f.n_orig = n0;
  f.m = m;
  f.sense = lp.sense;
  f.offset = lp.offset;
  f.row_class.resize(m);
  f.row_new_idx.resize(m);
  int n_slack = 0, n_eq = 0;
  for (int i = 0; i < m; i++) {   // pdhg.cc:175-198
    const bool lo = lp.row_lower[i] > -inf, up = lp.row_upper[i] < inf;
    int c;
    if (lo && up) c = (lp.row_lower[i] == lp.row_upper[i]) ? kEq : kBound;
    else if (lo) c = kGeq;
    else if (up) c = kLeq;
    else c = kFreeRow;
    f.row_class[i] = c;
    if (c == kBound || c == kFreeRow) n_slack++;
    if (c == kEq || c == kBound || c == kFreeRow) n_eq++;
  }
  f.neq = n_eq;
  f.n = n0 + n_slack;
  f.rhs.assign(m, 0.0);
  f.row_upper.assign(m, 0.0);
  {
    int head = 0, tail = n_eq;   // equality-like rows first, original order inside each group (:213-222)
    for (int i = 0; i < m; i++) {
      const int c = f.row_class[i];
      const int k = (c == kEq || c == kBound || c == kFreeRow) ? head++ : tail++;
      f.row_new_idx[i] = k;
      switch (c) {               // :247-270
        case kEq: f.rhs[k] = lp.row_lower[i]; f.row_upper[k] = lp.row_upper[i]; break;
        case kGeq: f.rhs[k] = lp.row_lower[i]; f.row_upper[k] = inf; break;
        case kLeq: f.rhs[k] = -lp.row_upper[i]; f.row_upper[k] = inf; break;
        default: f.rhs[k] = 0.0; f.row_upper[k] = 0.0; break;
      }
    }
  }
  f.cost.assign(f.n, 0.0);
  f.lower.resize(f.n);
  f.upper.resize(f.n);
  for (int j = 0; j < n0; j++) { f.cost[j] = lp.col_cost[j]; f.lower[j] = lp.col_lower[j]; f.upper[j] = lp.col_upper[j]; }
  const int nnz0 = lp.a_start[n0];
  f.nnz = nnz0 + n_slack;
  f.cbeg.resize(f.n + 1);
  f.cidx.resize(f.nnz);
  f.cval.resize(f.nnz);
  {
    // structural columns keep their entry count: column j starts at a_start[j]; entries sorted by (row, value) (:300-333)
    parallel_chunks(n0, [&](int, long long j0, long long j1) {   // columns are independent
      std::vector<std::pair<int, double>> e;
      for (int j = (int)j0; j < (int)j1; j++) {
        e.clear();
        for (int p = lp.a_start[j]; p < lp.a_start[j + 1]; p++) {
          const int old = lp.a_index[p];
          e.emplace_back(f.row_new_idx[old], f.row_class[old] == kLeq ? -lp.a_value[p] : lp.a_value[p]);
        }
        std::sort(e.begin(), e.end());
        int k = lp.a_start[j];
        f.cbeg[j] = k;
        for (const auto& t : e) { f.cidx[k] = t.first; f.cval[k] = t.second; k++; }
      }
    }, 1 << 12);
  }
  int k = nnz0, j = n0;
  for (int i = 0; i < m; i++) {   // one slack column per BOUND / FREE row: A x - z = 0, z in the row's bounds (:235-244,336-346)
    if (f.row_class[i] != kBound && f.row_class[i] != kFreeRow) continue;
    f.cbeg[j] = k;
    f.cidx[k] = f.row_new_idx[i];
    f.cval[k] = -1.0;
    k++;
    f.lower[j] = lp.row_lower[i];
    f.upper[j] = lp.row_upper[i];
    j++;
  }
  f.cbeg[f.n] = k;
  f.col_scale.assign(f.n, 1.0);
  f.row_scale.assign(f.m, 1.0);
  double s = 0.0;   // norms of the UNSCALED processed data (:353-354): sequential sums like linalg::dot
  for (int q = 0; q < f.n; q++) s += f.cost[q] * f.cost[q];
  f.norm_cost = std::sqrt(s);
  s = 0.0;
  for (int i = 0; i < f.m; i++) s += f.rhs[i] * f.rhs[i];
  f.norm_rhs = std::sqrt(s);
}

namespace {
// one pass's factors into the data (Scaling::applyScaling, scaling.cc:232-263) and into the running scales
void apply_hipdlp(StdForm& f, const std::vector<double>& cs, const std::vector<double>& rs) {
  const double inf = std::numeric_limits<double>::infinity();
  parallel_chunks(f.n, [&](int, long long b, long long e) {
    for (int i = (int)b; i < (int)e; i++) {
      f.cost[i] /= cs[i];
      if (f.lower[i] > -inf) f.lower[i] *= cs[i];
      if (f.upper[i] < inf) f.upper[i] *= cs[i];
      f.col_scale[i] *= cs[i];
      const double cc = cs[i];
      for (int p = f.cbeg[i]; p < f.cbeg[i + 1]; p++) f.cval[p] /= (rs[f.cidx[p]] * cc);
    }
  }, 1 << 12);
  parallel_chunks(f.m, [&](int, long long b, long long e) {
    for (int i = (int)b; i < (int)e; i++) {
      if (f.rhs[i] > -inf) f.rhs[i] /= rs[i];
      if (f.row_upper[i] < inf) f.row_upper[i] /= rs[i];
      f.row_scale[i] *= rs[i];
    }
  }, 1 << 14);
}
// per-row reductions in the order of the reference's column-major scatter (rs[row] op= term, columns ascending) = the row's
// entries in row-major order: the row index (build_row_index) gives that order, so rows can be done in parallel
template <class Term, class Op>
void row_reduce(const StdForm& f, std::vector<double>& rs, Term term, Op op) {
  parallel_chunks(f.m, [&](int, long long b, long long e) {
    for (int i = (int)b; i < (int)e; i++) {
      double a = 0.0;
      for (int q = f.rptr[i]; q < f.rptr[i + 1]; q++) a = op(a, term(f.cval[f.rpos[q]]));
      rs[i] = a;
    }
  }, 1 << 12);
}
}  // namespace

void scale_hipdlp(StdForm& f, int scaling_mode, int ruiz_iterations) {
  const int n = f.n, m = f.m;
  std::vector<double> cs(n), rs(m);
  f.scaled = false;
  if ((scaling_mode & 7) && f.rptr.empty() && f.nnz > 0) build_row_index(f);   // row-major order of the entries (positions into cval)
  const auto fmax = [](double a, double v) { return std::max(a, v); };
  const auto fadd = [](double a, double v) { return a + v; };
  if (scaling_mode & 1) {   // Ruiz, infinity norm (scaling.cc:56-125)
    for (int it = 0; it < ruiz_iterations; it++) {
      parallel_chunks(n, [&](int, long long b, long long e) {
        for (int c = (int)b; c < (int)e; c++) {
          double mx = 0.0;
          for (int p = f.cbeg[c]; p < f.cbeg[c + 1]; p++) mx = std::max(mx, std::fabs(f.cval[p]));
          double v = (f.cbeg[c] < f.cbeg[c + 1]) ? std::sqrt(mx) : 0.0;
          if (v == 0.0) v = 1.0;
          cs[c] = v;
        }
      }, 1 << 12);
      row_reduce(f, rs, [](double v) { return std::fabs(v); }, fmax);
      parallel_chunks(m, [&](int, long long b, long long e) {
        for (int i = (int)b; i < (int)e; i++) rs[i] = (rs[i] == 0.0) ? 1.0 : std::sqrt(rs[i]);
      }, 1 << 14);
      apply_hipdlp(f, cs, rs);
    }
    f.scaled = true;
  }
  if (scaling_mode & 4) {   // Pock-Chambolle, alpha = 1 (:127-178); pow() kept as in the reference
    const double alpha = 1.0;
    parallel_chunks(n, [&](int, long long b, long long e) {
      for (int c = (int)b; c < (int)e; c++) {
        double sum = 0.0;
        for (int p = f.cbeg[c]; p < f.cbeg[c + 1]; p++) sum += std::pow(std::fabs(f.cval[p]), alpha);
        cs[c] = sum > 0.0 ? std::sqrt(std::pow(sum, 1.0 / alpha)) : 1.0;
      }
    }, 1 << 12);
    row_reduce(f, rs, [&](double v) { return std::pow(std::fabs(v), 2.0 - alpha); }, fadd);
    parallel_chunks(m, [&](int, long long b, long long e) {
      for (int i = (int)b; i < (int)e; i++) rs[i] = rs[i] > 0.0 ? std::sqrt(std::pow(rs[i], 1.0 / (2.0 - alpha))) : 1.0;
    }, 1 << 14);
    apply_hipdlp(f, cs, rs);
    f.scaled = true;
  }
  if (scaling_mode & 2) {   // L2 (:180-230)
    parallel_chunks(n, [&](int, long long b, long long e) {
      for (int c = (int)b; c < (int)e; c++) {
        double sq = 0.0;
        for (int p = f.cbeg[c]; p < f.cbeg[c + 1]; p++) sq += f.cval[p] * f.cval[p];
        cs[c] = sq > 0.0 ? std::sqrt(std::sqrt(sq)) : 1.0;
      }
    }, 1 << 12);
    row_reduce(f, rs, [](double v) { return v * v; }, fadd);
    parallel_chunks(m, [&](int, long long b, long long e) {
      for (int i = (int)b; i < (int)e; i++) rs[i] = rs[i] > 0.0 ? std::sqrt(std::sqrt(rs[i])) : 1.0;
    }, 1 << 14);
    apply_hipdlp(f, cs, rs);
    f.scaled = true;
  }
  double amax = 0.0;   // (max is order-free)
  for (int p = 0; p < f.nnz; p++) amax = std::max(amax, std::fabs(f.cval[p]));
  f.amax = amax;
}

// lambda_max(A A') estimate: 20 power iterations from the ones vector (pdhg.cc:1529-1671, "cuPDLP-C" branch), with
// HighsSparseMatrix::product / productTranspose's accumulation order (util/HighsSparseMatrix.cpp:1180-1218)
double power_method_hipdlp(const StdForm& f) {
  if (f.n == 0 || f.m == 0) return 1.0;
  std::vector<double> x(f.m, 1.0), y(f.n), z(f.m);
  double lambda = 0.0;
  auto at_times = [&](const std::vector<double>& v, std::vector<double>& out) {
    for (int c = 0; c < f.n; c++) {
      double s = 0.0;
      for (int p = f.cbeg[c]; p < f.cbeg[c + 1]; p++) s += v[f.cidx[p]] * f.cval[p];
      out[c] = s;
    }
  };
  for (int it = 0; it < 20; it++) {
    at_times(x, y);
    std::fill(z.begin(), z.end(), 0.0);
    for (int c = 0; c < f.n; c++)
      for (int p = f.cbeg[c]; p < f.cbeg[c + 1]; p++) z[f.cidx[p]] += y[c] * f.cval[p];
    double zz = 0.0;
    for (int i = 0; i < f.m; i++) zz += z[i] * z[i];
    const double zn = std::sqrt(zz);
    for (int i = 0; i < f.m; i++) z[i] /= zn;
    at_times(z, y);
    lambda = 0.0;
    for (int c = 0; c < f.n; c++) lambda += y[c] * y[c];
    x = z;
  }
  return lambda;
}

void HipController::init(double norm_cost_, double norm_rhs_, double op_norm_sq, double tol_, int strategy_) {
  *this = HipController();
  tol = tol_; norm_cost = norm_cost_; norm_rhs = norm_rhs_; strategy = strategy_;
  omega = (norm_cost + 1.0) / (norm_rhs + 1.0);
  primal_weight = omega;
  best_primal_weight = primal_weight;
  best_gap = std::numeric_limits<double>::infinity();
  eta = 0.998 / std::sqrt(op_norm_sq);
  primal_step = eta / omega;
  dual_step = eta * omega;
  last_trial = std::numeric_limits<double>::infinity();
}

double HipController::fixed_point_error(const double* s) const {
  const double movement = s[0] * omega + s[1] / omega;
  const double interaction = 2.0 * eta * s[2];
  return std::sqrt(std::max(0.0, movement + interaction));
}

bool HipController::converged(const double* s) {
  pfeas = std::sqrt(s[3]);
  dfeas = std::sqrt(s[4]);
  pobj = s[5];
  dobj = s[6];
  const double gap = pobj - dobj;
  relgap = std::fabs(gap) / (1.0 + std::fabs(pobj) + std::fabs(dobj));
  return block_converged();
}

bool HipController::after_block(const double* s) {
  fpe = fixed_point_error(s);
  halpern_iteration += 40;
  iters += 40;
  if (converged(s)) return false;
  bool restart = false;                     // checkRestartCriteria, :901-927
  if (iters == 40) restart = true;
  else if (iters > 40) {
    if (fpe <= 0.2 * fpe0) restart = true;
    else if (fpe <= 0.8 * fpe0 && fpe > last_trial) restart = true;
    else if (halpern_iteration >= 0.36 * iters) restart = true;
  }
  last_trial = fpe;
  if (!restart) return false;
  restarts++;
  if (strategy != 0) {                      // updatePrimalWeightAtRestart (PID controller), :1979-2050
    const double pd = std::sqrt(s[7]), dd = std::sqrt(s[8]);
    const double rel_p = pfeas / (1.0 + norm_rhs), rel_d = dfeas / (1.0 + norm_cost);
    const double ratio = (rel_p > 0.0) ? (rel_d / rel_p) : 1e300;
    if (pd > 1e-16 && dd > 1e-16 && pd < 1e12 && dd < 1e12 && ratio > 1e-8 && ratio < 1e8) {
      const double error = std::log(dd) - std::log(pd) - std::log(primal_weight);
      err_sum = 0.3 * err_sum + error;
      const double delta = error - last_err;
      primal_weight *= std::exp(0.99 * error + 0.01 * err_sum + 0.0 * delta);
      last_err = error;
    } else {
      primal_weight = best_primal_weight;
      err_sum = 0.0;
      last_err = 0.0;
    }
    const double gap = (rel_p > 0.0 && rel_d > 0.0) ? std::fabs(std::log10(rel_d / rel_p)) : best_gap;
    if (gap < best_gap) { best_gap = gap; best_primal_weight = primal_weight; }
    const double e2 = std::sqrt(primal_step * dual_step);
    primal_step = e2 / primal_weight;
    dual_step = e2 * primal_weight;
    omega = primal_weight;
  }
  halpern_iteration = 0;
  last_trial = std::numeric_limits<double>::infinity();
  pending_restart_fpe = true;
  return true;
}

}  // namespace b200
