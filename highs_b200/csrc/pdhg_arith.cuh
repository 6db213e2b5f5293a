// highs_b200/csrc/pdhg_arith.cuh -- per-element arithmetic of the PDHG pass and of the ordered-mode check, and of the HiPDLP
// step and check, shared by the one-problem kernels (pdhg_kernels.cu) and the batch kernels (batch_kernels.cu), so that both
// produce the same bits.
// Every function keeps the reference CPU path's operation order (see kernels.cuh; compiled with -fmad=false).
#pragma once
#include "kernels.cuh"
#include "pdhg_kernels.hpp"

namespace b200 {

// K1, PDHG_primalGradientStep (cupdlp_step.c:28-38): out = proj_[l,u](x - tau c + tau aty); returns |x - out|^2's term
__device__ __forceinline__ double primal_update(double xc, double ci, double ai, double u, double l, double tau, double ntau,
                                                double& out) {
  double v = xc + ntau * ci;
  v = v + tau * ai;
  v = v < u ? v : u;
  v = v > l ? v : l;
  out = v;
  const double d = xc - v;
  return d * d;
}

// K2, PDHG_dualGradientStep (cupdlp_step.c:55-67): y' = y + sigma b - 2 sigma ax' + sigma ax, max(., 0) on inequality rows
__device__ __forceinline__ double dual_update(double yc, double bi, double ax_new, double ax, double sigma, bool ineq) {
  double v = yc + sigma * bi;
  v = v + (-2.0 * sigma) * ax_new;
  v = v + sigma * ax;
  if (ineq) v = v > 0.0 ? v : 0.0;
  return v;
}

// K4: PDHG_Update_Iterate_Adaptive_Step_Size (cupdlp_step.c:236-307) + the bookkeeping of PDHG_Update_Average (:422-442),
// given st->dx2, st->dy2 and the interaction of the pass
__device__ __forceinline__ void step_rule(PdhgState* st, double inter) {
  const double rb = sqrt(st->beta);
  const double mov = st->dx2 * 0.5 * rb + st->dy2 / (2.0 * rb);   // cupdlp_linalg.c:800
  st->inter = inter;
  st->mov = mov;
  st->passes++;
  if (st->adaptive) {
    const int k = ++st->step_iter;
    const double eta = st->eta;
    const double lim = (inter != 0.0) ? mov / fabs(inter) : INFINITY;
    st->lim = lim;
    const bool accept = eta <= lim;
    int t = k - st->pow_base - 1;
    double pr, pg;
    if (t >= 0 && t < kPowTab) { pr = st->pow_red[t]; pg = st->pow_grow[t]; }
    else { pr = pow(k + 1.0, -0.3); pg = pow(k + 1.0, -0.6); }   // never hit: host refills the tables
    const double first = (1.0 - pr) * lim;
    const double second = (1.0 + pg) * eta;
    const double eta_new = fmin(first, second);
    if (accept) {
      st->tau = eta_new / rb;
      st->sigma = eta_new * rb;
      const double w = sqrt(st->tau * st->sigma);
      st->sum_step += w;
      st->w_pending = w;
      st->pending = 1;
      st->cur ^= 1;
      st->iter++;
      st->eta = w;   // next iteration starts from sqrt(dPrimalStep*dDualStep), cupdlp_step.c:230-231
    } else {
      st->eta = eta_new;
      st->pending = 0;
      st->rejects++;
    }
    st->tau_try = st->eta / rb;
    st->sigma_try = st->eta * rb;
  } else {
    // fixed step (PDHG_Update_Iterate_Constant_Step_Size): always accepted, steps unchanged
    const double w = sqrt(st->tau * st->sigma);
    st->sum_step += w;
    st->w_pending = w;
    st->pending = 1;
    st->cur ^= 1;
    st->iter++;
  }
}

// ordered-mode check, column side, sweep A (cupdlp_solver.c:23-24, :69-204, :255-262, :367):
// emit(k, term) for k = c.x, sp.lo_f, sn.up_f, |dual residual|^2, |sp|^2, |sn|^2, |x|^2 of one column.  (The check terms go
// out through a callback rather than an array: each term reaches its accumulator as soon as it is formed, which keeps the
// one-problem check kernels' code as it was.)
template <class Emit>
__device__ __forceinline__ void col_check_a_terms(double x, double aty, double ci, bool hl, bool hu, double lf, double uf,
                                                  double sc, Emit emit) {
  double rc = aty * -1.0;
  rc = rc + 1.0 * ci;
  double sp = rc > 0.0 ? rc : 0.0;
  sp = sp * (hl ? 1.0 : 0.0);
  double sn = rc < 0.0 ? rc : 0.0;
  sn = sn * -1.0;
  sn = sn * (hu ? 1.0 : 0.0);
  double rr = rc + -1.0 * sp;
  rr = rr + 1.0 * sn;
  rr = rr * sc;
  emit(0, x * ci);
  emit(1, sp * lf);
  emit(2, sn * uf);
  emit(3, rr * rr);
  emit(4, sp * sp);
  emit(5, sn * sn);
  emit(6, x * x);
}

// row side, sweep A (cupdlp_solver.c:36-63, :79): emit(k, term) for k = y.b, |primal residual|^2, |y|^2 of one row
template <class Emit>
__device__ __forceinline__ void row_check_a_terms(double y, double ax, double bi, double sc, bool ineq, Emit emit) {
  double r = ax + -1.0 * bi;
  if (ineq) r = r < 0.0 ? r : 0.0;
  r = r * sc;
  emit(0, y * bi);
  emit(1, r * r);
  emit(2, y * y);
}

// column side, sweep B (needs the ray scales of sweep A; cupdlp_solver.c:289-303, :395-423): emit(k, term) for k = |dual-ray
// constraint residual|^2, |lower-bound violation of the primal ray|^2, |upper ...|^2 of one column
template <class Emit>
__device__ __forceinline__ void col_check_b_terms(double x, double aty, double ci, double hl, double hu, double sc, double ids,
                                                  double ips, Emit emit) {
  double rc = aty * -1.0;
  rc = rc + 1.0 * ci;
  double sp = rc > 0.0 ? rc : 0.0;
  sp = sp * hl;
  double sn = rc < 0.0 ? rc : 0.0;
  sn = sn * -1.0;
  sn = sn * hu;
  double k = aty * ids;
  k = k + 1.0 * (sp * ids);
  k = k + -1.0 * (sn * ids);
  k = k * sc;
  const double ray = x * ips;
  double bl = ray < 0.0 ? ray : 0.0;
  bl = bl * hl;
  bl = bl / sc;
  double bu = ray > 0.0 ? ray : 0.0;
  bu = bu * hu;
  bu = bu / sc;
  emit(0, k * k);
  emit(1, bl * bl);
  emit(2, bu * bu);
}

// row side, sweep B (cupdlp_solver.c:381-392): |[A ray]_eq, min([A ray]_ineq, 0)|^2 term of one row
__device__ __forceinline__ double row_check_b_term(double ax, double ips, double sc, bool ineq) {
  double k = ax * ips;
  if (ineq) k = k < 0.0 ? k : 0.0;
  k = k * sc;
  return k * k;
}

// ---- HiPDLP mode (reflected Halpern PDHG, hipdlp/pdhg.cc): the one-problem kernels of pdhg_kernels.cu and the HiPDLP batch
// kernel (batch_kernels.cu)

__device__ __forceinline__ double std_max(double a, double b) { return a < b ? b : a; }   // std::max / std::min semantics
__device__ __forceinline__ double std_min(double a, double b) { return b < a ? b : a; }

// x-side of performHalpernPdhgStep (:974-986, :1006-1009) for column i; returns the reflected x
__device__ __forceinline__ double hip_primal_col(int i, double ps, double w, int is_major, double* __restrict__ x,
                                                 const double* __restrict__ xa, const double* __restrict__ c,
                                                 const double* __restrict__ aty, const double* __restrict__ lo,
                                                 const double* __restrict__ up, double* __restrict__ rx,
                                                 double* __restrict__ xn, double* __restrict__ hslack) {
  const double rho = 1.0;
  const double xc = x[i];
  const double temp = xc - ps * (c[i] - aty[i]);
  const double proj = std_max(lo[i], std_min(temp, up[i]));
  if (is_major) { xn[i] = proj; hslack[i] = (proj - temp) / ps; }
  const double r = 2.0 * proj - xc;
  rx[i] = r;
  const double blended = rho * r + (1.0 - rho) * xc;
  x[i] = w * blended + (1.0 - w) * xa[i];
  return r;
}

// y-side (:992-1003, :1010-1013) of row r, given s = (A * reflected x)[r] and the row's y, anchor ya and bounds: returns the
// blended y; a major step also stores the projected dual (y_next) in yn[r] and the reflected y in ry[r]
__device__ __forceinline__ double hip_dual_blend(int r, double y, double ya, double lo, double up, double s, double ds, double w,
                                                 int is_major, double* yn, double* ry) {
  const double rho = 1.0;
  const double temp = y / ds - s;
  const double proj = std_max(-up, std_min(temp, -lo));
  const double pd = (temp - proj) * ds;
  const double refl = 2.0 * pd - y;
  if (is_major) { yn[r] = pd; ry[r] = refl; }
  const double blended = rho * refl + (1.0 - rho) * y;
  return w * blended + (1.0 - w) * ya;
}

// dual slack of column i (computeDualSlacks, :1322-1378): the cached major-step slack when there is one, otherwise the
// residual projected by the signs of the bounds; sp / sn are its positive and negative parts
__device__ __forceinline__ void hip_dual_slacks(int i, int use_cached, const double* __restrict__ hslack,
                                                const double* __restrict__ c, const double* __restrict__ aty,
                                                const double* __restrict__ lo, const double* __restrict__ up, double& sp,
                                                double& sn) {
  double slack = 0.0;
  if (use_cached) slack = hslack[i];
  else {
    const double dres = c[i] - aty[i];
    const bool hl = lo[i] > -INFINITY, hu = up[i] < INFINITY;
    if (hl && hu) slack = dres;
    else if (hl) slack = std_max(0.0, dres);
    else if (hu) slack = std_min(0.0, dres);
  }
  sp = std_max(0.0, slack);
  sn = std_max(0.0, -slack);
}

// The terms of the nine sums of a HiPDLP check (hip_check_ordered_kernel; each sum adds its terms in index order):
//   0 |x_next - refl_x|^2  1 |y_next - refl_y|^2  2 (x_next - refl_x).(A' dy)        (fixed-point error, :709-740)
//   3 |primal residual|^2 (:1297-1320)  4 |dual residual|^2 (:1380-1408)  5 offset + c.x (:1496-1500)
//   6 offset + b.y + l.sp - u.sn (:1447-1472): rows, then lower bounds, then upper bounds, one running sum
//   7 |x_next - x_anchor|^2  8 |y_next - y_anchor|^2                                    (PID weight, :1984-1999)
__device__ __forceinline__ double hip_fpe_x_term(const HipCheckArgs& a, int i) { const double d = a.x[i] - a.rx[i]; return d * d; }
__device__ __forceinline__ double hip_fpe_y_term(const HipCheckArgs& a, int i) { const double d = a.y[i] - a.ry[i]; return d * d; }
__device__ __forceinline__ double hip_fpe_inter_term(const HipCheckArgs& a, int i) { return (a.x[i] - a.rx[i]) * a.atdy[i]; }
__device__ __forceinline__ double hip_primal_res_term(const HipCheckArgs& a, int i) {
  double r = a.ax[i] - a.rlo[i];
  if (i >= a.neq) r = std_min(0.0, r);
  if (a.scaled) r = r * a.rowscale[i];
  return r * r;
}
__device__ __forceinline__ double hip_dual_res_term(const HipCheckArgs& a, int i) {
  double r = (a.c[i] - a.aty[i]) - a.sp[i] + a.sn[i];
  if (a.scaled) r = r * a.colscale[i];
  return r * r;
}
__device__ __forceinline__ double hip_pobj_term(const HipCheckArgs& a, int i) { return a.c[i] * a.x[i]; }
__device__ __forceinline__ double hip_dobj_row_term(const HipCheckArgs& a, int i) { return a.rlo[i] * a.y[i]; }
// skipped (infinite-bound) columns add nothing in the reference: + 0.0 leaves the running sum unchanged
__device__ __forceinline__ double hip_dobj_lo_term(const HipCheckArgs& a, int i) { return a.lo[i] > -INFINITY ? a.lo[i] * a.sp[i] : 0.0; }
__device__ __forceinline__ double hip_dobj_up_term(const HipCheckArgs& a, int i) { return a.up[i] < INFINITY ? -(a.up[i] * a.sn[i]) : 0.0; }
__device__ __forceinline__ double hip_anchor_x_term(const HipCheckArgs& a, int i) { const double d = a.x[i] - a.xa[i]; return d * d; }
__device__ __forceinline__ double hip_anchor_y_term(const HipCheckArgs& a, int i) { const double d = a.y[i] - a.ya[i]; return d * d; }

}  // namespace b200
