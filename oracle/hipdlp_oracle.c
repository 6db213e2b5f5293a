/* oracle/hipdlp_oracle.c -- TEST INFRASTRUCTURE ONLY (see pdlp_oracle.h for the rules).
 *
 * Plain-C restatement of the reference's SECOND first-order LP engine, HiPDLP (`solver=hipdlp`:
 * reflected Halpern PDHG, fixed or PID-controlled primal weight, fixed-point-error restarts), as it
 * runs on the CPU:  solveLpHiPdlp (pdlp/HiPdlpWrapper.cpp:26-141) -> PDLPSolver::{preprocessLp,
 * scaleProblem, solve, unscaleSolution, postprocess} (pdlp/hipdlp/pdhg.cc, scaling.cc, linalg.cc).
 * SURVEY.md 8(a) row a20 / 8(f) rank 2.  Written from the algorithm with the reference's evaluation
 * ORDER kept expression by expression (including its libm calls), so that results can be pinned bit for
 * bit against oracle/_ref; every function cites the lines it follows (paths relative to
 * /root/reference/highs/pdlp/hipdlp/).  Quirks of the reference are kept, e.g. an iteration-limited
 * run returns x = y = 0 (pdhg.cc:784-899 copies the iterate out only on convergence).
 * Compile with -O2 -ffp-contract=off.
 */
#include "hipdlp_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#define NEW(T, k) ((T*)calloc((size_t)((k) > 0 ? (k) : 1), sizeof(T)))
#define CHECK_INTERVAL 40            /* PDHG_CHECK_INTERVAL, pdhg.cc:32 */

enum { T_EQ, T_LEQ, T_GEQ, T_BOUND, T_FREE };

typedef struct {
  /* processed LP (pdhg.cc:152-358), scaled in place by scaling.cc */
  int n, m, n0, nnz;
  double *cost, *lower, *upper, *rlo, *rup;
  int *cbeg, *cidx;
  double* cval;
  int *ctype, *new_idx, *is_eq;
  double c_norm, rhs_norm;           /* unscaled_c_norm_, unscaled_rhs_norm_ */
  double *col_scale, *row_scale;
  int is_scaled;
  /* solver state */
  double omega, eta, primal_step, dual_step, primal_weight, best_primal_weight, best_gap;
  double err_sum, last_err;
  double *x, *y, *xn, *yn, *rx, *ry, *xa, *ya, *ax_cache, *aty_cache, *ax_next;
  double *sp, *sn, *hslack;
  int hslack_valid, halpern_iteration;
  double pfeas, dfeas, pobj, dobj, gap, relgap;   /* results_ of the last check */
  double sums[9];                                 /* raw sums behind the last FPE / check / PID distances (trace) */
} hip;

/* ------------------------------------------------------------------ linalg.cc */
static void l_ax(const hip* s, const double* x, double* r) {           /* linalg.cc:36-47 */
  for (int i = 0; i < s->m; i++) r[i] = 0.0;
  for (int c = 0; c < s->n; c++)
    for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) r[s->cidx[p]] += s->cval[p] * x[c];
}
static void l_aty(const hip* s, const double* y, double* r) {          /* linalg.cc:49-61 */
  for (int c = 0; c < s->n; c++) r[c] = 0.0;
  for (int c = 0; c < s->n; c++)
    for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) r[c] += s->cval[p] * y[s->cidx[p]];
}
/* TEST SWITCH (not the reference's behaviour), like orc_set_sum_block in pdlp_oracle.c: hip_set_sum_block(k > 0) makes l_dot
 * (and so l_norm2, the power method's norms and the residual norms of the checks) add in blocks of k elements and then add
 * the block sums -- a different, equally valid rounding order, like the GPU engine's tree reductions.  Used to measure how
 * far a mere change of summation order moves a HiPDLP trajectory (tests/test_gpu_hipdlp_kernels.py).  0: sequential. */
static int g_sum_block = 0;
void hip_set_sum_block(int k) { g_sum_block = k; }
static double l_dot(int k, const double* a, const double* b) {         /* linalg.cc:63-73 */
  double r = 0.0;
  if (g_sum_block > 0) {
    for (int i0 = 0; i0 < k; i0 += g_sum_block) {
      double t = 0.0;
      const int i1 = i0 + g_sum_block < k ? i0 + g_sum_block : k;
      for (int i = i0; i < i1; i++) t += a[i] * b[i];
      r += t;
    }
    return r;
  }
  for (int i = 0; i < k; i++) r += a[i] * b[i];
  return r;
}
static double l_norm2(int k, const double* a) { return sqrt(l_dot(k, a, a)); }
static double dmax(double a, double b) { return a < b ? b : a; }       /* std::max(a,b): (a < b) ? b : a */
static double dmin(double a, double b) { return b < a ? b : a; }       /* std::min(a,b): (b < a) ? b : a */

/* ------------------------------------------------------------- preprocessLp */
typedef struct { int row; double val; } ent;
static int ent_cmp(const void* pa, const void* pb) {                   /* std::sort of pair<int,double>, pdhg.cc:324 */
  const ent *a = (const ent*)pa, *b = (const ent*)pb;
  if (a->row != b->row) return a->row < b->row ? -1 : 1;
  if (a->val < b->val) return -1;
  if (b->val < a->val) return 1;
  return 0;
}

static void preprocess(const orc_lp* lp, hip* s) {                     /* pdhg.cc:152-358 */
  const int m = lp->m, n0 = lp->n;
  int n_new = 0, neq = 0;
  s->ctype = NEW(int, m); s->new_idx = NEW(int, m); s->is_eq = NEW(int, m);
  for (int i = 0; i < m; i++) {
    const int has_lo = lp->row_lower[i] > -INFINITY, has_up = lp->row_upper[i] < INFINITY;
    if (has_lo && has_up) {
      if (lp->row_lower[i] == lp->row_upper[i]) { s->ctype[i] = T_EQ; neq++; }
      else { s->ctype[i] = T_BOUND; n_new++; neq++; }
    } else if (has_lo) s->ctype[i] = T_GEQ;
    else if (has_up) s->ctype[i] = T_LEQ;
    else { s->ctype[i] = T_FREE; n_new++; neq++; }
  }
  const int n = n0 + n_new;
  s->n = n; s->m = m; s->n0 = n0;
  s->cost = NEW(double, n); s->lower = NEW(double, n); s->upper = NEW(double, n);
  s->rlo = NEW(double, m); s->rup = NEW(double, m);
  int e = 0, q = neq;
  for (int i = 0; i < m; i++) {
    const int t = s->ctype[i];
    s->new_idx[i] = (t == T_EQ || t == T_BOUND || t == T_FREE) ? e++ : q++;
  }
  for (int i = 0; i < m; i++) {
    const int t = s->ctype[i];
    s->is_eq[s->new_idx[i]] = (t == T_EQ || t == T_BOUND || t == T_FREE);
  }
  for (int j = 0; j < n0; j++) { s->cost[j] = lp->cost[j]; s->lower[j] = lp->col_lower[j]; s->upper[j] = lp->col_upper[j]; }
  for (int i = 0, j = n0; i < m; i++)
    if (s->ctype[i] == T_BOUND || s->ctype[i] == T_FREE) {
      s->cost[j] = 0.0; s->lower[j] = lp->row_lower[i]; s->upper[j] = lp->row_upper[i]; j++;
    }
  for (int i = 0; i < m; i++) {
    const int k = s->new_idx[i];
    switch (s->ctype[i]) {
      case T_EQ: s->rlo[k] = lp->row_lower[i]; s->rup[k] = lp->row_upper[i]; break;
      case T_GEQ: s->rlo[k] = lp->row_lower[i]; s->rup[k] = INFINITY; break;
      case T_LEQ: s->rlo[k] = -lp->row_upper[i]; s->rup[k] = INFINITY; break;
      default: s->rlo[k] = 0.0; s->rup[k] = 0.0; break;
    }
  }
  const int nnz0 = lp->start[n0];
  s->nnz = nnz0 + n_new;
  s->cbeg = NEW(int, n + 1); s->cidx = NEW(int, s->nnz); s->cval = NEW(double, s->nnz);
  ent* tmp = NEW(ent, m + 1);
  int k = 0;
  for (int c = 0; c < n0; c++) {
    int cnt = 0;
    for (int p = lp->start[c]; p < lp->start[c + 1]; p++) {
      const int old = lp->index[p];
      double v = lp->value[p];
      if (s->ctype[old] == T_LEQ) v = -v;
      if (cnt > m) { tmp = (ent*)realloc(tmp, sizeof(ent) * (size_t)(2 * cnt + 2)); }
      tmp[cnt].row = s->new_idx[old]; tmp[cnt].val = v; cnt++;
    }
    qsort(tmp, (size_t)cnt, sizeof(ent), ent_cmp);
    s->cbeg[c] = k;
    for (int t = 0; t < cnt; t++) { s->cidx[k] = tmp[t].row; s->cval[k] = tmp[t].val; k++; }
  }
  free(tmp);
  for (int i = 0, j = n0; i < m; i++)
    if (s->ctype[i] == T_BOUND || s->ctype[i] == T_FREE) { s->cbeg[j] = k; s->cidx[k] = s->new_idx[i]; s->cval[k] = -1.0; k++; j++; }
  s->cbeg[n] = k;
  s->c_norm = l_norm2(n, s->cost);          /* linalg::vectorNorm(vec) = norm2, linalg.cc:104-109 */
  s->rhs_norm = l_norm2(m, s->rlo);
}

/* ---------------------------------------------------------------- scaling.cc */
static void apply_scaling(hip* s, const double* cs, const double* rs) {  /* scaling.cc:232-263 */
  for (int i = 0; i < s->n; i++) s->cost[i] /= cs[i];
  for (int i = 0; i < s->n; i++) {
    if (s->lower[i] > -INFINITY) s->lower[i] *= cs[i];
    if (s->upper[i] < INFINITY) s->upper[i] *= cs[i];
  }
  for (int i = 0; i < s->m; i++) {
    if (s->rlo[i] > -INFINITY) s->rlo[i] /= rs[i];
    if (s->rup[i] < INFINITY) s->rup[i] /= rs[i];
  }
  for (int c = 0; c < s->n; c++)
    for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) s->cval[p] /= (rs[s->cidx[p]] * cs[c]);
  for (int i = 0; i < s->n; i++) s->col_scale[i] *= cs[i];
  for (int i = 0; i < s->m; i++) s->row_scale[i] *= rs[i];
}

static void scale_problem(hip* s, const hip_params* prm) {             /* scaling.cc:23-54 */
  const int n = s->n, m = s->m;
  s->col_scale = NEW(double, n); s->row_scale = NEW(double, m);
  for (int i = 0; i < n; i++) s->col_scale[i] = 1.0;
  for (int i = 0; i < m; i++) s->row_scale[i] = 1.0;
  s->is_scaled = 0;
  double* cs = NEW(double, n);
  double* rs = NEW(double, m);
  if (prm->use_ruiz) {                                                  /* :56-125, infinity norm */
    for (int it = 0; it < prm->ruiz_iterations; it++) {
      for (int c = 0; c < n; c++) {
        cs[c] = 0.0;
        if (s->cbeg[c] < s->cbeg[c + 1]) {
          double mx = 0.0;
          for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) mx = dmax(mx, fabs(s->cval[p]));
          cs[c] = sqrt(mx);
        }
        if (cs[c] == 0.0) cs[c] = 1.0;
      }
      for (int i = 0; i < m; i++) rs[i] = 0.0;
      for (int c = 0; c < n; c++)
        for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) rs[s->cidx[p]] = dmax(rs[s->cidx[p]], fabs(s->cval[p]));
      for (int i = 0; i < m; i++) rs[i] = (rs[i] == 0.0) ? 1.0 : sqrt(rs[i]);
      apply_scaling(s, cs, rs);
    }
    s->is_scaled = 1;
  }
  if (prm->use_pc) {                                                    /* :127-178, alpha = 1 */
    const double alpha = 1.0;
    for (int c = 0; c < n; c++) {
      cs[c] = 0.0;
      for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) cs[c] += pow(fabs(s->cval[p]), alpha);
      cs[c] = cs[c] > 0.0 ? sqrt(pow(cs[c], 1.0 / alpha)) : 1.0;
    }
    for (int i = 0; i < m; i++) rs[i] = 0.0;
    for (int c = 0; c < n; c++)
      for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) rs[s->cidx[p]] += pow(fabs(s->cval[p]), 2.0 - alpha);
    for (int i = 0; i < m; i++) rs[i] = rs[i] > 0.0 ? sqrt(pow(rs[i], 1.0 / (2.0 - alpha))) : 1.0;
    apply_scaling(s, cs, rs);
    s->is_scaled = 1;
  }
  if (prm->use_l2) {                                                    /* :180-230 */
    for (int c = 0; c < n; c++) {
      double sq = 0.0;
      for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) sq += s->cval[p] * s->cval[p];
      cs[c] = sq > 0.0 ? sqrt(sqrt(sq)) : 1.0;
    }
    for (int i = 0; i < m; i++) rs[i] = 0.0;
    for (int c = 0; c < n; c++)
      for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) rs[s->cidx[p]] += s->cval[p] * s->cval[p];
    for (int i = 0; i < m; i++) rs[i] = rs[i] > 0.0 ? sqrt(sqrt(rs[i])) : 1.0;
    apply_scaling(s, cs, rs);
    s->is_scaled = 1;
  }
  free(cs); free(rs);
}

/* ------------------------------------------------------- step sizes, power method */
static double power_method(const hip* s) {                             /* pdhg.cc:1529-1671, the cuPDLP-C variant on A A' */
  if (s->n == 0 || s->m == 0) return 1.0;
  double* xv = NEW(double, s->m);
  double* yv = NEW(double, s->n);
  double* zv = NEW(double, s->m);
  for (int i = 0; i < s->m; i++) xv[i] = 1.0;
  double lambda = 0.0;
  for (int it = 0; it < 20; it++) {
    for (int c = 0; c < s->n; c++) {                                    /* productTranspose, HighsSparseMatrix.cpp:1200-1218 */
      yv[c] = 0.0;
      for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) yv[c] += xv[s->cidx[p]] * s->cval[p];
    }
    for (int i = 0; i < s->m; i++) zv[i] = 0.0;                         /* product, :1180-1198 */
    for (int c = 0; c < s->n; c++)
      for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) zv[s->cidx[p]] += yv[c] * s->cval[p];
    const double zn = sqrt(l_dot(s->m, zv, zv));
    for (int i = 0; i < s->m; i++) zv[i] /= zn;
    for (int c = 0; c < s->n; c++) {
      yv[c] = 0.0;
      for (int p = s->cbeg[c]; p < s->cbeg[c + 1]; p++) yv[c] += zv[s->cidx[p]] * s->cval[p];
    }
    lambda = l_dot(s->n, yv, yv);
    memcpy(xv, zv, sizeof(double) * (size_t)s->m);
  }
  free(xv); free(yv); free(zv);
  return lambda;
}

/* --------------------------------------------------------------- one Halpern step */
static void halpern_step(hip* s, int is_major, int k_offset) {         /* pdhg.cc:961-1018 */
  const double ps = s->primal_step, ds = s->dual_step, rho = 1.0;       /* halpern_gamma = 1 (:1912) */
  const int k = s->halpern_iteration + k_offset;
  const double w = (double)k / (k + 1.0);
  if (is_major) s->hslack_valid = 1;
  for (int i = 0; i < s->n; i++) {
    const double temp = s->x[i] - ps * (s->cost[i] - s->aty_cache[i]);
    const double proj = dmax(s->lower[i], dmin(temp, s->upper[i]));     /* projectBox, linalg.cc:17-19 */
    if (is_major) { s->xn[i] = proj; s->hslack[i] = (proj - temp) / ps; }
    s->rx[i] = 2.0 * proj - s->x[i];
  }
  l_ax(s, s->rx, s->ax_next);
  for (int j = 0; j < s->m; j++) {
    const double temp = s->y[j] / ds - s->ax_next[j];
    const double lo = -s->rup[j], up = -s->rlo[j];
    const double proj = dmax(lo, dmin(temp, up));
    const double pd = (temp - proj) * ds;
    if (is_major) s->yn[j] = pd;
    s->ry[j] = 2.0 * pd - s->y[j];
  }
  for (int i = 0; i < s->n; i++) {
    const double blended = rho * s->rx[i] + (1.0 - rho) * s->x[i];
    s->x[i] = w * blended + (1.0 - w) * s->xa[i];
  }
  for (int j = 0; j < s->m; j++) {
    const double blended = rho * s->ry[j] + (1.0 - rho) * s->y[j];
    s->y[j] = w * blended + (1.0 - w) * s->ya[j];
  }
  l_aty(s, s->y, s->aty_cache);
}

static double fixed_point_error(const hip* s) {                        /* pdhg.cc:709-740 */
  double pn = 0.0, dn = 0.0, cross = 0.0;
  double* dx = NEW(double, s->n);
  double* dy = NEW(double, s->m);
  double* atdy = NEW(double, s->n);
  for (int i = 0; i < s->n; i++) { dx[i] = s->xn[i] - s->rx[i]; pn += dx[i] * dx[i]; }
  for (int i = 0; i < s->m; i++) { dy[i] = s->yn[i] - s->ry[i]; dn += dy[i] * dy[i]; }
  l_aty(s, dy, atdy);
  for (int i = 0; i < s->n; i++) cross += dx[i] * atdy[i];
  const double movement = pn * s->omega + dn / s->omega;
  const double interaction = 2.0 * s->eta * cross;
  ((hip*)s)->sums[0] = pn; ((hip*)s)->sums[1] = dn; ((hip*)s)->sums[2] = cross;
  free(dx); free(dy); free(atdy);
  return sqrt(dmax(0.0, movement + interaction));
}

/* ---------------------------------------------------------------- convergence check */
/* checkConvergence (pdhg.cc:1474-1527) for the current iterate; use_cached = the Halpern major-step dual slack is
 * available and the slack vectors are the solver's own (computeDualSlacks, :1322-1378) */
static int check_convergence(hip* s, const double* x, const double* y, const double* ax, const double* aty, double eps) {
  const int n = s->n, m = s->m;
  double* r = NEW(double, m > n ? m : n);
  for (int i = 0; i < m; i++) {                                         /* computePrimalFeasibility, :1297-1320 */
    r[i] = ax[i] - s->rlo[i];
    if (!s->is_eq[i]) r[i] = dmin(0.0, r[i]);
  }
  if (s->is_scaled) for (int i = 0; i < m; i++) r[i] *= s->row_scale[i];
  s->sums[3] = l_dot(m, r, r);
  s->pfeas = l_norm2(m, r);
  double* dres = NEW(double, n);                                         /* computeDualFeasibility, :1380-1408 */
  for (int i = 0; i < n; i++) dres[i] = s->cost[i] - aty[i];
  for (int i = 0; i < n; i++) {
    double slack = 0.0;
    if (s->hslack_valid) slack = s->hslack[i];
    else {
      const int hl = s->lower[i] > -INFINITY, hu = s->upper[i] < INFINITY;
      if (hl && hu) slack = dres[i];
      else if (hl) slack = dmax(0.0, dres[i]);
      else if (hu) slack = dmin(0.0, dres[i]);
    }
    s->sp[i] = dmax(0.0, slack);
    s->sn[i] = dmax(0.0, -slack);
  }
  for (int i = 0; i < n; i++) r[i] = dres[i] - s->sp[i] + s->sn[i];
  if (s->is_scaled) for (int i = 0; i < n; i++) r[i] *= s->col_scale[i];
  s->sums[4] = l_dot(n, r, r);
  s->dfeas = l_norm2(n, r);
  double pobj = s->pobj;                                                /* caller preset pobj = offset */
  for (int i = 0; i < n; i++) pobj += s->cost[i] * x[i];
  s->pobj = pobj;
  double dobj = s->dobj;                                                /* computeDualObjective, :1447-1472 */
  for (int i = 0; i < m; i++) dobj += s->rlo[i] * y[i];
  for (int i = 0; i < n; i++) if (s->lower[i] > -INFINITY) dobj += s->lower[i] * s->sp[i];
  for (int i = 0; i < n; i++) if (s->upper[i] < INFINITY) dobj -= s->upper[i] * s->sn[i];
  s->dobj = dobj;
  s->sums[5] = pobj; s->sums[6] = dobj;
  const double gap = pobj - dobj;
  s->gap = fabs(gap);
  s->relgap = fabs(gap) / (1.0 + fabs(pobj) + fabs(dobj));
  free(r); free(dres);
  return s->pfeas < eps * (1.0 + s->rhs_norm) && s->dfeas < eps * (1.0 + s->c_norm) && s->relgap < eps;
}

/* runConvergenceCheck, pdhg.cc:784-899 (Halpern mode: only the current iterate is tested) */
static int run_check(hip* s, int iter, double offset, double eps, double* out_x, double* out_y) {
  int conv;
  s->pobj = offset; s->dobj = offset;
  if (iter > 0) {
    double* axp = NEW(double, s->m);
    double* atyp = NEW(double, s->n);
    l_ax(s, s->xn, axp);
    l_aty(s, s->yn, atyp);
    conv = check_convergence(s, s->xn, s->yn, axp, atyp, eps);
    free(axp); free(atyp);
  } else {
    conv = check_convergence(s, s->x, s->y, s->ax_cache, s->aty_cache, eps);
  }
  if (conv) {
    memcpy(out_x, iter > 0 ? s->xn : s->x, sizeof(double) * (size_t)s->n);
    memcpy(out_y, iter > 0 ? s->yn : s->y, sizeof(double) * (size_t)s->m);
  }
  return conv;
}

static int restart_criteria(double fpe, double fpe0, double last_trial, int hiter, int total) {   /* pdhg.cc:901-927 */
  if (total == CHECK_INTERVAL) return 1;
  if (total > CHECK_INTERVAL) {
    if (fpe <= 0.2 * fpe0) return 1;
    if (fpe <= 0.8 * fpe0) { if (fpe > last_trial) return 1; }
    if (hiter >= 0.36 * total) return 1;
  }
  return 0;
}

static void update_primal_weight(hip* s) {                             /* pdhg.cc:1979-2050, PID controller */
  const double k_p = 0.99, k_i = 0.01, k_d = 0.0, i_smooth = 0.3;       /* :1918-1920, defs.hpp:95 */
  double pd = 0.0, dd = 0.0;
  for (int i = 0; i < s->n; i++) { const double d = s->xn[i] - s->xa[i]; pd += d * d; }
  for (int j = 0; j < s->m; j++) { const double d = s->yn[j] - s->ya[j]; dd += d * d; }
  s->sums[7] = pd; s->sums[8] = dd;
  pd = sqrt(pd); dd = sqrt(dd);
  const double rel_p = s->pfeas / (1.0 + s->rhs_norm), rel_d = s->dfeas / (1.0 + s->c_norm);
  const double ratio = (rel_p > 0.0) ? (rel_d / rel_p) : 1e300;
  if (pd > 1e-16 && dd > 1e-16 && pd < 1e12 && dd < 1e12 && ratio > 1e-8 && ratio < 1e8) {
    const double error = log(dd) - log(pd) - log(s->primal_weight);
    s->err_sum = i_smooth * s->err_sum + error;
    const double delta = error - s->last_err;
    s->primal_weight *= exp(k_p * error + k_i * s->err_sum + k_d * delta);
    s->last_err = error;
  } else {
    s->primal_weight = s->best_primal_weight;
    s->err_sum = 0.0;
    s->last_err = 0.0;
  }
  const double gap = (rel_p > 0.0 && rel_d > 0.0) ? fabs(log10(rel_d / rel_p)) : s->best_gap;
  if (gap < s->best_gap) { s->best_gap = gap; s->best_primal_weight = s->primal_weight; }
  const double eta = sqrt(s->primal_step * s->dual_step);
  s->primal_step = eta / s->primal_weight;
  s->dual_step = eta * s->primal_weight;
  s->omega = s->primal_weight;
}

/* the processed + scaled LP and the power-method estimate, for parity tests of the product's host prologue:
 * arrays are caller-allocated (n0 + m columns, m rows, nnz0 + m nonzeros at most) */
int hip_form_build(const orc_lp* lp, const hip_params* prm, hip_form* f) {
  hip S; memset(&S, 0, sizeof(S));
  hip* s = &S;
  preprocess(lp, s);
  scale_problem(s, prm);
  f->n = s->n; f->m = s->m; f->nnz = s->nnz; f->neq = 0;
  for (int i = 0; i < s->m; i++) f->neq += s->is_eq[i];
  memcpy(f->cost, s->cost, sizeof(double) * (size_t)s->n); memcpy(f->lower, s->lower, sizeof(double) * (size_t)s->n);
  memcpy(f->upper, s->upper, sizeof(double) * (size_t)s->n); memcpy(f->col_scale, s->col_scale, sizeof(double) * (size_t)s->n);
  memcpy(f->rlo, s->rlo, sizeof(double) * (size_t)s->m); memcpy(f->rup, s->rup, sizeof(double) * (size_t)s->m);
  memcpy(f->row_scale, s->row_scale, sizeof(double) * (size_t)s->m);
  memcpy(f->new_idx, s->new_idx, sizeof(int) * (size_t)s->m); memcpy(f->ctype, s->ctype, sizeof(int) * (size_t)s->m);
  memcpy(f->cbeg, s->cbeg, sizeof(int) * (size_t)(s->n + 1)); memcpy(f->cidx, s->cidx, sizeof(int) * (size_t)s->nnz);
  memcpy(f->cval, s->cval, sizeof(double) * (size_t)s->nnz);
  f->c_norm = s->c_norm; f->rhs_norm = s->rhs_norm;
  f->op_norm_sq = power_method(s);
  free(s->cost); free(s->lower); free(s->upper); free(s->rlo); free(s->rup); free(s->cbeg); free(s->cidx); free(s->cval);
  free(s->ctype); free(s->new_idx); free(s->is_eq); free(s->col_scale); free(s->row_scale);
  return 0;
}

/* ------------------------------------------------------------------------- driver */
int hip_solve(const orc_lp* lp, const hip_params* prm, hip_result* out) {
  hip S; memset(&S, 0, sizeof(S));
  hip* s = &S;
  preprocess(lp, s);
  scale_problem(s, prm);
  const int n = s->n, m = s->m;
  /* initializeStepSizes, pdhg.cc:1944-1977 */
  s->omega = (s->c_norm + 1.0) / (s->rhs_norm + 1.0);
  s->primal_weight = s->omega;
  s->best_primal_weight = s->primal_weight;
  const double op_norm_sq = power_method(s);
  const double base_step = 0.998 / sqrt(op_norm_sq);
  s->eta = base_step;
  s->primal_step = base_step / s->omega;
  s->dual_step = base_step * s->omega;
  /* initialize, :1138-1178, and the start of solve, :494-560 */
  s->x = NEW(double, n); s->y = NEW(double, m); s->xn = NEW(double, n); s->yn = NEW(double, m);
  s->rx = NEW(double, n); s->ry = NEW(double, m); s->xa = NEW(double, n); s->ya = NEW(double, m);
  s->ax_cache = NEW(double, m); s->aty_cache = NEW(double, n); s->ax_next = NEW(double, m);
  s->sp = NEW(double, n); s->sn = NEW(double, n); s->hslack = NEW(double, n);
  s->best_gap = INFINITY;
  for (int i = 0; i < n; i++) {                                          /* projectBounds, linalg.cc:23-32 */
    if (s->x[i] > s->upper[i]) s->x[i] = s->upper[i];
    if (s->x[i] < s->lower[i]) s->x[i] = s->lower[i];
  }
  memcpy(s->xa, s->x, sizeof(double) * (size_t)n);
  memcpy(s->ya, s->y, sizeof(double) * (size_t)m);
  l_ax(s, s->x, s->ax_cache);
  l_aty(s, s->y, s->aty_cache);
  double* ox = NEW(double, n);   /* the x, y handed to solve(): written only on convergence */
  double* oy = NEW(double, m);
  int term = HIP_MAXITER, iters = 0, do_restart = 0;
  double fpe = 0.0, fpe0 = 0.0, last_trial = INFINITY;
  if (run_check(s, 0, lp->offset, prm->tolerance, ox, oy)) { term = HIP_OPTIMAL; }
  else {
    while (iters < prm->max_iterations) {
      double* tr = (out->trace && out->trace_len < out->trace_cap) ? out->trace + (size_t)out->trace_len * HIP_TRACE_COLS : NULL;
      if (tr) memset(tr, 0, sizeof(double) * HIP_TRACE_COLS);
      halpern_step(s, 1, 1);
      if (do_restart) {
        fpe = fixed_point_error(s); fpe0 = fpe; do_restart = 0;
        if (tr) { tr[10] = s->sums[0]; tr[11] = s->sums[1]; tr[12] = s->sums[2]; tr[13] = 1.0; }
      }
      for (int i = 2; i <= CHECK_INTERVAL - 1; i++) halpern_step(s, 0, i);
      halpern_step(s, 1, CHECK_INTERVAL);
      fpe = fixed_point_error(s);
      s->halpern_iteration += CHECK_INTERVAL;
      iters += CHECK_INTERVAL;
      const int conv = run_check(s, iters, lp->offset, prm->tolerance, ox, oy);
      if (tr) {
        /* the PID distances are part of the block's nine sums whether or not a restart follows */
        double pd2 = 0.0, dd2 = 0.0;
        for (int i = 0; i < n; i++) { const double d = s->xn[i] - s->xa[i]; pd2 += d * d; }
        for (int j = 0; j < m; j++) { const double d = s->yn[j] - s->ya[j]; dd2 += d * d; }
        s->sums[7] = pd2; s->sums[8] = dd2;
        tr[0] = iters;
        for (int q = 0; q < 9; q++) tr[1 + q] = s->sums[q];
        tr[18] = fpe; tr[19] = conv;
        out->trace_len++;
      }
      if (conv) { term = HIP_OPTIMAL; break; }
      do_restart = restart_criteria(fpe, fpe0, last_trial, s->halpern_iteration, iters);
      last_trial = fpe;
      if (tr) tr[14] = do_restart;
      if (do_restart) {
        if (prm->step_size_strategy == 3) update_primal_weight(s);
        if (tr) { tr[15] = s->primal_weight; tr[16] = s->primal_step; tr[17] = s->dual_step; }
        memcpy(s->xa, s->xn, sizeof(double) * (size_t)n); memcpy(s->ya, s->yn, sizeof(double) * (size_t)m);
        memcpy(s->x, s->xn, sizeof(double) * (size_t)n); memcpy(s->y, s->yn, sizeof(double) * (size_t)m);
        l_ax(s, s->x, s->ax_cache);
        l_aty(s, s->y, s->aty_cache);
        s->halpern_iteration = 0;
        last_trial = INFINITY;
      }
    }
  }
  /* unscaleSolution (pdhg.cc:1883-1897, scaling.cc:265-276) + postprocess (:359-492) */
  if (s->is_scaled) {
    for (int i = 0; i < n; i++) ox[i] /= s->col_scale[i];
    for (int i = 0; i < m; i++) oy[i] /= s->row_scale[i];
  }
  for (int i = 0; i < n; i++) { s->sp[i] *= s->col_scale[i]; s->sn[i] *= s->col_scale[i]; }
  for (int j = 0; j < lp->n; j++) out->col_value[j] = ox[j];
  for (int i = 0; i < lp->m; i++) {
    const double d = oy[s->new_idx[i]];
    out->row_dual[i] = s->ctype[i] == T_LEQ ? -d : d;
  }
  for (int i = 0; i < lp->m; i++) out->row_value[i] = 0.0;
  for (int c = 0; c < lp->n; c++) {
    const double xv = ox[c];
    for (int p = lp->start[c]; p < lp->start[c + 1]; p++) out->row_value[lp->index[p]] += lp->value[p] * xv;
  }
  for (int j = 0; j < lp->n; j++) { out->col_dual[j] = s->sp[j] - s->sn[j]; out->col_dual[j] *= lp->sense; }
  out->term_code = term;
  out->iters = iters;
  out->pfeas = s->pfeas; out->dfeas = s->dfeas; out->pobj = s->pobj; out->dobj = s->dobj; out->relgap = s->relgap;
  out->primal_weight = s->primal_weight; out->op_norm_sq = op_norm_sq;
  free(ox); free(oy);
  free(s->cost); free(s->lower); free(s->upper); free(s->rlo); free(s->rup); free(s->cbeg); free(s->cidx); free(s->cval);
  free(s->ctype); free(s->new_idx); free(s->is_eq); free(s->col_scale); free(s->row_scale);
  free(s->x); free(s->y); free(s->xn); free(s->yn); free(s->rx); free(s->ry); free(s->xa); free(s->ya);
  free(s->ax_cache); free(s->aty_cache); free(s->ax_next); free(s->sp); free(s->sn); free(s->hslack);
  return 0;
}
