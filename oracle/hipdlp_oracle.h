/* oracle/hipdlp_oracle.h -- TEST INFRASTRUCTURE ONLY (same rules as pdlp_oracle.h: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline leg may use it; the product never links it).
 *
 * CPU restatement of the reference's HiPDLP engine (`solver=hipdlp`, reflected Halpern PDHG):
 *   Highs::run -> solveLp -> solveLpHiPdlp (pdlp/HiPdlpWrapper.cpp:26-141) -> PDLPSolver (pdlp/hipdlp/).
 * SURVEY.md 8(a) row a20, 8(f) rank 2 -- the oracle for the NEXT algorithm mode of the engine.
 * Parity status: PINNED against oracle/_ref (tests/test_hipdlp_oracle.py: iteration counts and all four
 * HighsSolution vectors bit for bit on the reference's own LP instances, several option sets).
 */
#ifndef HIPDLP_ORACLE_H_
#define HIPDLP_ORACLE_H_

#include "pdlp_oracle.h"   /* orc_lp */

#ifdef __cplusplus
extern "C" {
#endif

enum { HIP_OPTIMAL = 0, HIP_MAXITER = 1 };

typedef struct {
  double tolerance;          /* pdlp_optimality_tolerance / kkt_tolerance (pdhg.cc:1822-1824) */
  int max_iterations;        /* pdlp_iteration_limit */
  int use_ruiz, use_pc, use_l2;   /* pdlp_scaling_mode bits 1 / 4 / 2 (default 5 = Ruiz + PC) */
  int ruiz_iterations;       /* pdlp_ruiz_iterations (default 10) */
  int step_size_strategy;    /* 0 fixed, 3 PID (every other option value means PID, pdhg.cc:1854-1863) */
} hip_params;

typedef struct {
  double *col_value, *col_dual, *row_value, *row_dual;   /* caller-allocated n, n, m, m */
  int term_code, iters;
  double pfeas, dfeas, pobj, dobj, relgap;               /* of the last convergence check (scaled-space objective) */
  double primal_weight, op_norm_sq;
  /* optional trace, one row per block of 40 steps: 0 iterations, 1..9 the nine sums of the block-end check (|dx|^2, |dy|^2,
   * cross term, |primal residual|^2, |dual residual|^2, primal objective, dual objective, |x_next - anchor|^2,
   * |y_next - anchor|^2), 10..12 the three fixed-point sums of the step after a restart (13 = 1 when present),
   * 14 restart decided, 15..17 primal weight / primal step / dual step after it, 18 fixed-point error, 19 converged */
  double* trace;
  int trace_cap, trace_len;
} hip_result;
#define HIP_TRACE_COLS 20

int hip_solve(const orc_lp* lp, const hip_params* prm, hip_result* out);

/* processed (pdhg.cc:152-358) + scaled (scaling.cc) LP and the power-method estimate of |A|^2 (pdhg.cc:1529-1671);
 * caller-allocated arrays: n0 + m columns, m rows, nnz0 + m nonzeros at most.
 * ctype: 0 EQ, 1 LEQ, 2 GEQ, 3 BOUND, 4 FREE by ORIGINAL row; new_idx: original row -> processed row */
typedef struct {
  int n, m, nnz, neq;
  double *cost, *lower, *upper, *rlo, *rup;
  int *cbeg, *cidx;
  double* cval;
  double *col_scale, *row_scale;
  int *new_idx, *ctype;
  double c_norm, rhs_norm, op_norm_sq;
} hip_form;
int hip_form_build(const orc_lp* lp, const hip_params* prm, hip_form* f);

/* test switch: k > 0 makes the dot products add in blocks of k (another rounding order); 0 (default) = the reference's */
void hip_set_sum_block(int k);

#ifdef __cplusplus
}
#endif
#endif
