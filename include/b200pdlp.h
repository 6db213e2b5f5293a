/* include/b200pdlp.h -- C ABI of the CUDA PDLP engine for the H100 (libb200pdlp.so).
 *
 * This is the drop-in boundary underneath HiGHS's
 *     HighsStatus solveLpCupdlp(HighsLpSolverObject&)
 * (/root/reference/highs/pdlp/CupdlpWrapper.cpp:23-278, called from
 * /root/reference/highs/lp_data/HighsSolve.cpp:97-104).  Plain pointers and
 * sizes only -- no HiGHS, torch or C++ types -- so the same library is bound
 * from the C++ shim in highs_b200/csrc/highs_shim.cpp (INTEGRATION.md) and from
 * Python (ctypes, highs_b200/engine.py).
 *
 * All arithmetic is IEEE fp64; indices are 32-bit (cupdlp_int,
 * highs/pdlp/cupdlp/glbopts.h:249-253; HighsInt without HIGHSINT64).
 * Every entry point returns 0 on success and a negative b200pdlp_error
 * otherwise; b200pdlp_last_error() gives the message.  There is NO CPU
 * fallback: without a CUDA device the compute entry points fail with
 * B200PDLP_ERR_CUDA.
 */
#ifndef B200PDLP_H_
#define B200PDLP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200PDLP_VERSION 100

typedef enum {
  B200PDLP_OK = 0,
  B200PDLP_ERR_ARG = -1,     /* bad argument */
  B200PDLP_ERR_CUDA = -2,    /* CUDA runtime / no device */
  B200PDLP_ERR_NCCL = -3,
  B200PDLP_ERR_ALLOC = -4,
  B200PDLP_ERR_STATE = -5
} b200pdlp_error;

/* termination codes: numbering of cupdlp_defs.h:61-68 */
typedef enum {
  B200PDLP_OPTIMAL = 0,
  B200PDLP_INFEASIBLE = 1,
  B200PDLP_UNBOUNDED = 2,
  B200PDLP_INFEASIBLE_OR_UNBOUNDED = 3,
  B200PDLP_TIMELIMIT_OR_ITERLIMIT = 4,
  B200PDLP_FEASIBLE = 5
} b200pdlp_term;

/* HighsLp members read by solveLpCupdlp (HighsLp.h:23-35, CupdlpWrapper.cpp:280-300).
 * The matrix is column-wise (asserted by the caller, Highs.cpp:4130). */
typedef struct {
  int32_t num_col, num_row;
  const int32_t* a_start;    /* [num_col+1] */
  const int32_t* a_index;    /* [nnz] row indices */
  const double* a_value;     /* [nnz] */
  const double* col_cost;    /* [num_col] */
  const double* col_lower;   /* [num_col]; <= -1e20 means -inf (CupdlpWrapper.cpp:375-378) */
  const double* col_upper;
  const double* row_lower;   /* [num_row]; thresholds +-1e20 (CupdlpWrapper.cpp:316-317) */
  const double* row_upper;
  double sense;              /* +1 minimise, -1 maximise (ObjSense) */
  double offset;
} b200pdlp_lp;

/* What getUserParamsFromOptions (CupdlpWrapper.cpp:642-717) hands to cuPDLP-C. */
typedef struct {
  int32_t iter_limit;        /* pdlp_iteration_limit (N_ITER_LIM) */
  double tol_primal;         /* D_PRIMAL_TOL */
  double tol_dual;           /* D_DUAL_TOL */
  double tol_gap;            /* D_GAP_TOL */
  double time_limit;         /* D_TIME_LIM, seconds; < 0 or inf = none; 0 = already over (the first check ends the run) */
  int32_t scaling;           /* IF_SCALING: 1 = Ruiz x10 + Pock-Chambolle(1) */
  int32_t adaptive_step;     /* E_LINE_SEARCH_METHOD: 1 adaptive, 0 fixed (power method) */
  int32_t restart;           /* E_RESTART_METHOD: 1 on, 0 off */
  int32_t log_level;         /* N_LOG_LEVEL 0/1/2 */
  int32_t check_interval;    /* CUPDLP_RELEASE_INTERVAL; 0 -> 40 */
  int32_t device;            /* CUDA device ordinal; -1 = current */
  int32_t graph_passes;      /* PDHG passes captured per CUDA graph; 0 -> check_interval */
  int32_t ordered_max;       /* problems with max(cols,rows) <= this reduce in the reference's
                                sequential order (bit-identical trajectories); 0 -> 4096, <0 -> off */
  int32_t device_scaling;    /* where the prologue (formulate, scaling, transposition, layouts) runs: 0 = on the device for one
                                GPU in tree mode (device_prep.cu; host threads otherwise), -1 = always host threads;
                                any other value is rejected (B200PDLP_ERR_ARG) */
  int32_t reserved[2];
} b200pdlp_params;

/* Hot start = incoming HighsSolution when value_valid && dual_valid
 * (PDHG_PreSolve, cupdlp_solver.c:1217-1279).  NULL pointer = cold start. */
typedef struct {
  const double* col_value;   /* [num_col] */
  const double* row_value;   /* [num_row] (slack of BOUND rows) */
  const double* row_dual;    /* [num_row] */
} b200pdlp_warm;

typedef struct {
  /* caller-allocated HighsSolution storage, original LP space, HiGHS signs
   * (PDHG_PostSolve, cupdlp_solver.c:1281-1435) */
  double* col_value;         /* [num_col] */
  double* col_dual;          /* [num_col] */
  double* row_value;         /* [num_row] */
  double* row_dual;          /* [num_row] */
  int32_t value_valid, dual_valid;
  int32_t term_code;         /* b200pdlp_term */
  int32_t term_iterate;      /* 0 last iterate, 1 average iterate */
  int32_t iters;             /* -> HighsInfo::pdlp_iteration_count */
  int32_t passes;            /* PDHG passes executed (iters + rejected line-search steps) */
  int32_t restarts;
  int32_t kernel_launches;   /* kernels this library launched inside the solve */
  /* cuPDLP-C's own residuals of the returned iterate (unscaled space) */
  double primal_obj, dual_obj, primal_feas, dual_feas, gap, rel_gap;
  /* timings, seconds */
  double setup_seconds;      /* formulate + scale + layout + H2D */
  double solve_seconds;      /* PDHG loop, host wall clock */
  double iter_device_ms;     /* CUDA-event time of the PDHG passes only */
  double loop_device_ms;     /* CUDA-event time of the whole loop: passes + check iterations + restarts */
  /* form dimensions actually solved */
  int32_t form_cols, form_rows, form_nnz, form_neq;
  /* optional trajectory trace, one row of B200PDLP_TRACE_COLS doubles per check iteration:
   * 0 iter, 1 pobj, 2 dobj, 3 pfeas, 4 dfeas (current iterate), 5-8 same for the average,
   * 9 tau, 10 sigma, 11 beta (after a restart's update), 12 restart (0 none, 1 average, 2 current),
   * 13 nStepSizeIter, 14 sum of step weights, 15 reserved */
  double* trace;             /* caller-allocated [trace_cap][16] or NULL */
  int32_t trace_cap, trace_len;
} b200pdlp_result;
#define B200PDLP_TRACE_COLS 16
/* The HiPDLP solves (b200pdlp_solve_hipdlp, _multi) write one row of B200PDLP_HIP_TRACE_COLS doubles per block of 40 steps
 * instead, from the block-end check (no extra device work): 0 iterations, 1-9 the nine sums of the check (|x_next - refl_x|^2,
 * |y_next - refl_y|^2, the fixed-point cross term, |primal residual|^2, |dual residual|^2, primal objective, dual objective,
 * |x_next - x_anchor|^2, |y_next - y_anchor|^2; see b200pdlp_hipdlp_check), 10 restart decided, 11-13 primal weight, primal
 * step, dual step after the restart's update (0 when there is no restart), 14 fixed-point error, 15 converged.  These are
 * columns 0-9 and 14-19 of the HiPDLP oracle's trace (oracle/hipdlp_oracle.h). */
#define B200PDLP_HIP_TRACE_COLS 16

/* ---- whole solve: the function the HiGHS shim calls ------------------------ */
void b200pdlp_default_params(b200pdlp_params* p);
int b200pdlp_solve(const b200pdlp_lp* lp, const b200pdlp_params* params,
                   const b200pdlp_warm* warm, b200pdlp_result* out);

/* The same solve on `ngpus` devices of THIS process (devices[g] or, if NULL, ordinals 0..ngpus-1): one problem per device
 * wired with b200pdlp_p2p_link_local, one host thread per rank, no NCCL.  ngpus <= 1 is b200pdlp_solve.
 * (what the HiGHS shim uses when B200PDLP_GPUS > 1; the one-process-per-GPU entry points are further below) */
int b200pdlp_solve_multi(const b200pdlp_lp* lp, const b200pdlp_params* params, const b200pdlp_warm* warm,
                         b200pdlp_result* out, int32_t ngpus, const int32_t* devices);

/* Solve `count` independent LPs on one GPU in one call.  Every member must be an ordered-mode problem of `params`
 * (standard form max(n, m) <= ordered_max); each returns exactly what b200pdlp_solve(lps[i], params, warms[i]) returns:
 * term_code, term_iterate, iters, passes, restarts, the residual scalars, the trace rows and all four vectors, bit for bit.
 * All members share `params` (tolerances, limits, check_interval, scaling, adaptive step, restart); `device` selects the GPU.
 * One CTA solves one member; the members' host prologues run on host threads.  The time limit counts from the start of the
 * batch's PDHG loop.  These fields are batch-wide, the same in every outs[i]: setup_seconds, solve_seconds, loop_device_ms,
 * iter_device_ms and kernel_launches (= the batch's rounds, one launch each).
 * Returns B200PDLP_ERR_ARG before any device work for count < 0, NULL arrays, a member that the checks of b200pdlp_solve
 * reject, ordered_max < 0, or a member whose standard form exceeds ordered_max; b200pdlp_last_error() names the member's
 * index, and no result is written.  count == 0: B200PDLP_OK.  No device: B200PDLP_ERR_CUDA.  The whole batch must fit in
 * device memory (B200PDLP_ERR_ALLOC otherwise).
 * STATUS: runs on hardware; tests/test_gpu_batch.py (byte equality with b200pdlp_solve and with the oracle), tools/batch_bench.py. */
int b200pdlp_solve_batch(int32_t count, const b200pdlp_lp* lps, const b200pdlp_params* params,
                         const b200pdlp_warm* warms /* [count] or NULL; a member whose pointers are NULL starts cold */,
                         b200pdlp_result* outs /* [count], caller-allocated like b200pdlp_result */);

/* b200pdlp_solve_batch for LPs that are already in GPU memory.  `lps`, `warms` and `outs` are host arrays of the usual
 * structs, but every array pointer inside them is device (or managed) memory of params->device (< 0: the current device):
 * the LP's eight arrays, the three warm vectors and the four result vectors.  num_col, num_row, sense and offset are host
 * scalars; `trace` stays a host pointer.  Each member returns exactly what b200pdlp_solve_batch returns for it with the same
 * arrays on the host (and so what b200pdlp_solve returns for it alone): term_code, term_iterate, iters, passes, restarts, the
 * residual scalars, the trace rows, the form dimensions and the four vectors, bit for bit.  Batch-wide fields as in
 * b200pdlp_solve_batch; setup_seconds covers validation, sizing and the device prologue.
 * The prologue (formulate, scaling, layouts, start point) and the postsolve run on the device, one CTA per member; the host
 * reads a few scalars per member, never an array.  The call returns once the outputs are complete on the device; it never
 * writes an input array.  The caller must have finished writing the inputs before the call (the library uses a stream of
 * its own).
 * Returns B200PDLP_ERR_ARG before any device work for count < 0, NULL arrays, ordered_max < 0, a bad device_scaling or a
 * sense other than +-1; then, naming the member and the field, for a pointer that is not device memory of the device; then,
 * before any solve work and naming the lowest failing member, for what b200pdlp_solve's checks reject in the arrays
 * (a_start[0] != 0, a decreasing a_start, an a_index outside [0, num_row)) and for a standard form larger than ordered_max.
 * No result field or array is written on an error.  count == 0: B200PDLP_OK.  No device: B200PDLP_ERR_CUDA.  The whole batch
 * must fit in device memory (B200PDLP_ERR_ALLOC otherwise).
 * STATUS: runs on hardware; tests/test_gpu_batch_device.py (byte equality with b200pdlp_solve_batch),
 * tools/batch_device_bench.py. */
int b200pdlp_solve_batch_device(int32_t count, const b200pdlp_lp* lps, const b200pdlp_params* params,
                                const b200pdlp_warm* warms /* [count] or NULL; device vectors; a member whose pointers are NULL starts cold */,
                                b200pdlp_result* outs /* [count]; vectors in device memory */);

/* b200pdlp_solve for an LP that is already in GPU memory, at any size.  Pointers follow b200pdlp_solve_batch_device's rules:
 * the LP's eight arrays, the three warm vectors and the four result vectors are device (or managed) memory of params->device
 * (< 0: the current device); num_col, num_row, sense and offset are host scalars; `trace` stays a host pointer.  Returns
 * exactly what b200pdlp_solve returns for host copies of the same arrays with the same params, cold or warm: term_code,
 * term_iterate, iters, passes, restarts, the residual scalars, the form dimensions, the trace rows and the four vectors, bit
 * for bit.  The call never writes an input, uses a stream of its own and returns once the outputs are complete on the device.
 * The four result vectors may be NULL only together (then none is written).  One grid-wide sizing kernel validates the arrays and counts the slack rows (one read-back); then the route:
 *  - tree mode (the standard form past ordered_max, and rows, columns and nonzeros): b200pdlp_solve's device prologue reads
 *    the eight arrays in place (no copy of the LP: B200PDLP_TIMING=1 prints "LP arrays copied to the device: 0 bytes"), the
 *    hot start goes straight to the initial point and the postsolve writes the caller's vectors.  device_scaling = -1 and
 *    B200PDLP_DEVICE_PREP=0 are ignored: the result is b200pdlp_solve's with its default, device prologue;
 *  - ordered mode: b200pdlp_solve_batch_device with this one LP; setup_seconds, solve_seconds, loop_device_ms,
 *    iter_device_ms and kernel_launches are then the batch's (kernel_launches = its rounds);
 *  - an LP without rows, columns or nonzeros past ordered_max (it has no matrix): its vectors are copied to the host, solved
 *    as b200pdlp_solve solves them (host prologue), and the four result vectors copied back.
 * Returns B200PDLP_ERR_ARG, with nothing written, in b200pdlp_solve_batch_device's order: before any device work for NULL
 * arguments, a bad device_scaling, a malformed b200pdlp_lp or a sense other than +-1; then, naming the field, for a pointer
 * that is not device memory of the device; then, with b200pdlp_solve's messages and in its order, for a malformed a_start or
 * a_index (a_index is read only once a_start has passed).  No device: B200PDLP_ERR_CUDA.
 * Known limitation: an LP without rows past ordered_max takes b200pdlp_solve's host path, which does not return on such an
 * LP today (b200pdlp_solve_hipdlp_device solves it).
 * STATUS: runs on hardware; tests/test_gpu_solve_device.py (byte equality with b200pdlp_solve on host copies),
 * tools/solve_device_bench.py. */
int b200pdlp_solve_device(const b200pdlp_lp* lp, const b200pdlp_params* params,
                          const b200pdlp_warm* warm /* NULL or device vectors */, b200pdlp_result* out /* device vectors */);

/* ---- persistent problem handle (bench + kernel-level parity tests) --------- */
typedef struct b200pdlp_problem b200pdlp_problem;

/* formulate + scale on the host, build the blocked row-major layouts of A and
 * A^T, upload to HBM.  rank/world select a contiguous, nnz-balanced block of
 * the (permuted) rows for multi-GPU; pass 0/1 for a single GPU. */
int b200pdlp_problem_create(const b200pdlp_lp* lp, const b200pdlp_params* params,
                            int32_t rank, int32_t world, b200pdlp_problem** out);
void b200pdlp_problem_destroy(b200pdlp_problem* p);
/* dims[0..7] = form cols, form rows (global), nnz (global), neq, local rows,
 * local row offset, local nnz, original cols */
int b200pdlp_problem_dims(const b200pdlp_problem* p, int32_t dims[8]);
/* host copies of the scaled standard form (for parity tests against the oracle):
 * which = 0 cost, 1 lower, 2 upper, 3 rhs, 4 col_scale, 5 row_scale (doubles);
 * returns number of doubles written (<= cap) */
int b200pdlp_problem_get_vector(const b200pdlp_problem* p, int32_t which, double* dst, int32_t cap);
/* CSR of the scaled matrix (global row numbering of this rank's rows) */
int b200pdlp_problem_get_csr(const b200pdlp_problem* p, int32_t* rowptr, int32_t* col, double* val);

/* single kernels on host vectors (H2D, kernel, D2H) -- parity tests only:
 * ax[m_local] = A_local x[n];  aty[n] = A_local^T y[m_local] */
int b200pdlp_spmv_ax(b200pdlp_problem* p, const double* x, double* ax);
int b200pdlp_spmv_aty(b200pdlp_problem* p, const double* y, double* aty);
/* single FUSED kernels of the hot path on host vectors in standard-form order (parity tests; single GPU).  Reference
 * analogues: the extern "C" launchers of highs/pdlp/cupdlp/cuda/cupdlp_cudalinalg.cu:13-386.
 *  primal step (K1): x_new = proj_[l,u](x - tau (c - aty))   (PDHG_primalGradientStep, cupdlp_step.c:16-40), *dx2 = |x - x_new|^2
 *  dual step (K2):   ax_new = A x_new;  y_new = y + sigma (b - 2 ax_new + ax), max(.,0) on inequality rows
 *                    (PDHG_dualGradientStep, cupdlp_step.c:43-69), *dy2 = |y - y_new|^2
 *  residuals:        out[10] = pobj, dobj, primal feasibility, dual feasibility, gap, relative gap, primal-ray objective
 *                    and residual, dual-ray objective and residual of (x, y) (cupdlp_solver.c:12-204, :206-471)
 * all on the SCALED standard form the problem holds (b200pdlp_problem_get_vector / get_csr return it). */
int b200pdlp_primal_step(b200pdlp_problem* p, const double* x, const double* aty, double tau, double* x_new, double* dx2);
int b200pdlp_dual_step(b200pdlp_problem* p, const double* x_new, const double* y, const double* ax, double sigma,
                       double* y_new, double* ax_new, double* dy2);
int b200pdlp_residuals(b200pdlp_problem* p, const double* x, const double* y, double out[10]);

/* One check iteration of a tree-mode solve, on the device (parity tests; one GPU): the launches the solve's check graphs
 * capture (engine.cu enqueue_check_device), run once without a graph.  C1 flushes the pending weight into xSum / ySum and
 * forms the averages, C2 multiplies them by A and A' (split variant only), C3 adds the 8 row-side and 20 column-side sums of
 * both iterates, C4 forms the residuals and decides (termination, infeasibility, limits, restart choice), C5 restarts the
 * vectors, C6 updates the step sizes and primal weight, writes the trace row, sets the next check iteration and fills the
 * step-rule power tables.  The scalars in `in` become the PdhgState / SolveCtl of the check (sense and offset are the
 * problem's; stop_iter = iter, so the check is due).  light = 1 runs the dense-check phase's variant: A xbar and A'ybar come
 * from the carried axsum = A xSum and atysum = A'ySum instead of two SpMVs.
 * Vectors are host arrays in standard-form order, read on entry and overwritten with their values after the check:
 * x, y (current iterate), ax, aty (its products, the caller's values), xsum, ysum, xlr, ylr (last restart point), and for
 * light = 1 axsum, atysum (NULL otherwise).  Written only: xavg, yavg (the averages), axavg = A xavg, atyavg = A'yavg.
 * Rejected with B200PDLP_ERR_ARG before anything is written: NULL arguments, a problem in ordered mode, on several GPUs or of
 * b200pdlp_hipdlp_problem_create, interval < 1, iter or step_iter < 0, and light = 1 when iter >= 10 (the dense-check
 * phase) or the problem carries no A xSum.  No device: B200PDLP_ERR_CUDA. */
typedef struct {
  int32_t iter, step_iter, adaptive, pending;    /* PdhgState */
  double beta, tau, sigma, sum_step, w_pending;
  double tol_p, tol_d, tol_gap;                  /* SolveCtl: tol_p / tol_d absolute (already times 1 + |b| / 1 + |c|) */
  int32_t iter_limit, interval, restart_on;
  int32_t time_flag;                             /* the value of the time-limit word the check reads */
  double pf_lr, df_lr, gap_lr, pf_lc, df_lc, gap_lc;   /* restart memo: at the last restart, at the last candidate */
  int32_t last_restart_iter;
  int32_t light;
} b200pdlp_check_in;
typedef struct {
  double sums[28];          /* 0-3 row side of the current iterate (y.b, |primal residual|^2, |y|^2, |ray residual|^2),
                               4-7 the same for the average, 8-17 column side of the current iterate, 18-27 of the average */
  double res[2][10];        /* current, average: pobj, dobj, pfeas, dfeas, gap, relgap, pinf_obj, pinf_res, dinf_obj, dinf_res */
  int32_t term;             /* -1 the solve goes on, else a b200pdlp_term */
  int32_t term_iterate;     /* 0 current, 1 average (term == OPTIMAL) */
  int32_t restart_choice;   /* 0 none, 1 to the average, 2 to the current iterate (trace column 12) */
  int32_t restarts, checks, trace_len, done, stop_iter, pending, pow_base;
  double pf_lr, df_lr, gap_lr, pf_lc, df_lc, gap_lc;   /* the memo after the check */
  int32_t last_restart_iter, reserved;
  double beta, tau, sigma, eta, tau_try, sigma_try, sum_step;   /* eta, tau_try, sigma_try enter as NaN */
  double restart_sq[2];     /* on a restart: |x - xlr|^2, |y - ylr|^2 as C6 added them (0 otherwise) */
  double pow_red[128], pow_grow[128];   /* enter as NaN */
  double trace[16];         /* the check's trace row (B200PDLP_TRACE_COLS) */
} b200pdlp_check_out;
int b200pdlp_check_device(b200pdlp_problem* p, const b200pdlp_check_in* in, double* x, double* y, double* ax, double* aty,
                          double* xsum, double* ysum, double* xlr, double* ylr, double* axsum, double* atysum, double* xavg,
                          double* yavg, double* axavg, double* atyavg, b200pdlp_check_out* out);

/* One PDHG pass of a tree-mode solve and the partial sums it leaves (parity tests; one GPU): K1 (primal step, |dx|^2), K2
 * (A x' + dual step, |dy|^2) and K3 (A'y' + interaction) by the launchers of the solve's pass graph under the problem's SpMV
 * shapes (zero-skip, tiled, persistent), then step_rule_kernel (K4).  Inputs are host arrays in standard-form order: x, aty
 * (n), y, ax (m) and the step sizes tau, sigma; written: x_new, aty_new (n), y_new, ax_new (m).
 * slots[3][cap]: the partial-sum slots of K1, K2 and K3 as the launches left them (out->slots[k] entries each).
 * long_rows[long_cap][3]: one record {standard-form row, first slot, segments} per long row of A (out->long_a records), then
 * per long row of A' = long column of A (out->long_at).  A long row's segments have the slots first .. first + segments - 1;
 * its epilogue term goes to the first one, and every other one holds +0.0.
 * out->dx2, dy2, inter: K4's sums, read from the state block.
 * Rejected with B200PDLP_ERR_ARG before anything is written: NULL arguments, a problem in ordered mode, on several GPUs or
 * of b200pdlp_hipdlp_problem_create, cap below the longest slot array and long_cap below the number of long rows.
 * No device: B200PDLP_ERR_CUDA. */
typedef struct {
  double dx2, dy2, inter;
  int32_t slots[3];         /* K1, K2, K3 */
  int32_t long_a, long_at;  /* long rows of A, of A' */
} b200pdlp_pass_out;
int b200pdlp_pass_partials(b200pdlp_problem* p, const double* x, const double* y, const double* ax, const double* aty,
                           double tau, double sigma, double* x_new, double* y_new, double* ax_new, double* aty_new,
                           double* slots, int32_t cap, int32_t* long_rows, int32_t long_cap, b200pdlp_pass_out* out);

/* device-pointer variants on the problem's stream (bench roofline loop):
 * time `reps` back-to-back launches with CUDA events; returns ms in *ms_total */
int b200pdlp_bench_spmv(b200pdlp_problem* p, int32_t which /*0 Ax, 1 ATy*/, int32_t reps, float* ms_total);

/* per-kernel CUDA-event timing of `reps` PDHG passes in their real sequence (K1 primal step,
 * K2 A x + dual step, K3 A'y + interaction [+ all-reduce and K3b when world > 1]); call after a
 * solve (it continues from that state).  ms[0..3] = summed ms of K1, K2, K3, rest */
int b200pdlp_bench_pass(b200pdlp_problem* p, int32_t reps, float ms[4]);

/* run the PDHG loop on an uploaded problem (bench "value": inputs resident in HBM) */
int b200pdlp_problem_solve(b200pdlp_problem* p, const b200pdlp_params* params,
                           const b200pdlp_warm* warm, b200pdlp_result* out);

/* ---- multi-GPU: one process per GPU, NCCL over NVLink ---------------------- */
/* rank 0 obtains the id and ships it to the other ranks (torch.distributed /
 * any byte transport); every rank then calls comm_init.  id is 128 bytes. */
int b200pdlp_nccl_unique_id(uint8_t id[128]);
int b200pdlp_comm_init(b200pdlp_problem* p, const uint8_t id[128]);

/* fused NVLink path (optional, after comm_init): every rank exports CUDA-IPC handles of its exchange
 * buffers (B200PDLP_IPC_BYTES bytes), the host application all-gathers them (rank order) and every rank
 * imports the world x B200PDLP_IPC_BYTES blob.  From then on the per-iteration reduce-scatter and
 * all-gather run inside the engine's own kernels over peer memory; NCCL is used at check iterations only. */
#define B200PDLP_IPC_BYTES 256
int b200pdlp_p2p_export(b200pdlp_problem* p, uint8_t handles[B200PDLP_IPC_BYTES]);
int b200pdlp_p2p_import(b200pdlp_problem* p, const uint8_t* all_handles);
/* unmap the peers' buffers (call on every rank, then synchronise the ranks, BEFORE any rank destroys its problem) */
int b200pdlp_p2p_release(b200pdlp_problem* p);
/* G logical shards inside ONE process (SURVEY.md 8(e): "the same code path must run with G logical shards on 1
 * device"): probs[] holds one problem per rank of the same world, all created by this process (normally on the
 * same device); their buffers are wired to each other directly instead of through CUDA IPC, and no NCCL
 * communicator is needed.  Every rank's b200pdlp_problem_solve must then run on its own host thread. */
int b200pdlp_p2p_link_local(b200pdlp_problem** probs, int32_t count);
/* device-side timeline of the fused path since the last call, per-pass averages in us: [0] primal-shard phase,
 * [1] barrier 0 total, [2] of which waiting, [3] A x + A'y phase, [4] barrier 1 total, [5] of which waiting, [6] passes */
int b200pdlp_p2p_timeline(b200pdlp_problem* p, double out_us[8]);

/* ---- host-only view of the standard form (no GPU needed; parity tests) -------
 * formulate (CupdlpWrapper.cpp:280-448) + scale (cupdlp_scaling.c:233-425) only. */
typedef struct b200pdlp_form b200pdlp_form;
int b200pdlp_form_create(const b200pdlp_lp* lp, int32_t scaling, b200pdlp_form** out);
void b200pdlp_form_destroy(b200pdlp_form* f);
/* dims[0..4] = cols, rows, nnz, neq, original cols; scalars[0..2] = |c|_2, |b|_2 (unscaled), max|a_ij| (scaled) */
int b200pdlp_form_dims(const b200pdlp_form* f, int32_t dims[5], double scalars[3]);
/* which = 0 cost, 1 lower, 2 upper, 3 rhs, 4 col_scale, 5 row_scale; returns count written */
int b200pdlp_form_get_vector(const b200pdlp_form* f, int32_t which, double* dst, int32_t cap);
int b200pdlp_form_get_csc(const b200pdlp_form* f, int32_t* start, int32_t* index, double* value);
/* row-major copy (the reference's csc2csr, cupdlp_utils.c:1222-1254): rowptr[rows+1], col[nnz], val[nnz] */
int b200pdlp_form_get_csr(b200pdlp_form* f, int32_t* rowptr, int32_t* col, double* val);
/* row_new_idx[m], row_class[m] by ORIGINAL row (EQ=0, LEQ=1, GEQ=2, BOUND=3) */
int b200pdlp_form_get_row_map(const b200pdlp_form* f, int32_t* row_new_idx, int32_t* row_class);

/* HiPDLP mode (solver=hipdlp; SURVEY.md 8(a) a20 / 8(f) rank 2), the host prologue (the device prologue's twin): PDLPSolver::preprocessLp
 * (hipdlp/pdhg.cc:152-358) + Scaling::scaleProblem (hipdlp/scaling.cc; scaling_mode bits 1 Ruiz, 4 Pock-Chambolle, 2 L2 =
 * HighsOptions::pdlp_scaling_mode, ruiz_iterations = pdlp_ruiz_iterations).  The form answers the b200pdlp_form_* getters;
 * rows carry an upper bound too: b200pdlp_form_get_vector(which = 6).  row_class uses 4 for FREE rows. */
int b200pdlp_hipdlp_form_create(const b200pdlp_lp* lp, int32_t scaling_mode, int32_t ruiz_iterations, b200pdlp_form** out);
/* The HiPDLP solve on one GPU: what a shim replacing pdlp/HiPdlpWrapper.cpp (solveLpHiPdlp, :26-141) forwards to.
 * Parameters are the HighsOptions the reference's setup() reads (hipdlp/pdhg.cc:1783-1874).  term_code is B200PDLP_OPTIMAL or
 * B200PDLP_TIMELIMIT_OR_ITERLIMIT (term_iterate = 2 when it was the time limit); like the reference, a run that does not
 * converge returns x = y = 0 (the iterate is copied out only on convergence, pdhg.cc:784-899).
 * Tree mode on one GPU (the standard form's max(n, m) > ordered_max) runs the prologue, the initial point and the postsolve
 * on the device by default (device_prep.cu; the same bits as the host prologue, tests/test_gpu_hipdlp_device_prep.py); ordered
 * mode, device_prep = -1 or B200PDLP_DEVICE_PREP=0 take the host prologue (host_prep_hipdlp.cpp).
 * STATUS: runs on hardware; tests/test_gpu_hipdlp.py (bit-exact against the oracle), tests/test_gpu_dropin.py (through
 * the shim), bench.py --solver hipdlp. */
typedef struct {
  double tolerance;           /* pdlp_optimality_tolerance, or kkt_tolerance when set */
  int32_t iter_limit;         /* pdlp_iteration_limit */
  int32_t scaling_mode;       /* pdlp_scaling_mode: bits 1 Ruiz, 2 L2, 4 Pock-Chambolle (default 5); 0 when scaling is off */
  int32_t ruiz_iterations;    /* pdlp_ruiz_iterations (default 10) */
  int32_t step_size_strategy; /* pdlp_step_size_strategy: 0 fixed primal weight, anything else PID */
  double time_limit;          /* seconds; < 0 or inf = none */
  int32_t ordered_max;        /* as in b200pdlp_params: checks add in the reference's order up to this size */
  int32_t device;             /* CUDA device ordinal; -1 = current */
  int32_t log_level;
  int32_t device_prep;        /* 0 = device prologue where it applies (tree mode; one GPU or shards), -1 = always the host prologue */
  int32_t reserved[2];
} b200pdlp_hipdlp_params;
void b200pdlp_hipdlp_default_params(b200pdlp_hipdlp_params* p);
int b200pdlp_solve_hipdlp(const b200pdlp_lp* lp, const b200pdlp_hipdlp_params* params, b200pdlp_result* out);
/* Solve `count` independent LPs in the HiPDLP mode on one GPU in one call.  Every member must be an ordered-mode problem of
 * `params` under HiPDLP's classification (standard form max(n, m) <= ordered_max, a slack column for every ranged and free
 * row, rows bounded by +-infinity only); each returns exactly what b200pdlp_solve_hipdlp(lps[i], params) returns: term_code,
 * term_iterate, iters, passes, restarts, the residual scalars, the form dimensions and all four vectors, bit for bit.
 * All members share `params` (tolerance, limits, scaling, step-size strategy); `device` selects the GPU; `device_prep` is
 * ignored (ordered mode always takes the host prologue); log_level prints nothing per block.  One CTA solves one member;
 * the members' host prologues and postsolves run on host threads.  The time limit counts from the start of the batch's
 * loop.  These fields are batch-wide, the same in every outs[i]: setup_seconds, solve_seconds, loop_device_ms,
 * iter_device_ms and kernel_launches (= the batch's rounds, one launch each; a round is one block of 40 steps).
 * Returns B200PDLP_ERR_ARG before any device work for count < 0, NULL arrays, a member that the checks of
 * b200pdlp_solve_hipdlp reject, ordered_max < 0, or a member whose standard form exceeds ordered_max; b200pdlp_last_error()
 * names the member's index, and no result is written.  count == 0: B200PDLP_OK.  No device: B200PDLP_ERR_CUDA.  The whole
 * batch must fit in device memory (B200PDLP_ERR_ALLOC otherwise).
 * STATUS: runs on hardware; tests/test_gpu_hipdlp_batch.py (byte equality with b200pdlp_solve_hipdlp and with the HiPDLP
 * oracle), tools/batch_bench.py --solver hipdlp. */
int b200pdlp_solve_hipdlp_batch(int32_t count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params* params,
                                b200pdlp_result* outs /* [count], caller-allocated like b200pdlp_result */);
/* b200pdlp_solve_hipdlp_batch for members of any size up to a cap, in any order (host arrays).  A member whose standard form
 * (HiPDLP's classification) has max(n, m) <= ordered_max is an ordered member and returns exactly what
 * b200pdlp_solve_hipdlp_batch returns for it; every other member is a tree member and returns exactly what
 * b200pdlp_solve_hipdlp(lps[i], params) returns for it alone: term_code, term_iterate, iters, passes, restarts, the residual
 * scalars, the form dimensions and all four vectors, bit for bit.  ordered_max < 0 makes every member a tree member.  With
 * trace storage (trace, trace_cap) every member writes the single solve's B200PDLP_HIP_TRACE_COLS rows.  Batch-wide fields
 * as in b200pdlp_solve_hipdlp_batch (kernel_launches = the rounds).  One CTA solves an ordered member; one thread-block
 * cluster of C CTAs (C in {1, 2, 4, 8}, the largest with which every tree member is resident at once, otherwise 1) solves a
 * tree member; a round is one upload, up to two launches and one read-back.  The environment variable
 * B200PDLP_BATCH_CLUSTER=1|2|4|8 forces C for tests and benchmarks; it changes no result.  B200PDLP_TIMING=1 prints the
 * laps and the tree-member count with C.
 * Returns B200PDLP_ERR_ARG before any device work, naming the lowest failing member, for count < 0, NULL arrays, a member
 * that the checks of b200pdlp_solve_hipdlp reject, and a tree member whose standard form exceeds max(n, m) = 262144 (solve
 * it with b200pdlp_solve_hipdlp); no result is written.  count == 0: B200PDLP_OK.  No device: B200PDLP_ERR_CUDA.  The whole
 * batch must fit in device memory (B200PDLP_ERR_ALLOC otherwise).
 * STATUS: runs on hardware; tests/test_gpu_hipdlp_batch_mixed.py (byte equality with b200pdlp_solve_hipdlp and with
 * b200pdlp_solve_hipdlp_batch), tools/hipdlp_batch_mixed_bench.py. */
int b200pdlp_solve_hipdlp_batch_mixed(int32_t count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params* params,
                                      b200pdlp_result* outs /* [count], caller-allocated like b200pdlp_result */);
/* b200pdlp_solve_hipdlp_batch for LPs that are already in GPU memory.  `lps` and `outs` are host arrays of the usual structs,
 * but every array pointer inside them is device (or managed) memory of params->device (< 0: the current device): the LP's
 * eight arrays and the four result vectors.  num_col, num_row, sense and offset are host scalars.  Each member returns exactly
 * what b200pdlp_solve_hipdlp_batch returns for it with the same arrays on the host (and so what b200pdlp_solve_hipdlp returns
 * for it alone): term_code, term_iterate, iters, passes, restarts, the residual scalars, the form dimensions and the four
 * vectors, bit for bit.  Batch-wide fields as in b200pdlp_solve_hipdlp_batch; setup_seconds covers validation, sizing and
 * the device prologue.  device_prep is ignored.
 * The prologue (formulate_hipdlp, scale_hipdlp, the ordered layouts) and the postsolve run on the device, one CTA per member;
 * the host reads one sizing record and two scalars per member, never an array.  A column whose stored rows repeat or descend
 * is sorted by (row, value) on the device; should one row of a column hold both +0.0 and -0.0, -0.0 goes first (std::sort
 * leaves that order unspecified; either order gives the same sums).  The call returns once the outputs are complete on the
 * device; it never writes an input array.  The caller must have finished writing the inputs before the call (the library
 * uses a stream of its own).
 * Returns B200PDLP_ERR_ARG before any device work for count < 0, NULL arrays, ordered_max < 0 or a sense other than +-1;
 * then, naming the member and the field, for a pointer that is not device memory of the device; then, before any solve
 * work and naming the lowest failing member, for what b200pdlp_solve_hipdlp's checks reject in the arrays (a_start[0] != 0,
 * a decreasing a_start, an a_index outside [0, num_row)) and for a standard form under HiPDLP's classification larger than
 * ordered_max.  No result field or array is written on an error.  count == 0: B200PDLP_OK.  No device: B200PDLP_ERR_CUDA.
 * The whole batch must fit in device memory (B200PDLP_ERR_ALLOC otherwise).
 * STATUS: runs on hardware; tests/test_gpu_hipdlp_batch_device.py (byte equality with b200pdlp_solve_hipdlp_batch),
 * tools/batch_device_bench.py --solver hipdlp. */
int b200pdlp_solve_hipdlp_batch_device(int32_t count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params* params,
                                       b200pdlp_result* outs /* [count]; vectors in device memory */);
/* b200pdlp_solve_hipdlp_batch_mixed for LPs that are already in GPU memory.  Pointers follow
 * b200pdlp_solve_hipdlp_batch_device's rules: the LP's eight arrays and the four result vectors are device (or managed)
 * memory of params->device (< 0: the current device); num_col, num_row, sense and offset are host scalars; the trace storage
 * (trace, trace_cap) stays in host memory.  Members are classified as in b200pdlp_solve_hipdlp_batch_mixed (ordered:
 * max(n, m) <= ordered_max under HiPDLP's classification; every other member a tree member up to max(n, m) = 262144;
 * ordered_max < 0 makes every member a tree member) and may come in any order.  Each member returns exactly what
 * b200pdlp_solve_hipdlp_batch_mixed returns for it from the same arrays on the host -- a tree member what
 * b200pdlp_solve_hipdlp returns for it alone, an ordered member what b200pdlp_solve_hipdlp_batch returns: term_code,
 * term_iterate, iters, passes, restarts, the residual scalars, the form dimensions, the four vectors and the trace rows, bit
 * for bit.  Batch-wide fields as in b200pdlp_solve_hipdlp_batch_mixed; setup_seconds covers validation, sizing and the
 * device prologue.  device_prep is ignored.  B200PDLP_BATCH_CLUSTER works as there and changes no result.
 * Every member's prologue and postsolve run on the device, one CTA per member: an ordered member's as in
 * b200pdlp_solve_hipdlp_batch_device; a tree member's builds formulate_hipdlp, scale_hipdlp and the tree-mode layouts (rows
 * and columns sorted by length in windows, long rows cut into segments) and packs the vectors in device order.  The host
 * reads fixed-size records per member, never an array.  The call never writes an input, uses a stream of its own and
 * returns once the outputs are complete.  B200PDLP_TIMING=1 prints the laps (validation + sizing, orderings + plans,
 * prologue, rounds, postsolve) and the tree-member count with C.
 * Returns B200PDLP_ERR_ARG, with nothing written, in b200pdlp_solve_hipdlp_batch_device's order: before any device work for
 * count < 0, NULL arrays or a sense other than +-1; then, naming the member and the field, for a pointer that is not device
 * memory of the device; then, naming the lowest failing member, for a malformed a_start or a_index and for a tree member
 * whose standard form exceeds max(n, m) = 262144 (solve it with b200pdlp_solve_hipdlp).  count == 0: B200PDLP_OK.  No
 * device: B200PDLP_ERR_CUDA.  The whole batch must fit in device memory (B200PDLP_ERR_ALLOC otherwise).
 * STATUS: runs on hardware; tests/test_gpu_hipdlp_batch_mixed_device.py (byte equality with
 * b200pdlp_solve_hipdlp_batch_mixed on host copies and with b200pdlp_solve_hipdlp), tools/hipdlp_batch_mixed_device_bench.py. */
int b200pdlp_solve_hipdlp_batch_mixed_device(int32_t count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params* params,
                                             b200pdlp_result* outs /* [count]; vectors in device memory */);
/* b200pdlp_solve_hipdlp for an LP that is already in GPU memory, at any size: b200pdlp_solve_device's pointer rules, bits,
 * routes and errors, with HiPDLP's classification (+-infinity row bounds, FREE rows with a slack column).  Tree mode reads
 * the LP in place through the HiPDLP device prologue (device_prep = -1 and B200PDLP_DEVICE_PREP=0 are ignored, as above); ordered mode
 * is b200pdlp_solve_hipdlp_batch_mixed_device with this one LP, whose trace rows are b200pdlp_solve_hipdlp's and whose
 * setup_seconds, solve_seconds, loop_device_ms, iter_device_ms and kernel_launches are the batch's.
 * STATUS: runs on hardware; tests/test_gpu_solve_device.py (byte equality with b200pdlp_solve_hipdlp on host copies),
 * tools/solve_device_bench.py. */
int b200pdlp_solve_hipdlp_device(const b200pdlp_lp* lp, const b200pdlp_hipdlp_params* params,
                                 b200pdlp_result* out /* device vectors */);
/* debug (tests): the tree-mode device prologue of b200pdlp_solve_hipdlp_batch_mixed_device on host LPs (uploaded first),
 * every member treated as a tree member, against formulate_hipdlp + scale_hipdlp(scaling_mode, ruiz_iterations) +
 * build_layout(ordered_max = -1), then the device postsolve of a fixed pseudo-random iterate against hip_host_postsolve.
 * report[count][31]: mismatch counts of dims; cost, lower, upper, rhs, row_upper, col_scale, row_scale (device order);
 * rperm, cperm; slices, col, val of A and of A'; segs, long_rows, lcol, lval of A and of A'; |c|, |b|; the scaled flag;
 * col_value, col_dual, row_value, row_dual (-1: not comparable).  B200PDLP_ERR_ARG for a malformed LP or one past
 * max(n, m) = 262144. */
int b200pdlp_debug_hipdlp_tree_prep_compare(int32_t count, const b200pdlp_lp* lps, int32_t scaling_mode,
                                            int32_t ruiz_iterations, double* report);
/* The HiPDLP solve on `ngpus` devices of THIS process (devices[g] or, if NULL, ordinals 0..ngpus-1; a device may repeat,
 * which gives logical shards on one device): the prologue, then each rank computes contiguous blocks of the one-GPU device
 * rows and columns, one host thread per rank, peer memory, no NCCL.  device_prep is honoured as on one GPU: 0 runs the
 * device prologue where it applies (tree mode, non-empty matrix) once per distinct device, which builds every rank's blocks
 * there and leaves the postsolve to rank 0's device; -1 (or B200PDLP_DEVICE_PREP=0) runs the host prologue once.  Either
 * way the result has the same bits as b200pdlp_solve_hipdlp with device_prep = -1 (iterations, termination and all four
 * vectors), for every ngpus.  ngpus <= 1 is b200pdlp_solve_hipdlp; ngpus > 16 or devices without peer access:
 * B200PDLP_ERR_ARG; device is ignored.  What the HiGHS shim uses for solver=hipdlp when B200PDLP_GPUS > 1.
 * STATUS: runs on hardware as logical shards on one H100 with both prologues (tests/test_gpu_hipdlp_shards.py,
 * tests/test_gpu_hipdlp_shard_prep.py, byte equality with one GPU); not yet run on two physical GPUs. */
int b200pdlp_solve_hipdlp_multi(const b200pdlp_lp* lp, const b200pdlp_hipdlp_params* params, b200pdlp_result* out,
                                int32_t ngpus, const int32_t* devices);

/* host-only (no GPU; parity tests): the HOST control of the HiPDLP loop -- step sizes, fixed-point error, convergence test,
 * restart criteria, PID primal weight (HipController, host_prep_hipdlp.cpp; hipdlp/pdhg.cc:494-707,901-927,1944-2050) --
 * replayed over `nblocks` blocks of 40 steps from recorded sums: sums[b][9] = the nine sums of block b's closing check,
 * restart_sums[b][3] = the three fixed-point sums of block b's first step (used when block b follows a restart);
 * out[b][8] = restart decided, primal weight, primal step, dual step, fixed-point error, converged, iterations, halpern_iteration */
int b200pdlp_hipdlp_controller_replay(double norm_cost, double norm_rhs, double op_norm_sq, double tolerance, int32_t strategy,
                                       int32_t nblocks, const double* sums, const double* restart_sums, double* out);

/* PDLPSolver::powerMethod (hipdlp/pdhg.cc:1529-1671): 20 iterations on A A' from the ones vector -> estimate of |A|_2^2 */
int b200pdlp_hipdlp_power_method(const b200pdlp_form* f, double* lambda);

/* ---- HiPDLP kernel-level entry points (parity tests; one GPU) ----------------------------------------------------------
 * A persistent HiPDLP problem, built exactly as b200pdlp_solve_hipdlp builds it: the same prologue choice (ordered_max,
 * device_prep, B200PDLP_DEVICE_PREP) and the same SpMV launch shapes (B200PDLP_TILE*, B200PDLP_SPMV_*; B200PDLP_TIMING=1
 * prints the `SpMV shapes:` line).  b200pdlp_problem_destroy and b200pdlp_problem_dims serve it.  The pdlp entry points on a
 * problem (spmv, primal / dual step, residuals, bench, problem_solve) reject it, and the functions below reject a problem of
 * b200pdlp_problem_create: B200PDLP_ERR_ARG.  Every vector is a host array in standard-form order (the problem's device
 * orderings are applied inside); the problem's iterate buffers serve as scratch.  No device: B200PDLP_ERR_CUDA. */
int b200pdlp_hipdlp_problem_create(const b200pdlp_lp* lp, const b200pdlp_hipdlp_params* params, b200pdlp_problem** out);
/* One Halpern step of the solve (performHalpernPdhgStep, hipdlp/pdhg.cc:961-1018): the primal kernel, A * reflected x fused
 * with the dual update, then A'y.  Weight w = k / (k + 1) with k = halpern_iteration + k_offset.  In/out: x, y (the blended
 * iterate), aty (A'y of the input y on entry, of the new y on return); xn, hslack, yn, ry (written by a major step only, a
 * minor step returns them as given).  Out: rx (the reflected x).  In: xa, ya (the anchors). */
int b200pdlp_hipdlp_step(b200pdlp_problem* p, double primal_step, double dual_step, int32_t halpern_iteration, int32_t k_offset,
                         int32_t is_major, double* x, const double* xa, double* aty, double* y, const double* ya, double* rx,
                         double* xn, double* hslack, double* yn, double* ry);
/* One check of the solve (the fixed-point error, convergence and PID sums) for the iterate (x, y) with anchors (xa, ya);
 * major = 1 checks a major step's x_next = x, y_next = y with its reflected rx, ry and cached slack hslack (otherwise those
 * may be NULL: the sums 0-2 are then 0 and the slacks are the projected dual residual).  out[9] = the nine sums
 * (B200PDLP_HIP_TRACE_COLS columns 1-9; 5 and 6 include the objective offset), in the reference's order in ordered mode,
 * as tree sums otherwise.  Also returns the vectors they were formed from: the slacks sp, sn, ax = A x, aty = A'y, and
 * atdy = A'(y - ry) (zeros when major = 0). */
int b200pdlp_hipdlp_check(b200pdlp_problem* p, int32_t major, const double* x, const double* y, const double* xa,
                          const double* ya, const double* rx, const double* ry, const double* hslack, double out[9],
                          double* sp, double* sn, double* ax, double* aty, double* atdy);
/* The solve's device power method (20 iterations on A A' from the ones vector) -> its estimate of |A|_2^2 */
int b200pdlp_hipdlp_problem_power_method(b200pdlp_problem* p, double* lambda);

/* host-only (no GPU): build the device layout of rank `rank` of `world` exactly as b200pdlp_problem_create does
 * (row block, length-sorted device orderings, sliced ELL of A_g and A_g', long-row segments, segmented column
 * positions, the A_g' output map) and evaluate it on the host in the kernels' traversal order.
 * x[n], y[m] in standard-form order; ax[m]: rows [r0,r1) receive A_g x (others untouched); aty[n] = A_g' y_g.
 * stats: [0] r0 [1] r1 [2] ordered mode [3] A padded slots [4] A long rows [5] A segments [6] A' padded slots
 *        [7] A' long rows [8] A' segments [9] shard_len [10] seg_len [11] layout build time, ms */
int b200pdlp_form_layout_eval(b200pdlp_form* f, int32_t rank, int32_t world, int32_t ordered_max, const double* x,
                              const double* y, double* ax, double* aty, double stats[12]);

/* host-only (no GPU): rank `rank` of `world` of b200pdlp_solve_hipdlp_multi -- its block of the one-GPU device rows and
 * of the one-GPU device columns, A_g and A_g' built as the solve builds them -- evaluated on the host in the kernels'
 * traversal order.  f from b200pdlp_hipdlp_form_create.  x[n], y[m] full, in standard-form order; ax[m] receives the
 * rank's rows of A x, aty[n] the rank's columns of A'y, both in standard-form order (other entries untouched).
 * stats: [0] R_g [1] R_g+1 (device rows) [2] C_g [3] C_g+1 (device columns) [4] ordered mode [5] A_g long rows
 *        [6] A_g' long rows */
int b200pdlp_hipdlp_shard_layout_eval(b200pdlp_form* f, int32_t rank, int32_t world, int32_t ordered_max, const double* x,
                                      const double* y, double* ax, double* aty, double stats[7]);

/* host-only helper (no GPU): nnz-balanced contiguous row partition of the
 * formulated LP; bounds[world+1] receives the row offsets (SURVEY.md 8(e)) */
int b200pdlp_partition_rows(const b200pdlp_lp* lp, int32_t world, int32_t* bounds);

/* Test entry point (needs a GPU): run the device-resident prologue (formulate + scale + row index + orderings +
 * sliced-ELL layouts as kernels, highs_b200/csrc/device_prep.cu) and its host twin (host_prep.cpp) on the same LP and
 * compare them array by array, bit for bit.  report[k] = number of mismatching entries:
 *  0-3 n, m, nnz, neq   4 cbeg 5 cidx 6 cval 7 cost 8 lower 9 upper 10 col_scale 11 rhs 12 row_scale (standard-form order)
 *  13 rptr 14 rpos (row-major index)  15 row_new_idx 16 row_class  17 row ordering 18 column ordering
 *  19-21 A: slice descriptors (-1: sizes differ), col, val   22-24 the same for A'   25, 26 long-row arrays of A, A'
 *  27 max|a_ij|  28, 29 relative error of |c|_2, |b|_2 (tree sums vs sequential)  30 vectors in device order
 *  31 (info) 1 if every column is stored with ascending rows */
int b200pdlp_debug_prep_compare(const b200pdlp_lp* lp, int32_t scaling, double report[32]);
/* The same for the HiPDLP mode: its device prologue against formulate_hipdlp + scale_hipdlp + build_layout (ordered_max = -1).
 * report[0..31] as above, except 28, 29: 1 if |c|_2, |b|_2 differ in any bit (both are sums in index order here), and
 *  32 row_upper (standard-form order)  33 row_upper in device order
 *  34 row pointer of the row-major copy of the caller's matrix  35 its column ids + values (a row's entries in column order)
 *  36 1 if the device and the host disagree on whether any scaling pass ran   37-39 unused (0) */
int b200pdlp_debug_prep_compare_hipdlp(const b200pdlp_lp* lp, int32_t scaling_mode, int32_t ruiz_iterations, double report[40]);
/* The device prologue and postsolve of b200pdlp_solve_batch_device (highs_b200/csrc/batch_prep.cu) against their host twins:
 * the `count` host LPs are uploaded as they are, prepared on the device (cold start, no ordered_max limit) and compared with
 * formulate + scale + build_layout + host_start_point; then a fixed pseudo-random iterate is postsolved on both sides.
 * report[27 * i + k] = mismatching entries (bit for bit) of member i:  0 n, m, nnz, neq (-1 everywhere else if they differ)
 *  1 cost 2 lower 3 upper 4 rhs 5 col_scale 6 row_scale  7 row_new_idx 8 row_class  9-11 A: slice descriptors (-1 for the
 *  rest if they differ), col, val  12-14 the same for A'  15 x0 16 y0 17 xsum  18 |c|_2 19 |b|_2 20 max|a_ij|  21, 22 the
 *  scaled |c|^2, |b|^2 that set beta  23 col_value 24 col_dual 25 row_value 26 row_dual */
int b200pdlp_debug_batch_prep_compare(int32_t count, const b200pdlp_lp* lps, int32_t scaling, double* report);
/* The device prologue and postsolve of b200pdlp_solve_hipdlp_batch_device (batch_prep.cu hip_batch_*_kernel) against their
 * host twins: the `count` host LPs are uploaded as they are, prepared on the device (no ordered_max limit) and compared with
 * formulate_hipdlp + scale_hipdlp + build_layout; then a fixed pseudo-random iterate (x, y and the slacks sp, sn of a member
 * converged at iteration 0) is postsolved on both sides (hip_host_postsolve).
 * report[24 * i + k] = mismatching entries (bit for bit) of member i:  0 n, m, nnz, neq (-1 everywhere else if they differ)
 *  1 cost 2 lower 3 upper 4 rhs 5 row_upper 6 col_scale 7 row_scale  8 row_new_idx 9 row_class  10-12 A: slice descriptors
 *  (-1 for the rest if they differ), col, val  13-15 the same for A'  16 |c|_2 17 |b|_2 of the unscaled form  18 1 if the
 *  device batch and scale_hipdlp disagree on whether the form is scaled  19 entries of build_layout's column and row orderings
 *  that are not the identity the batch assumes  20 col_value 21 col_dual 22 row_value 23 row_dual */
int b200pdlp_debug_hipdlp_batch_prep_compare(int32_t count, const b200pdlp_lp* lps, int32_t scaling_mode, int32_t ruiz_iterations,
                                             double* report);
/* The device prologue of b200pdlp_solve_hipdlp_multi (block mode, all `world` ranks on the current device, 2 <= world <= 16)
 * against formulate_hipdlp + scale_hipdlp + plan_hipdlp_shards (ordered_max = -1) + build_hipdlp_shard.  report[8 + 9 world]
 * = mismatch counts:  0 n, m, nnz, neq (nothing else is compared if they differ)  1 vectors in device order (cost, lower,
 *  upper, col_scale, rhs, row_scale)  2 row_upper in device order  3, 4 1 if |c|_2, |b|_2 differ in any bit  5 1 if the two
 *  disagree on whether any scaling pass ran  6 row and column orderings  7 unused (0);  rank g at 8 + 9 g:  +0 its block
 *  bounds (rows and columns)  +1..+4 A_g: slice descriptors (-1: sizes differ), col, val, long-row arrays  +5..+8 the same for A_g' */
int b200pdlp_debug_hipdlp_shard_prep_compare(const b200pdlp_lp* lp, int32_t scaling_mode, int32_t ruiz_iterations, int32_t world,
                                             double* report);

/* The engine keeps the device blocks of finished solves in a process-wide cache (a solve allocates ~60 buffers; cudaMalloc /
 * cudaFree would cost more than the prologue).  This returns them to the driver.  B200PDLP_CACHE_MB caps the cache. */
void b200pdlp_release_cache(void);

/* ---- post-solve KKT assessment (SURVEY.md 8(a) a21 / 8(f) rank 4) -------------------------------------------------
 * What Highs::run() does with the HighsSolution after solveLpCupdlp returns: lpKktCheck -> getKktFailures
 * (/root/reference/highs/lp_data/HighsSolution.cpp:1043-1327, :73-495): A x and A'y with double-double accumulation,
 * bound / sign violations, absolute and relative measures (relative to 1 + |active bounds|_inf, 1 + |costs with ~0 dual|_inf),
 * residual errors |A x - row_value|, |A'y - c + col_dual|, complementarity, P-D objective error, and the status rules for
 * a solution without a basis.  b200pdlp_kkt_check runs on the GPU (no CPU fallback); b200pdlp_kkt_check_host is its host
 * twin over the same per-variable arithmetic (highs_b200/csrc/kkt_logic.hpp), kept so that the logic is checked against
 * the reference's own lpKktCheck without a GPU.  Tolerances: the five HighsOptions after the kkt_tolerance override. */
typedef struct {
  double primal_feasibility_tolerance, dual_feasibility_tolerance, primal_residual_tolerance, dual_residual_tolerance,
         optimality_tolerance;
} b200pdlp_kkt_tolerances;
typedef struct {   /* HighsInfo fields of the same names (HighsInfo.h:91-131) */
  double objective_function_value, dual_objective_value, primal_dual_objective_error;
  double max_primal_infeasibility, sum_primal_infeasibilities, max_dual_infeasibility, sum_dual_infeasibilities;
  double max_relative_primal_infeasibility, max_relative_dual_infeasibility;
  double max_primal_residual_error, max_dual_residual_error, max_relative_primal_residual_error, max_relative_dual_residual_error;
  double max_complementarity_violation;
  double norm_bounds, norm_costs;   /* getKktFailures' highs_norm_bounds / highs_norm_costs */
  int32_t num_primal_infeasibilities, num_dual_infeasibilities, num_relative_primal_infeasibilities, num_relative_dual_infeasibilities;
  int32_t num_primal_residual_errors, num_dual_residual_errors, num_relative_primal_residual_errors, num_relative_dual_residual_errors;
  int32_t num_complementarity_violations;
  int32_t primal_solution_status, dual_solution_status;   /* kSolutionStatusInfeasible 1 / Feasible 2 */
  int32_t model_status;   /* in: HighsModelStatus code returned by the solver; out: after lpKktCheck's adjustment */
} b200pdlp_kkt_info;
void b200pdlp_kkt_default_tolerances(b200pdlp_kkt_tolerances* t, double kkt_tolerance /* <= 0: the default 1e-7 */);
int b200pdlp_kkt_check(const b200pdlp_lp* lp, const double* col_value, const double* col_dual, const double* row_value,
                       const double* row_dual, const b200pdlp_kkt_tolerances* tol, b200pdlp_kkt_info* inout);
int b200pdlp_kkt_check_host(const b200pdlp_lp* lp, const double* col_value, const double* col_dual, const double* row_value,
                            const double* row_dual, const b200pdlp_kkt_tolerances* tol, b200pdlp_kkt_info* inout);

/* The four vectors of a HighsSolution, original LP space, HiGHS signs (what b200pdlp_result returns) */
typedef struct {
  const double* col_value;   /* [num_col] */
  const double* col_dual;    /* [num_col] */
  const double* row_value;   /* [num_row] */
  const double* row_dual;    /* [num_row] */
} b200pdlp_solution;

/* The KKT assessment of `count` LP solutions in one call on one GPU (device < 0: the current device), one CTA per member:
 * the output side of the batch solves.  inout[i].model_status is read (the HighsModelStatus code from the solver, as for
 * b200pdlp_kkt_check); every other field is written.  `tol` is shared by all members.  Every member's b200pdlp_kkt_info
 * equals what b200pdlp_kkt_check_host returns for it alone, field for field and bit for bit, except that a NaN may have
 * another bit pattern.  There is no size limit: a large member only takes longer.
 * b200pdlp_kkt_check_batch takes host arrays and uploads the whole batch in one copy; b200pdlp_kkt_check_batch_device
 * requires every array pointer in lps[i] and sols[i] to be device (or managed) memory of the device, so the results of
 * b200pdlp_solve_batch_device and b200pdlp_solve_hipdlp_batch_device can be passed as they are (num_col, num_row, sense and
 * offset stay host scalars).  Neither call writes an input.  The caller must have finished writing device inputs before the
 * call (the library uses a stream of its own).
 * Errors, with nothing written to inout: B200PDLP_ERR_ARG before any device work for count < 0, NULL lps / sols / tol /
 * inout, a member with num_col < 0 or num_row < 0, or a NULL array whose length is positive, naming the member (count == 0:
 * B200PDLP_OK; no device: B200PDLP_ERR_CUDA); _device only: a pointer that is not device memory of the device, naming the
 * member and the field; then, naming the lowest failing member, a_start[0] != 0, a decreasing a_start or an a_index outside
 * [0, num_row) (the host variant checks these on the host before any device lookup); B200PDLP_ERR_ALLOC if the batch's
 * workspace (about 4 (m + 1) + 8 nnz + 8 (n + m) bytes per member, and the uploaded arrays for the host variant) does not fit.
 * STATUS: runs on hardware; tests/test_gpu_kkt_batch.py (bit equality with b200pdlp_kkt_check_host for every member),
 * tools/kkt_batch_bench.py. */
int b200pdlp_kkt_check_batch(int32_t count, const b200pdlp_lp* lps, const b200pdlp_solution* sols,
                             const b200pdlp_kkt_tolerances* tol, int32_t device, b200pdlp_kkt_info* inout);
int b200pdlp_kkt_check_batch_device(int32_t count, const b200pdlp_lp* lps, const b200pdlp_solution* sols,
                                    const b200pdlp_kkt_tolerances* tol, int32_t device, b200pdlp_kkt_info* inout);

/* Page-lock / unlock caller memory (cudaHostRegister) so that the copies of b200pdlp_solve run at PCIe speed; optional
 * (pageable buffers work, staged by the driver).  A host application that keeps its HighsLp / HighsSolution vectors for
 * many solves registers them once. */
int b200pdlp_host_register(void* ptr, size_t bytes);
int b200pdlp_host_unregister(void* ptr);

const char* b200pdlp_last_error(void);
int b200pdlp_version(void);
int b200pdlp_device_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200PDLP_H_ */
