// highs_b200/csrc/batch_kernels.cu -- batched ordered-mode PDHG (b200pdlp_solve_batch): one CTA owns one LP.
//
// A launch runs one ROUND for every unfinished member (engine_batch.cu solve_batch drives the rounds):
//   1. the host's decision from the last check: a restart (average -> current when chosen, sums cleared, last-restart point
//      taken) -- or, in round 0, the initial products A x0, A'y0 (after the power method of a fixed-step solve);
//   2. PDHG passes until state.iter == state.stop_iter (K1..K4 of pdhg_kernels.cu, same arithmetic through pdhg_arith.cuh);
//   3. the check: averages, A xbar and A'ybar, the sums of the ordered check (run_check's sweeps A, the ray scales, sweeps B)
//      and the four distances to the last restart point that a restart to either iterate needs.
// A member whose step-rule power tables run out before stop_iter ends its round early without a check (BatchCtl::checked
// = 0); the host refills the tables and the next launch continues its passes.
//
// Bits: every SpMV row is summed in its own entry order over the member's ordered-mode sliced-ELL layout, as
// spmv_sell_kernel does (ordered layouts have no long rows), and every reduction adds its terms in index order in ONE
// thread -- the ordered branch of grid_reduce / step_rule_kernel.  The terms are recomputed from the stored vectors by the
// reducing thread instead of being parked in scratch: the same expression on the same operands, so the same bits, and no
// term memory at all.  The reductions of one phase run on lane 0 of different warps, side by side.
// The transcendentals that must be glibc's (pow of the step rule, log / exp of the restart's beta update) stay on the host.
// No CTA waits on another CTA or on the host, so any number of members runs, resident or not.
#include "batch_kernels.hpp"
#include "pdhg_arith.cuh"

namespace b200 {
namespace {

// row r of a sliced-ELL matrix times `in`, in the row's entry order (the body of spmv_sell_kernel: lane = row, k ascending;
// padding entries add 0 * in[0])
__device__ __forceinline__ double sell_row(const int4* __restrict__ slices, const int* __restrict__ col,
                                           const double* __restrict__ val, int r, const double* __restrict__ in) {
  const int4 d = slices[r >> 5];
  const int* __restrict__ cp = col + d.x + (r & 31);
  const double* __restrict__ vp = val + d.x + (r & 31);
  double s = 0.0;
  for (int k = 0; k < d.y; k++) s += vp[32 * k] * in[cp[32 * k]];
  return s;
}

__device__ __forceinline__ void spmv(const int4* slices, const int* col, const double* val, int rows, const double* in,
                                     double* out) {
  for (int r = threadIdx.x; r < rows; r += kThreads) out[r] = sell_row(slices, col, val, r, in);
}

// |a - b|^2 (b != nullptr) or |a|^2 in index order: diff_norm2_kernel's terms, one thread
__device__ __forceinline__ double seq_norm2(int len, const double* __restrict__ a, const double* __restrict__ b) {
  double s = 0.0;
  for (int i = 0; i < len; i++) {
    const double d = b ? (a[i] + -1.0 * b[i]) : a[i];
    s += d * d;
  }
  return s;
}

// the thread that runs reduction job `w` of a phase: lane 0 of warp w
__device__ __forceinline__ bool job(int w) { return threadIdx.x == 32 * w; }

// PDHG_Power_Method (cupdlp_step.c:71-145) as engine.cu power_method runs it, aty0 / ax0 / ylr as scratch
__device__ double power_method(const BatchMember& M, double* sw) {
  const int n = M.n, m = M.m;
  double* q = M.ylr;
  for (int i = threadIdx.x; i < m; i += kThreads) q[i] = 1.0;
  double lambda = 0.0;
  for (int it = 0; it < 20; it++) {
    __syncthreads();
    spmv(M.at_slices, M.at_col, M.at_val, n, q, M.aty0);
    __syncthreads();
    spmv(M.a_slices, M.a_col, M.a_val, m, M.aty0, M.ax0);
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += kThreads) q[i] = M.ax0[i];
    __syncthreads();
    if (threadIdx.x == 0) sw[0] = 1.0 / sqrt(seq_norm2(m, q, nullptr));
    __syncthreads();
    const double w = sw[0];
    for (int i = threadIdx.x; i < m; i += kThreads) q[i] = q[i] * w;
    __syncthreads();
    spmv(M.at_slices, M.at_col, M.at_val, n, q, M.aty0);
    __syncthreads();
    if (threadIdx.x == 0) sw[1] = seq_norm2(n, M.aty0, nullptr);
    __syncthreads();
    lambda = sw[1];
  }
  for (int i = threadIdx.x; i < m; i += kThreads) q[i] = 0.0;
  return lambda;
}

// engine.cu do_restart's vector work: sums cleared, average -> current (choice 1), last-restart point <- current
__device__ void apply_restart(const BatchMember& M, int cur, int choice) {
  double* x = cur ? M.x1 : M.x0;
  double* aty = cur ? M.aty1 : M.aty0;
  double* y = cur ? M.y1 : M.y0;
  double* ax = cur ? M.ax1 : M.ax0;
  for (int i = threadIdx.x; i < M.n; i += kThreads) {
    M.xsum[i] = 0.0;
    if (choice == 1) { x[i] = M.xavg[i]; aty[i] = M.atyavg[i]; }
    M.xlr[i] = x[i];
  }
  for (int i = threadIdx.x; i < M.m; i += kThreads) {
    M.ysum[i] = 0.0;
    if (choice == 1) { y[i] = M.yavg[i]; ax[i] = M.axavg[i]; }
    M.ylr[i] = y[i];
  }
}

// one PDHG pass: K1 primal step, K2 A x' + dual step, K3 A'y', K4 the three sums in index order + the step rule
__device__ void pass(const BatchMember& M, PdhgState* st, double* red) {
  const int n = M.n, m = M.m, cur = st->cur;
  const double* __restrict__ x = cur ? M.x1 : M.x0;
  double* __restrict__ xn = cur ? M.x0 : M.x1;
  const double* __restrict__ aty = cur ? M.aty1 : M.aty0;
  double* __restrict__ atyn = cur ? M.aty0 : M.aty1;
  const double* __restrict__ y = cur ? M.y1 : M.y0;
  double* __restrict__ yn = cur ? M.y0 : M.y1;
  const double* __restrict__ ax = cur ? M.ax1 : M.ax0;
  double* __restrict__ axn = cur ? M.ax0 : M.ax1;
  const bool pend = st->pending != 0;
  const double w = st->w_pending;
  {
    const double tau = st->tau_try, ntau = -tau;
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const double xc = x[i];
      if (pend) M.xsum[i] = M.xsum[i] + w * xc;
      double o;
      primal_update(xc, M.cost[i], aty[i], M.upper[i], M.lower[i], tau, ntau, o);
      xn[i] = o;
    }
  }
  __syncthreads();
  {
    const double sigma = st->sigma_try;
    for (int r = threadIdx.x; r < m; r += kThreads) {
      const double s = sell_row(M.a_slices, M.a_col, M.a_val, r, xn);
      axn[r] = s;
      const double yc = y[r];
      if (pend) M.ysum[r] = M.ysum[r] + w * yc;
      yn[r] = dual_update(yc, M.rhs[r], s, ax[r], sigma, r >= M.neq);
    }
  }
  __syncthreads();
  spmv(M.at_slices, M.at_col, M.at_val, n, yn, atyn);
  __syncthreads();
  if (job(0)) {
    double s = 0.0;
    for (int i = 0; i < n; i++) { const double d = x[i] - xn[i]; s += d * d; }
    red[0] = s;
  } else if (job(1)) {
    double s = 0.0;
    for (int i = 0; i < m; i++) { const double d = y[i] - yn[i]; s += d * d; }
    red[1] = s;
  } else if (job(2)) {
    double s = 0.0;
    for (int i = 0; i < n; i++) { const double dx = x[i] - xn[i]; const double da = aty[i] - atyn[i]; s += dx * da; }
    red[2] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    st->dx2 = red[0];
    st->dy2 = red[1];
    step_rule(st, red[2]);
  }
  __syncthreads();
}

// the ordered check of engine.cu run_check for the current (t = 0) and the average (t = 1) iterate, plus the restart sums
__device__ void check(const BatchMember& M, PdhgState* st, double* o) {
  const int n = M.n, m = M.m, cur = st->cur;
  const double scale = st->sum_step > 0.0 ? 1.0 / st->sum_step : 1.0;
  const bool pend = st->pending != 0;
  const double w = st->w_pending;
  const double* xc = cur ? M.x1 : M.x0;
  const double* atyc = cur ? M.aty1 : M.aty0;
  const double* yc = cur ? M.y1 : M.y0;
  const double* axc = cur ? M.ax1 : M.ax0;
  // PDHG_Compute_Average_Iterate (engine.cu launch_average)
  for (int i = threadIdx.x; i < n; i += kThreads) {
    double s = M.xsum[i];
    if (pend) { s = s + w * xc[i]; M.xsum[i] = s; }
    M.xavg[i] = s * scale;
  }
  for (int i = threadIdx.x; i < m; i += kThreads) {
    double s = M.ysum[i];
    if (pend) { s = s + w * yc[i]; M.ysum[i] = s; }
    M.yavg[i] = s * scale;
  }
  __syncthreads();
  spmv(M.a_slices, M.a_col, M.a_val, m, M.xavg, M.axavg);
  spmv(M.at_slices, M.at_col, M.at_val, n, M.yavg, M.atyavg);
  __syncthreads();
  if (threadIdx.x == 0) st->pending = 0;
  const int wid = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    if (wid < 2) {   // column sweep A of iterate wid
      const double* x = wid ? M.xavg : xc;
      const double* aty = wid ? M.atyavg : atyc;
      double a[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      for (int i = 0; i < n; i++) {
        const double l = M.lower[i], u = M.upper[i];
        const bool hl = l > -INFINITY, hu = u < INFINITY;
        col_check_a_terms(x[i], aty[i], M.cost[i], hl, hu, hl ? l : 0.0, hu ? u : 0.0, M.colscale[i],
                          [&](int k, double v) { a[k] += v; });
      }
#pragma unroll
      for (int k = 0; k < 7; k++) o[7 * wid + k] = a[k];
    } else if (wid < 4) {   // row sweep A of iterate wid - 2
      const double* y = wid == 3 ? M.yavg : yc;
      const double* ax = wid == 3 ? M.axavg : axc;
      double a[3] = {0.0, 0.0, 0.0};
      for (int i = 0; i < m; i++) {
        row_check_a_terms(y[i], ax[i], M.rhs[i], M.rowscale[i], i >= M.neq, [&](int k, double v) { a[k] += v; });
      }
#pragma unroll
      for (int k = 0; k < 3; k++) o[14 + 3 * (wid - 2) + k] = a[k];
    } else if (wid == 4) {
      o[kBatchDxAvg] = seq_norm2(n, M.xavg, M.xlr);
    } else if (wid == 5) {
      o[kBatchDxCur] = seq_norm2(n, xc, M.xlr);
    } else if (wid == 6) {
      o[kBatchDyAvg] = seq_norm2(m, M.yavg, M.ylr);
    } else {
      o[kBatchDyCur] = seq_norm2(m, yc, M.ylr);
    }
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0 && wid < 4) {
    // the ray scales, in run_check's expression order
    const int t = wid & 1;
    const double* a = o + 7 * t;
    const double* r = o + 14 + 3 * t;
    double dscale = sqrt(r[2] + a[4] + a[5]);
    if (dscale < 1e-8) dscale = 1.0;
    double pscale = sqrt(a[6]);
    if (pscale < 1e-8) pscale = 1.0;
    const double ids = 1 / dscale, ips = 1.0 / pscale;
    if (wid < 2) {   // column sweep B of iterate t
      const double* x = t ? M.xavg : xc;
      const double* aty = t ? M.atyavg : atyc;
      double b[3] = {0.0, 0.0, 0.0};
      for (int i = 0; i < n; i++) {
        const double hl = M.lower[i] > -INFINITY ? 1.0 : 0.0, hu = M.upper[i] < INFINITY ? 1.0 : 0.0;
        col_check_b_terms(x[i], aty[i], M.cost[i], hl, hu, M.colscale[i], ids, ips, [&](int k, double v) { b[k] += v; });
      }
#pragma unroll
      for (int k = 0; k < 3; k++) o[24 + 3 * t + k] = b[k];
    } else {         // row sweep B of iterate t
      const double* ax = t ? M.axavg : axc;
      double b = 0.0;
      for (int i = 0; i < m; i++) b += row_check_b_term(ax[i], ips, M.rowscale[i], i >= M.neq);
      o[30 + t] = b;
    }
  }
  __syncthreads();
}

template <class T>
__device__ __forceinline__ void copy_words(T* dst, const T* src) {
  static_assert(sizeof(T) % 8 == 0, "8-byte words");
  const unsigned long long* s = reinterpret_cast<const unsigned long long*>(src);
  unsigned long long* d = reinterpret_cast<unsigned long long*>(dst);
  for (int i = threadIdx.x; i < (int)(sizeof(T) / 8); i += kThreads) d[i] = s[i];
}

__global__ void __launch_bounds__(kThreads, 3)
batch_round_kernel(const BatchMember* __restrict__ members, PdhgState* __restrict__ states, BatchCtl* __restrict__ ctls) {
  BatchCtl* ctl = ctls + blockIdx.x;
  if (!ctl->active) return;
  __shared__ BatchMember M;
  __shared__ PdhgState st;
  __shared__ double o[kBatchOuts];
  __shared__ double red[4];
  copy_words(&M, members + blockIdx.x);
  copy_words(&st, states + blockIdx.x);
  for (int i = threadIdx.x; i < kBatchOuts; i += kThreads) o[i] = 0.0;
  const int first = ctl->first, restart = ctl->restart, no_check = ctl->no_check;
  __syncthreads();
  if (first) {
    if (ctl->fixed_step) {
      const double lambda = power_method(M, red);
      if (threadIdx.x == 0) o[kBatchLambda] = lambda;
      __syncthreads();
    }
    spmv(M.a_slices, M.a_col, M.a_val, M.m, M.x0, M.ax0);
    spmv(M.at_slices, M.at_col, M.at_val, M.n, M.y0, M.aty0);
  } else if (restart) {
    apply_restart(M, st.cur, restart);
  }
  __syncthreads();
  // passes up to the check iteration, or until the step-rule tables are used up (the host refills them)
  while (st.iter < st.stop_iter && !(st.adaptive && st.step_iter - st.pow_base >= kPowTab)) pass(M, &st, red);
  const bool due = st.iter >= st.stop_iter && !(first && no_check);
  if (due) check(M, &st, o);
  __syncthreads();
  copy_words(states + blockIdx.x, &st);
  for (int i = threadIdx.x; i < kBatchOuts; i += kThreads) ctl->outs[i] = o[i];
  if (threadIdx.x == 0) {
    ctl->checked = due ? 1 : 0;
    ctl->first = 0;
    ctl->restart = 0;
  }
}

// ============================================================================================ HiPDLP batch
// b200pdlp_solve_hipdlp_batch: one round of one member = what solve_hipdlp_on_device (engine_hipdlp.cu) enqueues between two of
// its host decisions, with the same per-element arithmetic (pdhg_arith.cuh):
//   round 0    the power method (n > 0 and m > 0), x = xa = proj_[l,u](0), y = ya = 0, A'y, the iteration-0 check;
//   round k    the restart decided after block k - 1 (anchors and iterates <- (xn, yn), A'y), step 1 (major), the three
//              fixed-point sums of that step when the restart's reference error is due (step 2 overwrites rx, so they
//              cannot wait for the check), steps 2..39 (minor) and 40 (major), the block-end check.
// Every SpMV row is summed in entry order (sell_row over the ordered layout, as spmv_sell_kernel sums it), and every sum of
// a check or of the power method adds its terms in index order in one thread from the same init, as warp_ordered_sum
// does; the reducing thread forms the terms from the stored vectors.  The independent sums of one phase run on lane 0 of
// different warps.

// the sum of term(i), i < len, in index order from init (warp_ordered_sum's order), one thread
template <class Term>
__device__ __forceinline__ double seq_sum(int len, double init, Term term) {
  double s = init;
  for (int i = 0; i < len; i++) s = s + term(i);
  return s;
}

// PDLPSolver::powerMethod (pdhg.cc:1529-1671) as solve_hipdlp_on_device runs it in ordered mode: q = 1; 20 times w = A'q,
// z = A w, z = z / |z|, w' = A'z, lambda = |w'|^2, q = z.  q in dy, z in axp, w in atdy, w' in atyp (all set again later).
__device__ double hip_power_method(const HipBatchMember& M, double* sw) {
  const int n = M.n, m = M.m;
  double* q = M.dy;
  double* z = M.axp;
  for (int i = threadIdx.x; i < m; i += kThreads) q[i] = 1.0;
  double lambda = 0.0;
  for (int it = 0; it < 20; it++) {
    __syncthreads();
    spmv(M.at_slices, M.at_col, M.at_val, n, q, M.atdy);
    __syncthreads();
    spmv(M.a_slices, M.a_col, M.a_val, m, M.atdy, z);
    __syncthreads();
    if (threadIdx.x == 0) sw[0] = seq_sum(m, 0.0, [&](int i) { return z[i] * z[i]; });
    __syncthreads();
    const double nrm = sqrt(sw[0]);   // hip_div_norm_kernel
    for (int i = threadIdx.x; i < m; i += kThreads) z[i] = z[i] / nrm;
    __syncthreads();
    spmv(M.at_slices, M.at_col, M.at_val, n, z, M.atyp);
    __syncthreads();
    if (threadIdx.x == 0) sw[1] = seq_sum(n, 0.0, [&](int i) { return M.atyp[i] * M.atyp[i]; });
    for (int i = threadIdx.x; i < m; i += kThreads) q[i] = z[i];
    __syncthreads();
    lambda = sw[1];
  }
  return lambda;
}

// Halpern step k_offset of the block (hip_step: hip_primal_kernel, A * reflected x with HipDualEpilogue, A'y)
__device__ void hip_batch_step(const HipBatchMember& M, double ps, double ds, int hi, int k_offset, int is_major) {
  const int k = hi + k_offset;
  const double w = (double)k / (k + 1.0);
  for (int i = threadIdx.x; i < M.n; i += kThreads)
    hip_primal_col(i, ps, w, is_major, M.x, M.xa, M.cost, M.aty, M.lower, M.upper, M.rx, M.xn, M.hslack);
  __syncthreads();
  for (int r = threadIdx.x; r < M.m; r += kThreads) {
    const double s = sell_row(M.a_slices, M.a_col, M.a_val, r, M.rx);
    M.y[r] = hip_dual_blend(r, M.y[r], M.ya[r], M.rlo[r], M.rup[r], s, ds, w, is_major, M.yn, M.ry);
  }
  __syncthreads();
  spmv(M.at_slices, M.at_col, M.at_val, M.n, M.y, M.aty);
  __syncthreads();
}

// dy = yn - ry and A'dy: the dual movement of the last major step (hip_diff_kernel, then A')
__device__ void hip_batch_atdy(const HipBatchMember& M) {
  for (int r = threadIdx.x; r < M.m; r += kThreads) M.dy[r] = M.yn[r] - M.ry[r];
  __syncthreads();
  spmv(M.at_slices, M.at_col, M.at_val, M.n, M.dy, M.atdy);
}

// the check arguments of hip_check for (x, y), or with `major` for (xn, yn); thread 0 writes them
__device__ void hip_batch_args(const HipBatchMember& M, int major, HipCheckArgs& a) {
  a.n = M.n; a.m = M.m; a.neq = M.neq; a.scaled = M.scaled; a.offset = M.offset;
  a.x = major ? M.xn : M.x; a.y = major ? M.yn : M.y; a.ax = M.axp; a.aty = M.atyp; a.rx = M.rx; a.ry = M.ry; a.atdy = M.atdy;
  a.xa = M.xa; a.ya = M.ya; a.c = M.cost; a.lo = M.lower; a.up = M.upper; a.rlo = M.rlo;
  a.colscale = M.colscale; a.rowscale = M.rowscale; a.sp = M.sp; a.sn = M.sn;
}

// hip_check: A x and A'y of the checked iterate (and A'dy with `major`), the dual slacks (cached on a major step), then the
// nine sums of hip_check_ordered_kernel into out[0..8] (0..2 stay 0 without `major`); `a` is hip_batch_args(major)
__device__ void hip_batch_check(const HipBatchMember& M, int major, const HipCheckArgs& a, double* __restrict__ out) {
  if (major) hip_batch_atdy(M);
  spmv(M.a_slices, M.a_col, M.a_val, M.m, a.x, M.axp);
  spmv(M.at_slices, M.at_col, M.at_val, M.n, a.y, M.atyp);
  __syncthreads();
  for (int i = threadIdx.x; i < M.n; i += kThreads) {
    double sp, sn;
    hip_dual_slacks(i, major, M.hslack, M.cost, M.atyp, M.lower, M.upper, sp, sn);
    M.sp[i] = sp;
    M.sn[i] = sn;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
    switch (threadIdx.x >> 5) {   // 9 sums on 8 warps: warp 1 adds two m-length sums one after the other
      case 0: out[0] = major ? seq_sum(a.n, 0.0, [&](int i) { return hip_fpe_x_term(a, i); }) : 0.0; break;
      case 1:
        out[1] = major ? seq_sum(a.m, 0.0, [&](int i) { return hip_fpe_y_term(a, i); }) : 0.0;
        out[8] = seq_sum(a.m, 0.0, [&](int i) { return hip_anchor_y_term(a, i); });
        break;
      case 2: out[2] = major ? seq_sum(a.n, 0.0, [&](int i) { return hip_fpe_inter_term(a, i); }) : 0.0; break;
      case 3: out[3] = seq_sum(a.m, 0.0, [&](int i) { return hip_primal_res_term(a, i); }); break;
      case 4: out[4] = seq_sum(a.n, 0.0, [&](int i) { return hip_dual_res_term(a, i); }); break;
      case 5: out[5] = seq_sum(a.n, a.offset, [&](int i) { return hip_pobj_term(a, i); }); break;
      case 6: {
        double v = seq_sum(a.m, a.offset, [&](int i) { return hip_dobj_row_term(a, i); });
        v = seq_sum(a.n, v, [&](int i) { return hip_dobj_lo_term(a, i); });
        out[6] = seq_sum(a.n, v, [&](int i) { return hip_dobj_up_term(a, i); });
        break;
      }
      default: out[7] = seq_sum(a.n, 0.0, [&](int i) { return hip_anchor_x_term(a, i); }); break;
    }
  }
}

__global__ void __launch_bounds__(kThreads, 3)
hip_batch_round_kernel(const HipBatchMember* __restrict__ members, const HipState* __restrict__ states,
                       HipBatchCtl* __restrict__ ctls) {
  HipBatchCtl* ctl = ctls + blockIdx.x;
  if (!ctl->active) return;
  __shared__ HipBatchMember M;
  __shared__ HipCheckArgs args;
  __shared__ double sw[2];
  copy_words(&M, members + blockIdx.x);
  const HipState st = states[blockIdx.x];
  const int first = ctl->first, restart = ctl->restart, fpe = ctl->fpe;
  double* out = ctl->outs;
  __syncthreads();
  if (first) {
    if (M.n > 0 && M.m > 0) {
      const double lambda = hip_power_method(M, sw);
      if (threadIdx.x == 0) out[kHipBatchLambda] = lambda;
    }
    // x = xa = proj_[l,u](0) (hip_init_kernel: upper first, then lower), y = ya = 0, the other iterate vectors 0
    for (int i = threadIdx.x; i < M.n; i += kThreads) {
      double v = 0.0;
      if (v > M.upper[i]) v = M.upper[i];
      if (v < M.lower[i]) v = M.lower[i];
      M.x[i] = v; M.xa[i] = v;
      M.xn[i] = 0.0; M.rx[i] = 0.0; M.hslack[i] = 0.0; M.sp[i] = 0.0; M.sn[i] = 0.0; M.atdy[i] = 0.0;
    }
    for (int r = threadIdx.x; r < M.m; r += kThreads) {
      M.y[r] = 0.0; M.ya[r] = 0.0; M.yn[r] = 0.0; M.ry[r] = 0.0; M.dy[r] = 0.0;
    }
    if (threadIdx.x == 0) hip_batch_args(M, 0, args);
    __syncthreads();
    spmv(M.at_slices, M.at_col, M.at_val, M.n, M.y, M.aty);
    __syncthreads();
    hip_batch_check(M, 0, args, out);
    return;
  }
  if (restart) {   // anchors and iterates <- the PDHG iterate of the last major step (:664-688)
    for (int i = threadIdx.x; i < M.n; i += kThreads) { const double v = M.xn[i]; M.xa[i] = v; M.x[i] = v; }
    for (int r = threadIdx.x; r < M.m; r += kThreads) { const double v = M.yn[r]; M.ya[r] = v; M.y[r] = v; }
    __syncthreads();
    spmv(M.at_slices, M.at_col, M.at_val, M.n, M.y, M.aty);
    __syncthreads();
  }
  if (threadIdx.x == 0) hip_batch_args(M, 1, args);
  hip_batch_step(M, st.primal_step, st.dual_step, st.halpern_iteration, 1, 1);
  if (fpe) {   // the restart's reference fixed-point error is that of the first step after it (:600-608)
    hip_batch_atdy(M);
    __syncthreads();
    if (threadIdx.x == 0) out[kHipBatchFpe] = seq_sum(M.n, 0.0, [&](int i) { return hip_fpe_x_term(args, i); });
    else if (threadIdx.x == 32) out[kHipBatchFpe + 1] = seq_sum(M.m, 0.0, [&](int i) { return hip_fpe_y_term(args, i); });
    else if (threadIdx.x == 64) out[kHipBatchFpe + 2] = seq_sum(M.n, 0.0, [&](int i) { return hip_fpe_inter_term(args, i); });
    __syncthreads();
  }
  for (int k = 2; k <= 39; k++) hip_batch_step(M, st.primal_step, st.dual_step, st.halpern_iteration, k, 0);
  hip_batch_step(M, st.primal_step, st.dual_step, st.halpern_iteration, 40, 1);
  hip_batch_check(M, 1, args, out);
}

}  // namespace

void launch_batch_round(cudaStream_t s, int count, const BatchMember* members, PdhgState* states, BatchCtl* ctls) {
  if (count > 0) batch_round_kernel<<<count, kThreads, 0, s>>>(members, states, ctls);
}

void launch_hip_batch_round(cudaStream_t s, int count, const HipBatchMember* members, const HipState* states,
                            HipBatchCtl* ctls) {
  if (count > 0) hip_batch_round_kernel<<<count, kThreads, 0, s>>>(members, states, ctls);
}

}  // namespace b200
