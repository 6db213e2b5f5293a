// highs_b200/csrc/batch_kernels.hpp -- the batched ordered-mode solve (b200pdlp_solve_batch): one CTA per LP.
#pragma once
#include "kernels.cuh"

namespace b200 {

// One member of a batch on the device: its ordered-mode sliced-ELL layouts (identity orderings, no long rows) and its
// vectors, all inside the batch's pooled buffers.
struct BatchMember {
  int n, m, neq;
  const int4* a_slices;  const int* a_col;  const double* a_val;    // A  (m rows)
  const int4* at_slices; const int* at_col; const double* at_val;   // A' (n rows)
  const double *cost, *lower, *upper, *colscale, *rhs, *rowscale;
  double *x0, *x1, *aty0, *aty1, *xsum, *xavg, *atyavg, *xlr;      // n-vectors
  double *y0, *y1, *ax0, *ax1, *ysum, *yavg, *axavg, *ylr;         // m-vectors
};

// Sums a check leaves in BatchCtl::outs (indices 0..31 are those of the one-problem ordered check in engine.cu run_check)
//   0..13   column sweep A, 7 per iterate (current, average)     14..19  row sweep A, 3 per iterate
//   24..29  column sweep B, 3 per iterate                         30..31  row sweep B, 1 per iterate
//   32 |xbar - x_lr|^2  33 |x - x_lr|^2  34 |ybar - y_lr|^2  35 |y - y_lr|^2  (what a restart to either iterate needs)
//   36 the power method's estimate of |A|_2^2 (round 0 of a fixed-step solve)
constexpr int kBatchOuts = 40;
constexpr int kBatchDxAvg = 32, kBatchDxCur = 33, kBatchDyAvg = 34, kBatchDyCur = 35, kBatchLambda = 36;

// Per member, written by the host before a round and read back after it
struct BatchCtl {
  int active;        // 0: finished (its CTA returns at once)
  int first;         // 1: round 0 -- [power method,] A x0, A'y0, then the iteration-0 check
  int fixed_step;    // round 0 runs the power method (adaptive_step = 0)
  int no_check;      // iter_limit <= 0: round 0 prepares the iterate and checks nothing
  int restart;       // restart decided at the last check, applied first thing in this round: 0 none, 1 average, 2 current
  int checked;      // out: 1 the round ended with a check (outs valid); 0 the step-rule power tables ran out first
  int pad[2];
  double outs[kBatchOuts];
};

// One round for every active member: blockIdx.x = member
void launch_batch_round(cudaStream_t s, int count, const BatchMember* members, PdhgState* states, BatchCtl* ctls);

}  // namespace b200
