// highs_b200/csrc/batch_kernels.hpp -- the batched ordered-mode solves (b200pdlp_solve_batch, b200pdlp_solve_hipdlp_batch):
// one CTA per LP.
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

// A member's vectors lie in one block of doubles: its n-vectors, one slot of n doubles each, then its m-vectors, one slot of
// m doubles each.  These slots are the only place the order is written; the host (engine_batch.cu) and the kernels of
// batch_prep.cu address a block through them.  The two halves of each double buffer (x0 / x1, aty0 / aty1, y0 / y1,
// ax0 / ax1) are adjacent, so the half of parity cur is slot k0 + cur.
struct BatchVec {
  enum Col { kCost, kLower, kUpper, kColscale, kX0, kX1, kAty0, kAty1, kXsum, kXavg, kAtyavg, kXlr, kCols };
  enum Row { kRhs, kRowscale, kY0, kY1, kAx0, kAx1, kYsum, kYavg, kAxavg, kYlr, kRows };
  static size_t len(int n, int m) { return (size_t)kCols * n + (size_t)kRows * m; }
  template <class T> __host__ __device__ static T* col(T* v, int n, int k) { return v + k * n; }
  template <class T> __host__ __device__ static T* row(T* v, int n, int m, int k) { return v + kCols * n + k * m; }
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

// ---- the batched HiPDLP solve (b200pdlp_solve_hipdlp_batch): one CTA per LP, one round = one block of 40 Halpern steps

// One member of a HiPDLP batch on the device: its ordered-mode sliced-ELL layouts and its vectors, inside the pooled buffers
struct HipBatchMember {
  int n, m, neq, scaled;
  double offset;
  const int4* a_slices;  const int* a_col;  const double* a_val;    // A  (m rows)
  const int4* at_slices; const int* at_col; const double* at_val;   // A' (n rows)
  const double *cost, *lower, *upper, *colscale, *rlo, *rup, *rowscale;
  double *x, *xa, *xn, *rx, *aty, *hslack, *atyp, *atdy, *sp, *sn;   // n-vectors
  double *y, *ya, *yn, *ry, *axp, *dy;                                // m-vectors
};

// A HiPDLP member's vector block, laid out as BatchVec's
struct HipBatchVec {
  enum Col { kCost, kLower, kUpper, kColscale, kX, kXa, kXn, kRx, kAty, kHslack, kAtyp, kAtdy, kSp, kSn, kCols };
  enum Row { kRlo, kRup, kRowscale, kY, kYa, kYn, kRy, kAxp, kDy, kRows };
  static size_t len(int n, int m) { return (size_t)kCols * n + (size_t)kRows * m; }
  template <class T> __host__ __device__ static T* col(T* v, int n, int k) { return v + k * n; }
  template <class T> __host__ __device__ static T* row(T* v, int n, int m, int k) { return v + kCols * n + k * m; }
};

// Sums a round leaves in HipBatchCtl::outs
//   0..8    the nine sums of the round's closing check (HipController's s[0..8]; 0..2 are 0 in round 0)
//   9..11   the fixed-point sums of the round's first step (HipController::restart_reference), when HipBatchCtl::fpe is set
//   12      the power method's estimate of |A|_2^2 (round 0, when n > 0 and m > 0)
constexpr int kHipBatchOuts = 16;
constexpr int kHipBatchFpe = 9, kHipBatchLambda = 12;

// Per member, written by the host before a round and read back after it
struct HipBatchCtl {
  int active;    // 0: finished (its CTA returns at once)
  int first;     // 1: round 0 -- power method, initial point, A'y, the iteration-0 check
  int restart;   // a restart decided after the last block, applied first thing in this round: anchors and iterates <- (xn, yn)
  int fpe;       // the restart's reference fixed-point error is due: the three sums of this round's first step
  double outs[kHipBatchOuts];
};

// One round for every active member: blockIdx.x = member; states[i] holds the steps and halpern_iteration of the round
void launch_hip_batch_round(cudaStream_t s, int count, const HipBatchMember* members, const HipState* states,
                            HipBatchCtl* ctls);

}  // namespace b200
