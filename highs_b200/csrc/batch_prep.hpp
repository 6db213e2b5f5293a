// highs_b200/csrc/batch_prep.hpp -- the device prologue and postsolve of b200pdlp_solve_batch_device and
// b200pdlp_solve_hipdlp_batch_device: one CTA per member.
#pragma once
#include "kernels.cuh"

namespace b200 {

// One member of a device-resident batch, filled by the host.  The LP arrays (and the warm vectors) are the caller's device
// memory and are only read.  Every other pointer lies in the batch's pools.
struct BatchPrep {
  // ---- the caller's LP (num_col, num_row, sense are host scalars copied here)
  int n0, m;
  double sense;
  const int* a_start; const int* a_index; const double* a_value;
  const double *col_cost, *col_lower, *col_upper, *row_lower, *row_upper;
  const double *warm_x, *warm_rv, *warm_rd;   // nullptr: cold start
  // ---- scratch of the sizing kernel, kept for the prologue and the postsolve
  int* row_class;     // [m] RowClass (formulate's +-1e20 rule)
  int* row_new_idx;   // [m] the row's standard-form index
  int* slack;         // [m] BOUND row: its slack column's index among the slacks; else -1
  int* rptr;          // [m + 1] row lengths of the standard form (sizing), then the row pointer (prologue)
  // ---- set by the host after sizing (sizes from BatchSize)
  int n, nnz, neq;
  int* cbeg; int* cidx; int* pcol; int* rpos; int* rwork;   // [n + 1], [nnz] x 3, [m]
  double* cval; double* cs; double* cs_next; double* rs;    // [nnz], [n], [n], [m]
  double* vec;                                              // the member's vector block (batch_kernels.hpp BatchVec)
  int4* a_slices; int* a_col; double* a_val;                // the ordered sliced-ELL layouts in the pooled format
  int4* at_slices; int* at_col; double* at_val;             //   batch_round_kernel reads (BatchMember)
  double* rec;                                              // [kPrepRec]
};

// What the sizing kernel reads back per member.  err != 0: a malformed LP, nothing else is valid.
enum BatchPrepErr { kPrepOk = 0, kPrepStart0 = 1, kPrepDecreasing = 2, kPrepIndex = 3, kPrepNull = 4 };
struct BatchSize {
  int err;
  int n, nnz, neq;      // the standard form: num_col + #BOUND, nnz + #BOUND, #EQ + #BOUND
  int pad_a, pad_at;    // padded entries of the ordered sliced-ELL layouts of A (m rows) and A' (n rows), 32 rows a slice
  int pad[2];
};

// What the prologue reads back per member, rec[kPrepRec]: |c|^2, |b|^2 of the unscaled form (index order), amax, and |c|^2,
// |b|^2 of the scaled form (index order: what sets beta)
enum PrepRec { kRecCostSq, kRecRhsSq, kRecAmax, kRecScaledCostSq, kRecScaledRhsSq, kPrepRec };

// Per member, for the postsolve: which iterate to return and where (the caller's device vectors; any NULL: none written)
struct BatchPost {
  double *col_value, *col_dual, *row_value, *row_dual;
  int sel;          // 0 / 1: the current iterate in that half of the double buffers; 2: the average
  int have_check;   // 0: no check ran (iter_limit <= 0): the slacks are zero
};

// What lp_size_kernel reads back for one LP of b200pdlp_solve_device / _hipdlp_device (only lp's LP fields are read)
struct LpSize {
  unsigned err_bits;   // 1 << BatchPrepErr for every rule the LP breaks (0: well-formed, and the fields below are valid)
  int nslack;          // rows with a slack column under the mode's classification (BOUND rows; HiPDLP: BOUND and FREE)
  int nnz;             // a_start[num_col]
  int pad;
};
constexpr int kLpSizeBlocks = 1024;   // lp_size_kernel's grid: about one resident wave of kThreads-thread CTAs on an H100

void launch_batch_size(cudaStream_t s, int count, const BatchPrep* prep, BatchSize* sizes);
void launch_lp_size(cudaStream_t s, const BatchPrep& lp, bool hip, LpSize* out);   // both passes; out: zeroed by the caller
void launch_batch_prep(cudaStream_t s, int count, const BatchPrep* prep, int do_scale);
void launch_batch_post(cudaStream_t s, int count, const BatchPrep* prep, const BatchPost* post);

// ---- the HiPDLP batch (b200pdlp_solve_hipdlp_batch_device): the same BatchPrep per member, read with HiPDLP's meaning --
// row_class under formulate_hipdlp's rule (FREE rows a class of their own), slack[i] >= 0 for BOUND and FREE rows, vec a
// block laid out as HipBatchVec (batch_kernels.hpp), rec[kRecCostSq], rec[kRecRhsSq] = |c|^2, |b|^2 of the unscaled form -- plus these arrays
// (pooled, like BatchPrep's):
struct HipBatchPrep {
  int* optr;       // [m + 1] row pointer of the row-major index of the caller's matrix
  int* opos;       // [nnz0]  its positions into a_index / a_value: per row columns ascending, then stored order
  int* sortcols;   // [num_col] structural columns whose stored rows do not ascend strictly (the prologue's work list)
};

// Per member, for the HiPDLP postsolve: the caller's device vectors (any NULL: none written) and the iterate to return
struct HipBatchPost {
  double *col_value, *col_dual, *row_value, *row_dual;
  int sol;          // -1: not converged (x = y = 0); 0: (x, y) of the iteration-0 check; 1: (xn, yn) after a block
  int pad;
};

// ---- tree members of b200pdlp_solve_hipdlp_batch_mixed_device (batch_tree_prep.cu): the same BatchPrep and HipBatchPrep
// per member (P.a_slices / P.at_slices: the tree layouts' slice descriptors, P.a_col ... : their bodies; P.vec in device
// order), plus the device orders and the long rows of A and A' (build_layout(f, 0, 1, -1): rows sorted by descending length
// in windows, rows longer than kTreeLongRow cut into segments of kNnzPerBlock entries).
constexpr int kTreeLongRow = 512;   // build_layout's long_threshold in tree mode
constexpr int kTreeSortTile = 2048;   // unsorted columns: tiles ranked in shared memory, then merged in HipTreePrep::srt

struct HipSortRec { int row, idx; unsigned long long key; };   // an entry of an unsorted column: (new row, stored index, value key)

// What the orderings-and-plans kernel reads back per member.  err != 0: a layout past 32-bit offsets.
struct HipTreePlan {
  int err;
  int pad_a, pad_at;        // padded body entries of A (m rows) and A' (n rows), before the 32 trailing zeros
  int nseg_a, nlong_a;      // A's long-row segments (= its partial sums) and long rows
  int nseg_at, nlong_at;
  int maxcol;               // the longest structural column of the caller's matrix (the sort scratch)
  long long lcount_a, lcount_at;   // entries of the long-row arrays (rows padded to multiples of 4, + 8)
};

struct HipTreePrep {
  int* rperm; int* rinv;    // [m] device row order: rperm[device row] = form row; rinv its inverse
  int* cperm; int* cinv;    // [n] the same for the columns
  int cap;                  // capacity of each of the four descriptor arrays below (>= any count a plan can reach)
  int4* a_segs; int4* a_long;     // {row, nnz_begin, nnz_end, long_id}, {row, first_seg, nseg, partial_offset}
  int4* at_segs; int4* at_long;
  int* a_lcol; double* a_lval;    // [lcount_a] (zeroed by the host), set after the plan
  int* at_lcol; double* at_lval;
  HipSortRec* srt;          // [2 maxcol] when maxcol > kTreeSortTile, else unused
};

void launch_hip_tree_plan(cudaStream_t s, int count, const BatchPrep* prep, const HipTreePrep* tprep, HipTreePlan* plans);
void launch_hip_tree_prep(cudaStream_t s, int count, const BatchPrep* prep, const HipBatchPrep* hprep, const HipTreePrep* tprep,
                          const HipTreePlan* plans, int scaling_mode, int ruiz_iterations);
void launch_hip_tree_post(cudaStream_t s, int count, const BatchPrep* prep, const HipBatchPrep* hprep, const HipTreePrep* tprep,
                          const HipBatchPost* post, int scaled);

void launch_hip_batch_size(cudaStream_t s, int count, const BatchPrep* prep, BatchSize* sizes);
void launch_hip_batch_prep(cudaStream_t s, int count, const BatchPrep* prep, const HipBatchPrep* hprep, int scaling_mode,
                           int ruiz_iterations);
void launch_hip_batch_post(cudaStream_t s, int count, const BatchPrep* prep, const HipBatchPrep* hprep,
                           const HipBatchPost* post, int scaled);

}  // namespace b200
