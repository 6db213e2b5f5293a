// highs_b200/csrc/batch_prep.hpp -- the device prologue and postsolve of b200pdlp_solve_batch_device: one CTA per member.
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
  double* vec;                                              // the member's vector block (engine.cu batch_vec_len)
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

// What the prologue reads back per member: rec[0..4] = |c|^2, |b|^2 of the unscaled form (index order), amax, and |c|^2,
// |b|^2 of the scaled form (index order: what sets beta)
constexpr int kPrepRec = 5;

// Per member, for the postsolve: which iterate to return and where (the caller's device vectors; any NULL: none written)
struct BatchPost {
  double *col_value, *col_dual, *row_value, *row_dual;
  int sel;          // 0 / 1: the current iterate in that half of the double buffers; 2: the average
  int have_check;   // 0: no check ran (iter_limit <= 0): the slacks are zero
};

void launch_batch_size(cudaStream_t s, int count, const BatchPrep* prep, BatchSize* sizes);
void launch_batch_prep(cudaStream_t s, int count, const BatchPrep* prep, int do_scale);
void launch_batch_post(cudaStream_t s, int count, const BatchPrep* prep, const BatchPost* post);

}  // namespace b200
