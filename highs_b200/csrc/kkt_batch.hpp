// highs_b200/csrc/kkt_batch.hpp -- b200pdlp_kkt_check_batch and b200pdlp_kkt_check_batch_device: lpKktCheck for many LP
// solutions in one call, one CTA per member (kkt_batch.cu), each member's bits those of the host twin (kkt_check.cu kkt_host).
#pragma once
#include <cuda_runtime.h>

#include "../../include/b200pdlp.h"
#include "kkt_logic.hpp"

namespace b200 {

// One member, filled by the host.  The LP and solution arrays are only read; the four workspace arrays lie in the batch's
// pool.
struct KktBatchMember {
  int n, m;
  double sense;
  const int* a_start; const int* a_index; const double* a_value;
  const double *col_cost, *col_lower, *col_upper, *row_lower, *row_upper;
  const double *col_value, *col_dual, *row_value, *row_dual;
  int* rptr;      // [m + 1] row lengths, then the row pointer of the row-major index
  int* rpos;      // [nnz]   its positions into a_index / a_value: per row ascending (columns ascending, then stored order)
  int* colof;     // [nnz]   the column of each position
  double* rres;   // [m]     the row cursor of the walk (as ints), then |A x - row_value|
  double* cres;   // [n]     |A'y - c + col_dual|
};

// What the check kernel of the device-pointer variant writes per member: err, a BatchPrepErr (batch_prep.hpp) of the array
// checks, and nnz = a_start[num_col], valid when err is kPrepOk.  Only a_start, a_index and a_value are read.
struct KktBatchSize {
  int err, nnz;
};

// What the assessment writes per member: getKktFailures' two norms and pass 1's sums
struct KktBatchRec {
  double norm_bounds, norm_costs;
  KktSums sums;
};

void launch_kkt_batch_check(cudaStream_t s, int count, const KktBatchMember* members, KktBatchSize* sizes);
// every member's arrays must be valid: the host checked them (b200pdlp_kkt_check_batch) or launch_kkt_batch_check did
void launch_kkt_batch(cudaStream_t s, int count, const KktBatchMember* members, KktTolerances t, KktBatchRec* recs);

// kkt_check.cu: the HighsInfo fields and lpKktCheck's status rules from the sums (the epilogue every KKT check shares)
void finalize_kkt(const KktSums& s, double offset, const KktTolerances& t, b200pdlp_kkt_info* out);
KktTolerances tolerances_of(const b200pdlp_kkt_tolerances* t);

}  // namespace b200
