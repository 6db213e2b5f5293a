// highs_b200/csrc/kkt_batch.cu -- HiGHS's post-solve KKT assessment (lpKktCheck) for many LP solutions in one launch
// (engine_batch.cu kkt_check_batch): one CTA per member, and no CTA waits on another, so any number of members of any size runs.
//
//   kkt_batch_check_kernel   the device-pointer variant only: a_start[0] == 0, a_start non-decreasing, a_index in
//                            [0, num_row), and a_start[num_col], which the host needs to lay out the workspace
//   kkt_batch_kernel         the row-major index, both residual vectors, pass 0 and pass 1
//
// Bits: every member's norms and sums are those of the host twin (kkt_check.cu kkt_host), because every floating-point
// accumulator receives the same terms in the same order, through the same kkt_logic.hpp functions:
//   |A x - row_value|      one thread per row, a DD over the row's positions ascending (the row-major index).  kkt_host's
//                          column sweep adds into a row's DD in exactly that order: columns ascending, then stored order;
//   |A'y - c + col_dual|   one thread per column, a DD over its positions ascending;
//   pass 0, pass 1         one thread, columns then rows.
// DD addition is not associative, so the warp-wide sums of kkt_check.cu's row_residual_k / col_residual_k and the block
// partials of its pass1_k cannot be used here; they are why the single device check matches the host twin only to tolerances.
// The build compiles this file with -fmad=false and IEEE division, and the host twin with -ffp-contract=off.
#include "batch_prep.hpp"
#include "kkt_batch.hpp"
#include "row_index.cuh"

namespace b200 {
namespace {

__global__ void __launch_bounds__(kThreads)
kkt_batch_check_kernel(const KktBatchMember* __restrict__ members, KktBatchSize* __restrict__ sizes) {
  __shared__ int flag[3];
  const KktBatchMember& M = members[blockIdx.x];
  KktBatchSize& S = sizes[blockIdx.x];
  const int t = threadIdx.x, n = M.n, m = M.m;
  if (t < 3) flag[t] = 0;
  __syncthreads();
  if (t == 0 && M.a_start[0] != 0) flag[0] = kPrepStart0;
  for (int j = t; j < n; j += kThreads)
    if (M.a_start[j + 1] < M.a_start[j]) flag[1] = kPrepDecreasing;
  __syncthreads();
  const int nnz = M.a_start[n];
  int err = flag[0] ? flag[0] : flag[1];
  if (!err && nnz > 0 && (!M.a_index || !M.a_value)) err = kPrepNull;
  if (err) {   // (uniform over the CTA)
    if (t == 0) { S.err = err; S.nnz = 0; }
    return;
  }
  for (int p = t; p < nnz; p += kThreads)
    if ((unsigned)M.a_index[p] >= (unsigned)m) flag[2] = kPrepIndex;
  __syncthreads();
  if (t == 0) { S.err = flag[2]; S.nnz = nnz; }
}

__global__ void __launch_bounds__(kThreads)
kkt_batch_kernel(const KktBatchMember* __restrict__ members, KktTolerances tol, KktBatchRec* __restrict__ recs) {
  __shared__ int sm[kThreads + 1];
  const KktBatchMember& M = members[blockIdx.x];
  const int t = threadIdx.x, n = M.n, m = M.m;
  const int nnz = M.a_start[n];

  // ---- the row-major index: row lengths (integer atomics: order-free), their scan, the walk by warp 0; the other warps
  // record each position's column meanwhile
  int* cursor = reinterpret_cast<int*>(M.rres);
  for (int i = t; i <= m; i += kThreads) M.rptr[i] = 0;
  __syncthreads();
  for (int p = t; p < nnz; p += kThreads) atomicAdd(&M.rptr[M.a_index[p]], 1);
  __syncthreads();
  const int total = block_scan(M.rptr, 1, m, sm);
  if (t == 0) M.rptr[m] = total;
  for (int i = t; i < m; i += kThreads) cursor[i] = M.rptr[i];
  __syncthreads();
  if (t < 32) {
    row_walk(nnz, M.a_index, cursor, M.rpos);
  } else {
    for (int j = t - 32; j < n; j += kThreads - 32)
      for (int p = M.a_start[j]; p < M.a_start[j + 1]; p++) M.colof[p] = j;
  }
  __syncthreads();

  // ---- the residual vectors (productQuad / productTransposeQuad: every product rounded, the sum carried in a DD)
  for (int i = t; i < m; i += kThreads) {
    DD v;
    for (int q = M.rptr[i]; q < M.rptr[i + 1]; q++) {
      const int p = M.rpos[q];
      v.add(M.col_value[M.colof[p]] * M.a_value[p]);
    }
    M.rres[i] = fabs(v.value() - M.row_value[i]);
  }
  for (int j = t; j < n; j += kThreads) {
    DD v;
    for (int p = M.a_start[j]; p < M.a_start[j + 1]; p++) v.add(M.row_dual[M.a_index[p]] * M.a_value[p]);
    const double dact = v.value() - M.col_cost[j];
    M.cres[j] = fabs(dact + M.col_dual[j]);
  }
  __syncthreads();

  // ---- pass 0 (the norms) and pass 1 (the sums), columns then rows, in one thread: kkt_host's loops
  if (t == 0) {
    const double sense = M.sense;
    double nb = 0, nc = 0;
    for (int j = 0; j < n; j++)
      kkt_pass0(tol, true, M.col_cost[j], M.col_lower[j], M.col_upper[j], M.col_value[j], M.col_dual[j], sense, nb, nc);
    for (int i = 0; i < m; i++)
      kkt_pass0(tol, false, 0.0, M.row_lower[i], M.row_upper[i], M.row_value[i], M.row_dual[i], sense, nb, nc);
    KktSums s;
    for (int j = 0; j < n; j++)
      kkt_pass1(tol, true, M.col_cost[j], M.col_lower[j], M.col_upper[j], M.col_value[j], M.col_dual[j], sense, nb, nc,
                M.cres[j], s);
    for (int i = 0; i < m; i++)
      kkt_pass1(tol, false, 0.0, M.row_lower[i], M.row_upper[i], M.row_value[i], M.row_dual[i], sense, nb, nc, M.rres[i], s);
    KktBatchRec& R = recs[blockIdx.x];
    R.norm_bounds = nb; R.norm_costs = nc; R.sums = s;
  }
}

}  // namespace

void launch_kkt_batch_check(cudaStream_t s, int count, const KktBatchMember* members, KktBatchSize* sizes) {
  if (count > 0) kkt_batch_check_kernel<<<count, kThreads, 0, s>>>(members, sizes);
}
void launch_kkt_batch(cudaStream_t s, int count, const KktBatchMember* members, KktTolerances t, KktBatchRec* recs) {
  if (count > 0) kkt_batch_kernel<<<count, kThreads, 0, s>>>(members, t, recs);
}

}  // namespace b200
