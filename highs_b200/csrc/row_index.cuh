// highs_b200/csrc/row_index.cuh -- the row-major index of a column-major matrix, built by one CTA of kThreads threads:
// the row pointer by a block scan of the row lengths, the positions by one warp's walk.  batch_prep.cu and kkt_batch.cu
// include it.
#pragma once
#include "kernels.cuh"

namespace b200 {

// in-place exclusive scan of a[0], a[stride], ... a[(len - 1) * stride] by one CTA (each thread owns a contiguous chunk);
// returns the total in every thread.  sm: kThreads + 1 ints of shared memory.
static __device__ int block_scan(int* a, int stride, int len, int* sm) {
  const int t = threadIdx.x;
  const int chunk = (len + kThreads - 1) / kThreads;
  const int b = min(t * chunk, len), e = min(b + chunk, len);
  int s = 0;
  for (int i = b; i < e; i++) s += a[(size_t)i * stride];
  sm[t] = s;
  __syncthreads();
  if (t == 0) {
    int run = 0;
    for (int k = 0; k < kThreads; k++) { const int v = sm[k]; sm[k] = run; run += v; }
    sm[kThreads] = run;
  }
  __syncthreads();
  int run = sm[t];
  for (int i = b; i < e; i++) { const int v = a[(size_t)i * stride]; a[(size_t)i * stride] = run; run += v; }
  const int total = sm[kThreads];
  __syncthreads();
  return total;
}

// the row-major index by one warp (build_row_index): position p of row[p] goes to slot rwork[row[p]]++, positions ascending.
// The warp walks the positions in order, 32 at a time; lanes that hit the same row take consecutive slots in lane order.
__device__ __forceinline__ void row_walk(int nnz, const int* row, int* rwork, int* rpos) {
  const int lane = threadIdx.x & 31;
  for (int base = 0; base < nnz; base += 32) {
    const int p = base + lane;
    const int i = p < nnz ? row[p] : -1 - lane;
    const unsigned same = __match_any_sync(0xffffffffu, i);
    int q = 0;
    if (p < nnz) q = rwork[i] + __popc(same & ((1u << lane) - 1u));
    __syncwarp();
    if (p < nnz) {
      rpos[q] = p;
      if (lane == __ffs(same) - 1) rwork[i] += __popc(same);
    }
    __syncwarp();
  }
}

}  // namespace b200
