// highs_b200/csrc/setup_kernels.cu -- PDHG_Scale_Data on the device (the scaling stage of device_prep.cu).
//
// What cupdlp_scaling.c:47-120 (10 Ruiz passes), :174-231 (Pock-Chambolle, alpha = 1) and :17-45
// (scale_problem) do in 44 host sweeps over the nonzeros, on the column-major matrix resident in HBM:
//
//   * Ruiz norms are maxima -- order-free -- so one thread per nonzero divides its entry (row factor
//     first, then column factor, scale_problem's order) and folds |a_ij| into the next pass's row and
//     column norms with atomicMax on the bit pattern (non-negative doubles order like their bits).
//   * The Pock-Chambolle 1-norms must be added in the reference's order (a column's entries in storage
//     order; a row's entries with the columns ascending).  One warp per column / row: the lanes load 32
//     entries at once, then every lane adds the 32 values in index order (shuffle broadcast), so the
//     loads are parallel and the additions sequential.  Rows go through the row-major index of the
//     nonzeros (rptr / rpos).
//   * sqrt and division are IEEE-correctly rounded on the device as on the host (nvcc defaults
//     -prec-sqrt=true -prec-div=true; the file is compiled with -fmad=false like the rest), so the scaled
//     data are bit-identical to host_prep.cpp::scale and to the reference.
//
// STATUS: runs on hardware as the scaling stage of the device prologue (device_prep.cu, the default;
// tests/test_gpu_device_prep.py compares it bit for bit with the host path).
#include "setup_kernels.hpp"
#include "kernels.cuh"

#include <math.h>

namespace b200 {

namespace {
constexpr int kTpb = 256;

__device__ __forceinline__ void atomic_max_nonneg(double* addr, double v) {
  atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}

// norms of the first Ruiz pass: max |a_ij| per column and per row
__global__ void __launch_bounds__(kTpb)
first_norms_kernel(int nnz, const int* __restrict__ cidx, const int* __restrict__ colof, const double* __restrict__ cval,
                   double* __restrict__ cnorm, double* __restrict__ rnorm) {
  const int stride = gridDim.x * kTpb;
  for (int p = blockIdx.x * kTpb + threadIdx.x; p < nnz; p += stride) {
    const double a = fabs(cval[p]);
    atomic_max_nonneg(cnorm + colof[p], a);
    atomic_max_nonneg(rnorm + cidx[p], a);
  }
}

// norms -> factors (sqrt, with 0 -> 1), applied to the vectors (scale_problem :17-31, and the running
// scales :110-111); the norm slots are cleared for the next pass's atomicMax
__global__ void __launch_bounds__(kTpb)
col_factors_kernel(int n, double* __restrict__ cnorm, double* __restrict__ cs, double* __restrict__ cost,
                   double* __restrict__ lower, double* __restrict__ upper, double* __restrict__ colscale) {
  const int stride = gridDim.x * kTpb;
  for (int j = blockIdx.x * kTpb + threadIdx.x; j < n; j += stride) {
    const double v = sqrt(cnorm[j]);
    const double c = (v == 0.0) ? 1.0 : v;
    cs[j] = c;
    cost[j] = cost[j] / c;
    lower[j] = lower[j] * c;
    upper[j] = upper[j] * c;
    colscale[j] = colscale[j] * c;
    cnorm[j] = 0.0;
  }
}
__global__ void __launch_bounds__(kTpb)
row_factors_kernel(int m, double* __restrict__ rnorm, double* __restrict__ rs, double* __restrict__ rhs,
                   double* __restrict__ rowscale) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < m; i += stride) {
    const double q = rnorm[i];
    const double r = (q == 0.0) ? 1.0 : sqrt(q);
    rs[i] = r;
    rhs[i] = rhs[i] / r;
    rowscale[i] = rowscale[i] * r;
    rnorm[i] = 0.0;
  }
}

// one scaling sweep: a_ij <- (a_ij / r_i) / c_j.  mode 0: also gather the next Ruiz norms (max);
// mode 1: nothing else (the pass before Pock-Chambolle: its 1-norms are summed in order by
// ordered_abs_sums_kernel); mode 2: the last sweep, gather max |a_ij| of the final matrix
__global__ void __launch_bounds__(kTpb)
sweep_kernel(int nnz, int mode, const int* __restrict__ cidx, const int* __restrict__ colof, double* __restrict__ cval,
             const double* __restrict__ rs, const double* __restrict__ cs, double* __restrict__ cnorm,
             double* __restrict__ rnorm, double* __restrict__ amax) {
  __shared__ double sm[kTpb / 32];
  double am = 0.0;
  const int stride = gridDim.x * kTpb;
  for (int p = blockIdx.x * kTpb + threadIdx.x; p < nnz; p += stride) {
    const int i = cidx[p], j = colof[p];
    double v = cval[p] / rs[i];   // row division first, then column division (cupdlp_scaling.c:33-41)
    v = v / cs[j];
    cval[p] = v;
    const double a = fabs(v);
    if (mode == 0) {
      // the nonzeros are stored by column, so a warp's 32 consecutive entries fall into a few CONTIGUOUS runs of equal
      // columns: a segmented suffix-maximum with shuffles (max is order-free: exact) leaves each run's maximum in its
      // first lane, and only that lane issues the column atomic (~8x fewer same-address atomics)
      if (__activemask() == 0xffffffffu) {
        const int lane = threadIdx.x & 31;
        double cm = a;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const double v2 = __shfl_down_sync(0xffffffffu, cm, o);
          const int j2 = __shfl_down_sync(0xffffffffu, j, o);
          if (lane + o < 32 && j2 == j) cm = v2 > cm ? v2 : cm;
        }
        const int jprev = __shfl_up_sync(0xffffffffu, j, 1);
        if (lane == 0 || jprev != j) atomic_max_nonneg(cnorm + j, cm);
      } else {
        atomic_max_nonneg(cnorm + j, a);
      }
      atomic_max_nonneg(rnorm + i, a);
    } else if (mode == 2) {
      am = a > am ? a : am;
    }
  }
  if (mode == 2) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const double t = __shfl_down_sync(0xffffffffu, am, o); am = t > am ? t : am; }
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = am;
    __syncthreads();
    if (threadIdx.x == 0) {
      double b = 0.0;
      for (int w = 0; w < kTpb / 32; w++) b = sm[w] > b ? sm[w] : b;
      atomic_max_nonneg(amax, b);
    }
  }
}

// out[r] = sum over q in [ptr[r], ptr[r+1]) of |val[pos ? pos[q] : q]|, added in q order (see the header).
// One THREAD per row for rows of up to 64 entries (the usual case: a lane just walks its row; neighbouring lanes walk
// neighbouring rows, so the lines are shared through L1); longer rows are then taken one at a time by the whole warp: the
// lanes load 32 entries at once and every lane adds them in index order (shuffle broadcast) -- same order, parallel loads.
constexpr int kShortRow = 64;
__global__ void __launch_bounds__(kTpb)
ordered_abs_sums_kernel(int nrows, const int* __restrict__ ptr, const int* __restrict__ pos,
                        const double* __restrict__ val, double* __restrict__ out) {
  const int r = blockIdx.x * kTpb + threadIdx.x, lane = threadIdx.x & 31;
  int b = 0, e = 0;
  if (r < nrows) { b = ptr[r]; e = ptr[r + 1]; }
  const bool is_long = e - b > kShortRow;
  if (r < nrows && !is_long) {
    double sum = 0.0;
    for (int q = b; q < e; q++) sum = sum + fabs(val[pos ? pos[q] : q]);
    out[r] = sum;
  }
  unsigned todo = __ballot_sync(0xffffffffu, is_long);   // (whole warps reach this point together)
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    const int lb = __shfl_sync(0xffffffffu, b, src), le = __shfl_sync(0xffffffffu, e, src);
    double sum = 0.0;
    for (int base = lb; base < le; base += 32) {
      const int q = base + lane;
      double a = 0.0;
      if (q < le) a = fabs(val[pos ? pos[q] : q]);
      const int cnt = (le - base) < 32 ? (le - base) : 32;   // warp-uniform
      for (int k = 0; k < cnt; k++) sum = sum + __shfl_sync(0xffffffffu, a, k);
    }
    if (lane == 0) out[(r - lane) + src] = sum;
  }
}

// max |a_ij| of an unscaled matrix (scaling switched off: PDHG_Init_Step_Sizes still needs it)
__global__ void __launch_bounds__(kTpb) abs_max_kernel(int nnz, const double* __restrict__ val, double* __restrict__ amax) {
  double am = 0.0;
  const int stride = gridDim.x * kTpb;
  for (int p = blockIdx.x * kTpb + threadIdx.x; p < nnz; p += stride) { const double a = fabs(val[p]); am = a > am ? a : am; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const double t = __shfl_down_sync(0xffffffffu, am, o); am = t > am ? t : am; }
  if ((threadIdx.x & 31) == 0) atomic_max_nonneg(amax, am);
}

// ---- HiPDLP mode (Scaling::scaleProblem, hipdlp/scaling.cc; host twin host_prep_hipdlp.cpp::scale_hipdlp)
// OP 0: max |v| (Ruiz), 1: sum |v| (Pock-Chambolle, alpha = 1), 2: sum v^2 (L2).  The host evaluates the Pock-Chambolle terms as
// std::pow(|v|, 2 - alpha) and std::pow(|v|, alpha) with alpha = 1; glibc's pow returns its argument exactly for an exponent of
// 1.0, so |v| IS that term.  CUDA's pow is only guaranteed to 2 ulp, so it is not called here.
template <int OP> __device__ __forceinline__ double hip_term(double v) { return OP == 2 ? v * v : fabs(v); }
template <int OP> __device__ __forceinline__ double hip_op(double a, double t) {
  return OP == 0 ? (a < t ? t : a) : a + t;   // std::max(a, t) / a + t, the host's folds
}
// out[r] = fold of the terms of entries [ptr[r], ptr[r+1]) (through pos when given) in index order; same scheme as
// ordered_abs_sums_kernel: one thread per short row, one warp (loads in parallel, additions in order) per long row
template <int OP>
__global__ void __launch_bounds__(kTpb)
hip_ordered_reduce_kernel(int nrows, const int* __restrict__ ptr, const int* __restrict__ pos, const double* __restrict__ val,
                          double* __restrict__ out) {
  const int r = blockIdx.x * kTpb + threadIdx.x, lane = threadIdx.x & 31;
  int b = 0, e = 0;
  if (r < nrows) { b = ptr[r]; e = ptr[r + 1]; }
  const bool is_long = e - b > kShortRow;
  if (r < nrows && !is_long) {
    double a = 0.0;
    for (int q = b; q < e; q++) a = hip_op<OP>(a, hip_term<OP>(val[pos ? pos[q] : q]));
    out[r] = a;
  }
  unsigned todo = __ballot_sync(0xffffffffu, is_long);
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    const int lb = __shfl_sync(0xffffffffu, b, src), le = __shfl_sync(0xffffffffu, e, src);
    double a = 0.0;
    for (int base = lb; base < le; base += 32) {
      const int q = base + lane;
      const double t = q < le ? hip_term<OP>(val[pos ? pos[q] : q]) : 0.0;
      const int cnt = (le - base) < 32 ? (le - base) : 32;
      for (int k = 0; k < cnt; k++) a = hip_op<OP>(a, __shfl_sync(0xffffffffu, t, k));
    }
    if (lane == 0) out[(r - lane) + src] = a;
  }
}
// fold -> factor in place (scaling.cc: Ruiz sqrt with 0 -> 1; Pock-Chambolle sqrt(pow(sum, 1 / alpha)) = sqrt(sum); L2
// sqrt(sqrt(sum)); empty / zero -> 1)
__global__ void __launch_bounds__(kTpb) hip_factors_kernel(int len, int op, double* __restrict__ v) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) {
    const double q = v[i];
    double f;
    if (op == 0) { f = sqrt(q); if (f == 0.0) f = 1.0; }
    else if (op == 1) f = q > 0.0 ? sqrt(q) : 1.0;
    else f = q > 0.0 ? sqrt(sqrt(q)) : 1.0;
    v[i] = f;
  }
}
// Scaling::applyScaling (scaling.cc:232-263)
__global__ void __launch_bounds__(kTpb)
hip_apply_cols_kernel(int n, const double* __restrict__ cs, double* __restrict__ cost, double* __restrict__ lower,
                      double* __restrict__ upper, double* __restrict__ colscale) {
  const int stride = gridDim.x * kTpb;
  for (int j = blockIdx.x * kTpb + threadIdx.x; j < n; j += stride) {
    const double c = cs[j];
    cost[j] = cost[j] / c;
    if (lower[j] > -INFINITY) lower[j] = lower[j] * c;
    if (upper[j] < INFINITY) upper[j] = upper[j] * c;
    colscale[j] = colscale[j] * c;
  }
}
__global__ void __launch_bounds__(kTpb)
hip_apply_rows_kernel(int m, const double* __restrict__ rs, double* __restrict__ rhs, double* __restrict__ rup,
                      double* __restrict__ rowscale) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < m; i += stride) {
    const double r = rs[i];
    if (rhs[i] > -INFINITY) rhs[i] = rhs[i] / r;
    if (rup[i] < INFINITY) rup[i] = rup[i] / r;
    rowscale[i] = rowscale[i] * r;
  }
}
__global__ void __launch_bounds__(kTpb)
hip_apply_nnz_kernel(int nnz, const int* __restrict__ cidx, const int* __restrict__ colof, const double* __restrict__ rs,
                     const double* __restrict__ cs, double* __restrict__ cval) {
  const int stride = gridDim.x * kTpb;
  for (int p = blockIdx.x * kTpb + threadIdx.x; p < nnz; p += stride) cval[p] = cval[p] / (rs[cidx[p]] * cs[colof[p]]);   // ONE division by the product
}

inline int grid_for(long long work) {
  long long g = (work + kTpb - 1) / kTpb;
  if (g < 1) g = 1;
  return (int)(g > kGridUnit * 32LL ? kGridUnit * 32LL : g);
}
inline int warp_grid(int rows) { return (int)(((long long)rows * 32 + kTpb - 1) / kTpb); }

template <int OP>
void hip_pass(cudaStream_t s, const DevForm& F, DevScaleScratch& w, const int* rptr, const int* rpos, double* row_upper) {
  if (F.n > 0) {
    hip_ordered_reduce_kernel<OP><<<(F.n + kTpb - 1) / kTpb, kTpb, 0, s>>>(F.n, F.cbeg, nullptr, F.cval, w.cs);
    hip_factors_kernel<<<grid_for(F.n), kTpb, 0, s>>>(F.n, OP, w.cs);
  }
  if (F.m > 0) {
    hip_ordered_reduce_kernel<OP><<<(F.m + kTpb - 1) / kTpb, kTpb, 0, s>>>(F.m, rptr, rpos, F.cval, w.rs);
    hip_factors_kernel<<<grid_for(F.m), kTpb, 0, s>>>(F.m, OP, w.rs);
  }
  if (F.n > 0) hip_apply_cols_kernel<<<grid_for(F.n), kTpb, 0, s>>>(F.n, w.cs, F.cost, F.lower, F.upper, F.colscale);
  if (F.nnz > 0) hip_apply_nnz_kernel<<<grid_for(F.nnz), kTpb, 0, s>>>(F.nnz, F.cidx, F.colof, w.rs, w.cs, F.cval);
  if (F.m > 0) hip_apply_rows_kernel<<<grid_for(F.m), kTpb, 0, s>>>(F.m, w.rs, F.rhs, row_upper, F.rowscale);
}
}  // namespace

bool device_scale_hipdlp(cudaStream_t s, const DevForm& F, DevScaleScratch& w, const int* rptr, const int* rpos,
                         double* row_upper, int scaling_mode, int ruiz_iterations) {
  bool scaled = false;
  if (scaling_mode & 1) {
    for (int it = 0; it < ruiz_iterations; it++) hip_pass<0>(s, F, w, rptr, rpos, row_upper);
    scaled = true;
  }
  if (scaling_mode & 4) { hip_pass<1>(s, F, w, rptr, rpos, row_upper); scaled = true; }
  if (scaling_mode & 2) { hip_pass<2>(s, F, w, rptr, rpos, row_upper); scaled = true; }
  device_abs_max(s, F.nnz, F.cval, w.amax);
  return scaled;
}

void device_abs_max(cudaStream_t s, int nnz, const double* val, double* amax) {
  cudaMemsetAsync(amax, 0, sizeof(double), s);
  if (nnz > 0) abs_max_kernel<<<grid_for(nnz), kTpb, 0, s>>>(nnz, val, amax);
}

void device_scale_ruiz(cudaStream_t s, const DevForm& F, DevScaleScratch& w) {
  cudaMemsetAsync(w.cnorm, 0, sizeof(double) * (size_t)(F.n > 0 ? F.n : 1), s);
  cudaMemsetAsync(w.rnorm, 0, sizeof(double) * (size_t)(F.m > 0 ? F.m : 1), s);
  if (F.nnz > 0) first_norms_kernel<<<grid_for(F.nnz), kTpb, 0, s>>>(F.nnz, F.cidx, F.colof, F.cval, w.cnorm, w.rnorm);
  constexpr int kRuiz = 10;
  for (int it = 0; it < kRuiz; it++) {
    if (F.n > 0) col_factors_kernel<<<grid_for(F.n), kTpb, 0, s>>>(F.n, w.cnorm, w.cs, F.cost, F.lower, F.upper, F.colscale);
    if (F.m > 0) row_factors_kernel<<<grid_for(F.m), kTpb, 0, s>>>(F.m, w.rnorm, w.rs, F.rhs, F.rowscale);
    if (F.nnz > 0)
      sweep_kernel<<<grid_for(F.nnz), kTpb, 0, s>>>(F.nnz, it == kRuiz - 1 ? 1 : 0, F.cidx, F.colof, F.cval, w.rs, w.cs,
                                                    w.cnorm, w.rnorm, w.amax);
  }
}

void device_scale_pock_chambolle(cudaStream_t s, const DevForm& F, DevScaleScratch& w, const int* rptr, const int* rpos) {
  // 1-norms in the reference's summation order (empty columns / rows sum to 0 -> factor 1)
  if (F.n > 0) ordered_abs_sums_kernel<<<(F.n + kTpb - 1) / kTpb, kTpb, 0, s>>>(F.n, F.cbeg, nullptr, F.cval, w.cnorm);
  if (F.m > 0) ordered_abs_sums_kernel<<<(F.m + kTpb - 1) / kTpb, kTpb, 0, s>>>(F.m, rptr, rpos, F.cval, w.rnorm);
  if (F.n > 0) col_factors_kernel<<<grid_for(F.n), kTpb, 0, s>>>(F.n, w.cnorm, w.cs, F.cost, F.lower, F.upper, F.colscale);
  if (F.m > 0) row_factors_kernel<<<grid_for(F.m), kTpb, 0, s>>>(F.m, w.rnorm, w.rs, F.rhs, F.rowscale);
  cudaMemsetAsync(w.amax, 0, sizeof(double), s);
  if (F.nnz > 0)
    sweep_kernel<<<grid_for(F.nnz), kTpb, 0, s>>>(F.nnz, 2, F.cidx, F.colof, F.cval, w.rs, w.cs, w.cnorm, w.rnorm, w.amax);
}

}  // namespace b200

// ------------------------------------------------------------------ sliced-ELL fill on the device
// Given the PLAN of a sliced-ELL matrix (host_prep.cpp::plan_sell: slice offsets / lengths / masks, long-row
// segments) the body and the long-row arrays are filled straight from the scaled matrix in HBM, so the 100 MB
// layouts are never built on the host nor sent over PCIe.  One warp per slice, lane = row: the lane walks ITS
// row's entries in source order (row-major index for A, a column's storage order for A') and stores them k-major /
// lane-minor, i.e. fully coalesced; padding is written as (0, 0) by the same lane.
namespace b200 {
namespace {
__global__ void __launch_bounds__(kTpb)
fill_sell_body_kernel(int nrows, int nslices, const int4* __restrict__ slices, const int* __restrict__ perm, SellSource S,
                      int* __restrict__ col, double* __restrict__ val) {
  const int s = (blockIdx.x * kTpb + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (s >= nslices) return;
  const int4 sl = slices[s];
  const int row = s * 32 + lane;
  const bool live = row < nrows && !(((unsigned)sl.z >> lane) & 1u);
  int b = 0, ln = 0;
  if (live) { const int r = perm[row]; b = S.beg[r]; ln = S.end[r] - b; }
  for (int k = 0; k < sl.y; k++) {
    int c = 0;
    double v = 0.0;
    if (k < ln) {
      const int q = b + k;
      const int src = S.pos ? S.pos[q] : q;
      c = S.colmap[S.idx[src] - S.idx_offset];
      v = S.val[src];
    }
    const size_t o = (size_t)sl.x + 32 * (size_t)k + lane;
    col[o] = c;
    val[o] = v;
  }
}

// one CTA per long row: its entries, in source order, into lcol / lval at the offset the plan assigned
__global__ void __launch_bounds__(kTpb)
fill_sell_long_kernel(const int4* __restrict__ long_rows, const int4* __restrict__ segs, const int* __restrict__ perm,
                      SellSource S, int* __restrict__ lcol, double* __restrict__ lval) {
  const int4 lr = long_rows[blockIdx.x];
  const int r = perm[lr.x];
  const int b = S.beg[r], ln = S.end[r] - b;
  const int base = segs[lr.y].y;
  for (int e = threadIdx.x; e < ln; e += kTpb) {
    const int q = b + e;
    const int src = S.pos ? S.pos[q] : q;
    lcol[base + e] = S.colmap[S.idx[src] - S.idx_offset];
    lval[base + e] = S.val[src];
  }
}
}  // namespace

void device_fill_sell(cudaStream_t s, int nrows, int nslices, const int4* slices, const int* perm, const SellSource& S,
                      int* col, double* val, long long padded, int n_long, const int4* long_rows, const int4* segs,
                      int* lcol, double* lval) {
  if (nslices > 0) fill_sell_body_kernel<<<warp_grid(nslices), kTpb, 0, s>>>(nrows, nslices, slices, perm, S, col, val);
  cudaMemsetAsync(col + padded, 0, 32 * sizeof(int), s);
  cudaMemsetAsync(val + padded, 0, 32 * sizeof(double), s);
  if (n_long > 0) fill_sell_long_kernel<<<n_long, kTpb, 0, s>>>(long_rows, segs, perm, S, lcol, lval);
}

}  // namespace b200
