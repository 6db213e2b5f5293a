// highs_b200/csrc/hip_form.cuh -- formulate_hipdlp, scale_hipdlp and hip_host_postsolve on device arrays, one CTA of kThreads
// threads per LP.  hip_form (formulate_hipdlp, the row-major indexes, scale_hipdlp) is the prologue of both
// hip_batch_prep_kernel (batch_prep.cu, ordered members) and hip_tree_form_kernel (batch_tree_prep.cu, tree members);
// hip_postsolve is the postsolve of both hip_batch_post_kernel and hip_tree_post_kernel.  Every value is the host's
// (host_prep_hipdlp.cpp) with the same operations on the same operands; both files are compiled with -fmad=false and IEEE
// division and square root.
#pragma once
#include "batch_kernels.hpp"
#include "batch_prep.hpp"
#include "host_prep.hpp"
#include "row_index.cuh"

namespace b200 {
namespace {

constexpr double kInf = __builtin_huge_val();

// a double as a radix key: ascending numeric order, -0.0 before +0.0 (device_prep.cu value_key_kernel's convention)
__device__ __forceinline__ unsigned long long value_key(double v) {
  const unsigned long long u = (unsigned long long)__double_as_longlong(v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

// The fold of one scaling pass over a column's or a row's terms, and its factor (Scaling::scaleProblem).  OP 0: Ruiz, max |v|
// -> sqrt, 0 -> 1; 1: Pock-Chambolle with alpha = 1, sum |v| -> sqrt; 2: L2, sum v^2 -> sqrt(sqrt).  The host evaluates the
// Pock-Chambolle terms and factors as std::pow(x, 1.0), which glibc returns exactly as x, so the identity is used here.
template <int OP> __device__ __forceinline__ double hip_fold(double a, double v) {
  if (OP == 0) { const double t = fabs(v); return (a < t) ? t : a; }   // std::max(a, t)
  return OP == 1 ? a + fabs(v) : a + v * v;
}
template <int OP> __device__ __forceinline__ double hip_factor(double a) {
  if (OP == 0) { const double f = sqrt(a); return f == 0.0 ? 1.0 : f; }
  return a > 0.0 ? (OP == 1 ? sqrt(a) : sqrt(sqrt(a))) : 1.0;
}

// one scaling pass (scale_hipdlp's pass + apply_hipdlp): column folds in cbeg order, row folds in row-major order, then
// every entry divided once by the product rs[i] * cs[j]; only finite bounds, rhs and row upper bounds are scaled
template <int OP>
__device__ void hip_scale_pass(const BatchPrep& P, double* cost, double* lower, double* upper, double* colscale, double* rlo,
                               double* rup, double* rowscale) {
  const int t = threadIdx.x, n = P.n, m = P.m;
  for (int j = t; j < n; j += kThreads) {
    double a = 0.0;
    for (int p = P.cbeg[j]; p < P.cbeg[j + 1]; p++) a = hip_fold<OP>(a, P.cval[p]);
    P.cs[j] = hip_factor<OP>(a);
  }
  for (int i = t; i < m; i += kThreads) {
    double a = 0.0;
    for (int q = P.rptr[i]; q < P.rptr[i + 1]; q++) a = hip_fold<OP>(a, P.cval[P.rpos[q]]);
    P.rs[i] = hip_factor<OP>(a);
  }
  __syncthreads();
  for (int j = t; j < n; j += kThreads) {
    const double c = P.cs[j];
    cost[j] /= c;
    if (lower[j] > -kInf) lower[j] *= c;
    if (upper[j] < kInf) upper[j] *= c;
    colscale[j] *= c;
    for (int p = P.cbeg[j]; p < P.cbeg[j + 1]; p++) P.cval[p] /= (P.rs[P.cidx[p]] * c);
  }
  for (int i = t; i < m; i += kThreads) {
    const double r = P.rs[i];
    if (rlo[i] > -kInf) rlo[i] /= r;
    if (rup[i] < kInf) rup[i] /= r;
    rowscale[i] *= r;
  }
  __syncthreads();
}

// The form's data vectors in standard-form order, where the prologue builds and scales them
struct HipFormVecs {
  double *cost, *lower, *upper, *colscale, *rlo, *rup, *rowscale;
};

// ---- formulate_hipdlp.  A structural column keeps cbeg[j] = a_start[j], its entries ordered by (new row, value) with LEQ
// rows negated.  Stored rows strictly ascending: the new rows ascend inside the equality-like group and inside the rest, so
// that order is the stable partition.  Other columns go on the work list H.sortcols (*nsort of them, a shared counter that
// starts at 0) for a sort by (new row, value key, stored index).  Costs keep their sign and bounds are not clamped.
__device__ __forceinline__ void hip_formulate(const BatchPrep& P, const HipBatchPrep& H, const HipFormVecs& F, int* nsort) {
  const int t = threadIdx.x;
  const int n0 = P.n0, m = P.m, n = P.n, nnz = P.nnz;
  const int nnz0 = nnz - (n - n0);
  const int* rni = P.row_new_idx;
  const int* rcl = P.row_class;
  for (int j = t; j < n0; j += kThreads) {
    const int p0 = P.a_start[j], p1 = P.a_start[j + 1];
    P.cbeg[j] = p0;
    bool ascending = true;
    for (int p = p0 + 1; p < p1; p++)
      if (P.a_index[p] <= P.a_index[p - 1]) ascending = false;
    if (ascending) {
      int k = p0;
      for (int p = p0; p < p1; p++) {
        const int i = P.a_index[p];
        if (rni[i] < P.neq) { P.cidx[k] = rni[i]; P.cval[k] = rcl[i] == kLeq ? -P.a_value[p] : P.a_value[p]; P.pcol[k] = j; k++; }
      }
      for (int p = p0; p < p1; p++) {
        const int i = P.a_index[p];
        if (rni[i] >= P.neq) { P.cidx[k] = rni[i]; P.cval[k] = rcl[i] == kLeq ? -P.a_value[p] : P.a_value[p]; P.pcol[k] = j; k++; }
      }
    } else {
      H.sortcols[atomicAdd(nsort, 1)] = j;
    }
    F.cost[j] = P.col_cost[j];
    F.lower[j] = P.col_lower[j];
    F.upper[j] = P.col_upper[j];
    F.colscale[j] = 1.0;
  }
  for (int i = t; i < m; i += kThreads) {
    const int r = rni[i], c = rcl[i];
    F.rlo[r] = (c == kEq || c == kGeq) ? P.row_lower[i] : c == kLeq ? -P.row_upper[i] : 0.0;
    F.rup[r] = c == kEq ? P.row_upper[i] : (c == kGeq || c == kLeq) ? kInf : 0.0;
    F.rowscale[r] = 1.0;
    H.optr[i] = P.rptr[r] - (P.slack[i] >= 0);   // the caller's row length (rptr: the form's, before its scan)
    if (P.slack[i] >= 0) {   // one -1 slack column per BOUND / FREE row, in row order, with the row's raw bounds
      const int j = n0 + P.slack[i], q = nnz0 + P.slack[i];
      P.cbeg[j] = q; P.cidx[q] = r; P.cval[q] = -1.0; P.pcol[q] = j;
      F.cost[j] = 0.0;
      F.lower[j] = P.row_lower[i];
      F.upper[j] = P.row_upper[i];
      F.colscale[j] = 1.0;
    }
  }
  if (t == 0) P.cbeg[n] = nnz;
}

// Entries [k0, k1) of the caller's column j (stored at a_start[j] + k), each ranked by the whole CTA among those entries
// under (new row, value key, stored index): put(rank, k, row, value) for each.  The other entries are streamed through
// shared memory (s_row, s_key: kThreads each) a tile at a time.  (value_key orders -0.0 before +0.0, which std::sort leaves
// in either order.)  Costs (k1 - k0)^2 / kThreads comparisons per thread.
template <class Put>
__device__ __forceinline__ void hip_rank_entries(const BatchPrep& P, int j, int k0, int k1, int* s_row,
                                                 unsigned long long* s_key, Put&& put) {
  const int t = threadIdx.x;
  const int* rni = P.row_new_idx;
  const int* rcl = P.row_class;
  const int p0 = P.a_start[j] + k0, len = k1 - k0;
  for (int b0 = 0; b0 < len; b0 += kThreads) {
    const int k = b0 + t;
    int row = 0;
    double v = 0.0;
    unsigned long long key = 0;
    if (k < len) {
      const int i = P.a_index[p0 + k];
      row = rni[i];
      v = rcl[i] == kLeq ? -P.a_value[p0 + k] : P.a_value[p0 + k];
      key = value_key(v);
    }
    int rank = 0;
    for (int h0 = 0; h0 < len; h0 += kThreads) {
      __syncthreads();
      if (h0 + t < len) {
        const int i = P.a_index[p0 + h0 + t];
        s_row[t] = rni[i];
        s_key[t] = value_key(rcl[i] == kLeq ? -P.a_value[p0 + h0 + t] : P.a_value[p0 + h0 + t]);
      }
      __syncthreads();
      if (k < len) {
        const int cnt = min(kThreads, len - h0);
        for (int h = 0; h < cnt; h++) {
          const int rh = s_row[h];
          const unsigned long long kh = s_key[h];
          rank += rh < row || (rh == row && (kh < key || (kh == key && h0 + h < k)));
        }
      }
    }
    if (k < len) put(rank, k0 + k, row, v, key);
  }
}

// ---- the row-major indexes (build_row_index) of the form and of the caller's matrix (the postsolve's row sums), and |c|^2,
// |b|^2 of the unscaled form in index order (formulate_hipdlp's norms, squared) into P.rec
__device__ __forceinline__ void hip_row_indexes(const BatchPrep& P, const HipBatchPrep& H, const HipFormVecs& F, int* sm) {
  const int t = threadIdx.x, wid = t >> 5;
  const int n0 = P.n0, m = P.m, n = P.n, nnz = P.nnz;
  const int nnz0 = nnz - (n - n0);
  const int rtotal = block_scan(P.rptr, 1, m, sm);
  if (t == 0) P.rptr[m] = rtotal;
  const int ototal = block_scan(H.optr, 1, m, sm);
  if (t == 0) H.optr[m] = ototal;
  for (int i = t; i < m; i += kThreads) P.rwork[i] = P.rptr[i];
  __syncthreads();
  if (wid == 0) {
    row_walk(nnz, P.cidx, P.rwork, P.rpos);
    for (int i = t; i < m; i += 32) P.rwork[i] = H.optr[i];
    __syncwarp();
    row_walk(nnz0, P.a_index, P.rwork, H.opos);
  } else if (t == 32 || t == 64) {
    const double* v = t == 32 ? F.cost : F.rlo;
    const int len = t == 32 ? n : m;
    double s = 0.0;
    for (int q = 0; q < len; q++) s += v[q] * v[q];
    P.rec[t == 32 ? kRecCostSq : kRecRhsSq] = s;
  }
  __syncthreads();
}

// ---- scale_hipdlp: Ruiz x ruiz_iterations, then Pock-Chambolle, then L2, each pass as its bit of scaling_mode says
__device__ __forceinline__ void hip_scale(const BatchPrep& P, const HipFormVecs& F, int scaling_mode, int ruiz_iterations) {
  if (scaling_mode & 1)
    for (int it = 0; it < ruiz_iterations; it++)
      hip_scale_pass<0>(P, F.cost, F.lower, F.upper, F.colscale, F.rlo, F.rup, F.rowscale);
  if (scaling_mode & 4) hip_scale_pass<1>(P, F.cost, F.lower, F.upper, F.colscale, F.rlo, F.rup, F.rowscale);
  if (scaling_mode & 2) hip_scale_pass<2>(P, F.cost, F.lower, F.upper, F.colscale, F.rlo, F.rup, F.rowscale);
}

// ---- the whole HiPDLP prologue up to the layouts: formulate_hipdlp with its listed columns ranked, the row-major indexes and
// scale_hipdlp, the data vectors at F.  long_sort(j, len, s_row, s_key) sorts a listed column in its own way and returns
// true, or returns false to have it ranked whole here.  sm: kThreads + 1 ints of shared memory.
template <class LongSort>
__device__ __forceinline__ void hip_form(const BatchPrep& P, const HipBatchPrep& H, const HipFormVecs& F, int scaling_mode,
                                         int ruiz_iterations, int* sm, LongSort&& long_sort) {
  __shared__ int s_row[kThreads];
  __shared__ unsigned long long s_key[kThreads];
  __shared__ int nsort;
  if (threadIdx.x == 0) nsort = 0;
  __syncthreads();
  hip_formulate(P, H, F, &nsort);
  __syncthreads();
  const int ns = nsort;
  for (int s = 0; s < ns; s++) {
    const int j = H.sortcols[s];
    const int p0 = P.a_start[j], len = P.a_start[j + 1] - p0;
    if (long_sort(j, len, s_row, s_key)) continue;
    hip_rank_entries(P, j, 0, len, s_row, s_key, [&](int rank, int, int row, double val, unsigned long long) {
      const int q = p0 + rank;
      P.cidx[q] = row; P.cval[q] = val; P.pcol[q] = j;
    });
  }
  __syncthreads();
  hip_row_indexes(P, H, F, sm);
  hip_scale(P, F, scaling_mode, ruiz_iterations);
}

// ---- hip_host_postsolve of the returned iterate into the caller's device vectors.  The member's vectors are in device
// order: standard-form column j is device column cpos(j), row r device row rpos(r) (the identities for an ordered member).
template <class CPos, class RPos>
__device__ __forceinline__ void hip_postsolve(const BatchPrep& P, const HipBatchPrep& H, const HipBatchPost& Q, int scaled,
                                              CPos cpos, RPos rpos) {
  if (!(Q.col_value && Q.col_dual && Q.row_value && Q.row_dual)) return;
  const int n0 = P.n0, m = P.m, n = P.n;
  using V = HipBatchVec;
  const double* v = P.vec;
  const double* x = Q.sol == 1 ? V::col(v, n, V::kXn) : V::col(v, n, V::kX);
  const double* y = Q.sol == 1 ? V::row(v, n, m, V::kYn) : V::row(v, n, m, V::kY);
  const double *colscale = V::col(v, n, V::kColscale), *sp = V::col(v, n, V::kSp), *sn = V::col(v, n, V::kSn);
  const double* rowscale = V::row(v, n, m, V::kRowscale);
  const bool conv = Q.sol >= 0;
  const double sense = P.sense;
  // the unscaled primal value of structural column j (hip_host_postsolve's hx[j])
  const auto xval = [&](int j) {
    const int k = cpos(j);
    double xv = conv ? x[k] : 0.0;
    if (scaled) xv /= colscale[k];
    return xv;
  };
  for (int j = threadIdx.x; j < n0; j += kThreads) {
    const int k = cpos(j);
    const double cs = colscale[k];
    Q.col_value[j] = xval(j);
    const double a = sp[k] * cs, b = sn[k] * cs;
    double d = a - b;
    d *= sense;
    Q.col_dual[j] = d;
  }
  for (int i = threadIdx.x; i < m; i += kThreads) {
    const int r = rpos(P.row_new_idx[i]);
    double d = conv ? y[r] : 0.0;
    if (scaled) d /= rowscale[r];
    Q.row_dual[i] = P.row_class[i] == kLeq ? -d : d;
    double s = 0.0;   // A x along the caller's row: columns ascending, then stored order
    for (int q = H.optr[i]; q < H.optr[i + 1]; q++) {
      const int p = H.opos[q];
      s += P.a_value[p] * xval(P.pcol[p]);
    }
    Q.row_value[i] = s;
  }
}

}  // namespace
}  // namespace b200
