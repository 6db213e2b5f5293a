// highs_b200/csrc/batch_prep.cu -- the device prologue and postsolve of the ordered members of the device-array batches:
// b200pdlp_solve_batch_device (engine_batch.cu solve_batch_device) and b200pdlp_solve_hipdlp_batch_device / _mixed_device
// (engine_batch.cu solve_hipdlp_batch_device).  One CTA per member, and no CTA waits on another, so any number of members runs.
//
//   batch_size_kernel       check_lp(deep) on the device, formulate's row classes and row order, the standard form's
//                           dimensions and the padded lengths of its ordered sliced-ELL layouts: what the host needs to lay
//                           out the pools
//   batch_prep_kernel       formulate, the row-major index, scale, the sliced-ELL bodies of A and A', host_start_point,
//                           xSum = proj(0) and the sums that set the tolerances and beta
//   batch_post_kernel       host_postsolve of the returned iterate, into the caller's device vectors
//   hip_batch_size_kernel   batch_size_kernel under formulate_hipdlp's row classes (every HiPDLP member, tree members too)
//   hip_batch_prep_kernel   hip_form.cuh hip_form (formulate_hipdlp, the row-major indexes of the form and of the caller's
//                           matrix, scale_hipdlp, |c|^2 and |b|^2 of the unscaled form), then the sliced-ELL bodies of A and A'
//   hip_batch_post_kernel   hip_host_postsolve of the returned iterate, into the caller's device vectors
//   lp_size_kernel          check_lp(deep) and the slack rows of ONE LP of any size, grid-wide: what
//                           b200pdlp_solve_device / _hipdlp_device need to choose their route (engine.cu device_lp_route)
//
// Bits: every value is the host prologue's (host_prep.cpp formulate / build_row_index / scale / build_layout,
// host_prep_hipdlp.cpp formulate_hipdlp / scale_hipdlp, engine.cu host_start_point / host_postsolve, engine_hipdlp.cu
// hip_host_postsolve) with the same operations on the same operands: the build compiles this file with -fmad=false and IEEE
// division and square root.  Maxima are order-free; every sum is taken in the host's order -- a row's 1-norm column-ascending
// by the thread that owns the row, |c|^2 and |b|^2 in index order by one thread.
#include "batch_kernels.hpp"
#include "batch_prep.hpp"
#include "hip_form.cuh"
#include "host_prep.hpp"
#include "row_index.cuh"

namespace b200 {
namespace {

// (block_scan and row_walk, which build the row-major indexes: row_index.cuh; kInf and the HiPDLP prologue's pieces:
// hip_form.cuh)

// max over the CTA with std::max's comparison ((a < b) ? b : a); result in every thread
__device__ double block_max(double v, double* sm) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int o = 16; o > 0; o >>= 1) { const double u = __shfl_down_sync(0xffffffffu, v, o); v = (v < u) ? u : v; }
  if (lane == 0) sm[wid] = v;
  __syncthreads();
  double r = sm[0];
  for (int w = 1; w < kThreads / 32; w++) r = (r < sm[w]) ? sm[w] : r;
  __syncthreads();
  return r;
}

__device__ __forceinline__ double lower_inf(double v) { return v < -1e20 ? -kInf : v; }   // formulate's bound rule
__device__ __forceinline__ double upper_inf(double v) { return v > 1e20 ? kInf : v; }

__device__ __forceinline__ double project(double v, double lo, double up) {   // PDHG_Project_Bounds: upper first
  v = v < up ? v : up;
  v = v > lo ? v : lo;
  return v;
}

// the padded length of an ordered sliced-ELL layout: rows of length len(r), r < rows, 32 rows a slice
template <class Len>
__device__ long long padded(int rows, Len len, unsigned long long* acc) {
  if (threadIdx.x == 0) *acc = 0ull;
  __syncthreads();
  unsigned long long mine = 0;
  for (int s = threadIdx.x; s < (rows + 31) / 32; s += kThreads) {
    int mx = 0;
    for (int r = 32 * s; r < min(32 * s + 32, rows); r++) mx = max(mx, len(r));
    mine += 32ull * (unsigned long long)mx;
  }
  atomicAdd(acc, mine);
  __syncthreads();
  const long long total = (long long)*acc;
  __syncthreads();
  return total;
}

// formulate's row classes (host_prep.cpp formulate): +-1e20 thresholds; ranged and free rows are BOUND rows
struct PdlpRows {
  __device__ static int row_class(double rl, double ru) {
    const bool lo = rl > -1e20, up = ru < 1e20;
    int c;
    if (lo && up && rl == ru) c = kEq;
    else if (lo && !up) c = kGeq;
    else if (!lo && up) c = kLeq;
    else c = kBound;
    return c;
  }
};
// formulate_hipdlp's row classes: +-infinity thresholds (a bound of 1e25 is finite), FREE rows a class of their own
struct HipRows {
  __device__ static int row_class(double rl, double ru) {
    const bool lo = rl > -kInf, up = ru < kInf;
    int c;
    if (lo && up) c = (rl == ru) ? kEq : kBound;
    else if (lo) c = kGeq;
    else if (up) c = kLeq;
    else c = kFreeRow;
    return c;
  }
};

// check_lp(deep)'s rules, one entry at a time, for every sizing kernel (batch_size per CTA, lp_size_kernel over a grid):
// a_start[0] == 0, a_start non-decreasing, a_index in [0, num_row).  (The fourth, a_index and a_value present when
// a_start[num_col] > 0, stays written out in both: as a function it changes batch_size's code.)
__device__ __forceinline__ bool start_bad(const BatchPrep& P) { return P.a_start[0] != 0; }
__device__ __forceinline__ bool descent_at(const BatchPrep& P, int j) { return P.a_start[j + 1] < P.a_start[j]; }
__device__ __forceinline__ bool index_bad(const BatchPrep& P, int p) { return (unsigned)P.a_index[p] >= (unsigned)P.m; }
// a row of class c has a slack column in the standard form
__device__ __forceinline__ bool has_slack(int c) { return c == kBound || c == kFreeRow; }

// check_lp(deep), the row classes under Rows, the row order, the standard form's dimensions and the padded lengths of its
// ordered layouts, for one member.  BOUND and FREE rows are equality-like, each with a slack column (PdlpRows makes no FREE
// rows).
template <class Rows>
__device__ __forceinline__ void batch_size(const BatchPrep& P, BatchSize& S) {
  __shared__ int flag[4];
  __shared__ int sm_eq[kThreads + 1], sm_bnd[kThreads + 1];
  __shared__ unsigned long long acc;
  const int t = threadIdx.x, n0 = P.n0, m = P.m;
  if (t < 4) flag[t] = 0;
  __syncthreads();
  if (t == 0 && start_bad(P)) flag[0] = kPrepStart0;
  for (int j = t; j < n0; j += kThreads)
    if (descent_at(P, j)) flag[1] = kPrepDecreasing;
  __syncthreads();
  const int nnz0 = P.a_start[n0];
  if (t == 0 && nnz0 > 0 && (!P.a_index || !P.a_value)) flag[2] = kPrepNull;
  __syncthreads();
  const int early = flag[0] ? flag[0] : flag[1] ? flag[1] : flag[2];
  if (early) {
    if (t == 0) S.err = early;
    return;
  }
  for (int p = t; p < nnz0; p += kThreads)
    if (index_bad(P, p)) flag[3] = kPrepIndex;
  __syncthreads();
  if (flag[3]) {
    if (t == 0) S.err = kPrepIndex;
    return;
  }
  for (int i = t; i < m; i += kThreads) {
    const double rl = P.row_lower[i], ru = P.row_upper[i];
    P.row_class[i] = Rows::row_class(rl, ru);
  }
  for (int i = t; i <= m; i += kThreads) P.rptr[i] = 0;
  __syncthreads();
  // the new row order: equality-like rows (EQ / BOUND / FREE) first, then LEQ / GEQ, each in original order;
  // slack columns in the order of their rows
  const int chunk = (m + kThreads - 1) / kThreads;
  const int b = min(t * chunk, m), e = min(b + chunk, m);
  int eq = 0, bnd = 0;
  for (int i = b; i < e; i++) {
    const int c = P.row_class[i];
    eq += (c == kEq || c == kBound || c == kFreeRow);
    bnd += has_slack(c);
  }
  sm_eq[t] = eq; sm_bnd[t] = bnd;
  __syncthreads();
  if (t == 0) {
    int re = 0, rb = 0;
    for (int k = 0; k < kThreads; k++) {
      const int ve = sm_eq[k], vb = sm_bnd[k];
      sm_eq[k] = re; sm_bnd[k] = rb;
      re += ve; rb += vb;
    }
    sm_eq[kThreads] = re; sm_bnd[kThreads] = rb;
  }
  __syncthreads();
  const int neq = sm_eq[kThreads], nb = sm_bnd[kThreads];
  {
    int head = sm_eq[t], tail = neq + (b - sm_eq[t]), sl = sm_bnd[t];
    for (int i = b; i < e; i++) {
      const int c = P.row_class[i];
      P.row_new_idx[i] = (c == kEq || c == kBound || c == kFreeRow) ? head++ : tail++;
      P.slack[i] = (c == kBound || c == kFreeRow) ? sl++ : -1;
    }
  }
  __syncthreads();
  // the standard form's row lengths (integer counts: order-free), a slack row's slack entry included
  for (int p = t; p < nnz0; p += kThreads) atomicAdd(&P.rptr[P.row_new_idx[P.a_index[p]]], 1);
  for (int i = t; i < m; i += kThreads)
    if (P.slack[i] >= 0) atomicAdd(&P.rptr[P.row_new_idx[i]], 1);
  __syncthreads();
  const long long pa = padded(m, [&](int r) { return P.rptr[r]; }, &acc);
  const long long pat = padded(n0 + nb, [&](int j) { return j < n0 ? P.a_start[j + 1] - P.a_start[j] : 1; }, &acc);
  if (t == 0) {
    S.err = kPrepOk;
    S.n = n0 + nb; S.nnz = nnz0 + nb; S.neq = neq;
    // (ordered_max keeps these far below 2^31; the host checks the dimensions before it trusts them)
    S.pad_a = (int)min(pa, 2000000000ll); S.pad_at = (int)min(pat, 2000000000ll);
  }
}

__global__ void __launch_bounds__(kThreads) batch_size_kernel(const BatchPrep* __restrict__ prep, BatchSize* __restrict__ sizes) {
  batch_size<PdlpRows>(prep[blockIdx.x], sizes[blockIdx.x]);
}

__global__ void __launch_bounds__(kThreads) hip_batch_size_kernel(const BatchPrep* __restrict__ prep, BatchSize* __restrict__ sizes) {
  batch_size<HipRows>(prep[blockIdx.x], sizes[blockIdx.x]);
}

// check_lp(deep) and the slack rows under Rows of one LP of any size, grid-stride, in two passes over one record zeroed by
// the host.  Pass 0: a_start (a_start[0] == 0 and a_start[num_col] >= 0, no descent), the matrix arrays present, the slack
// rows.  Pass 1, the next launch on the stream: a_index in [0, num_row), only when pass 0 found nothing -- as check_lp, which
// reads a_index only once a_start has passed, so a malformed a_start never sends the sweep past a_index's end.  Every warp
// ORs its broken rules and adds its slack rows with one atomic each.
template <class Rows>
__global__ void __launch_bounds__(kThreads) lp_size_kernel(const BatchPrep P, int index_pass, LpSize* __restrict__ out) {
  const long long stride = (long long)gridDim.x * kThreads, t = (long long)blockIdx.x * kThreads + threadIdx.x;
  const int n0 = P.n0, m = P.m, nnz0 = P.a_start[n0];
  unsigned bits = 0;
  int slack = 0;
  if (index_pass) {
    if (out->err_bits) return;
    for (long long p = t; p < nnz0; p += stride)
      if (index_bad(P, (int)p)) bits |= 1u << kPrepIndex;
  } else {
    if (t == 0) {
      if (start_bad(P) || nnz0 < 0) bits |= 1u << kPrepStart0;
      if (nnz0 > 0 && (!P.a_index || !P.a_value)) bits |= 1u << kPrepNull;
      out->nnz = nnz0;
    }
    for (long long j = t; j < n0; j += stride)
      if (descent_at(P, (int)j)) bits |= 1u << kPrepDecreasing;
    for (long long i = t; i < m; i += stride) slack += has_slack(Rows::row_class(P.row_lower[i], P.row_upper[i]));
  }
  bits = __reduce_or_sync(0xffffffffu, bits);
  slack = __reduce_add_sync(0xffffffffu, slack);
  if ((threadIdx.x & 31) == 0) {
    if (bits) atomicOr(&out->err_bits, bits);
    if (slack) atomicAdd(&out->nslack, slack);
  }
}

// one ordered sliced-ELL body: rows r < rows, 32 a slice, entry k of row r at ptr + 32 k + (r & 31); padding (0, 0), and 32
// zero entries after the last slice (fill_sell_host).  The slice descriptors {ptr, len, skipmask, 0} are written first.
template <class Len, class Entry>
__device__ void sell_body(int rows, int4* slices, int* col, double* val, int* sm, Len len, Entry entry) {
  const int nsl = (rows + 31) / 32;
  for (int s = threadIdx.x; s < nsl; s += kThreads) {
    int mx = 0;
    unsigned mask = 0;
    for (int l = 0; l < 32; l++) {
      const int r = 32 * s + l;
      if (r >= rows) { mask |= 1u << l; continue; }
      mx = max(mx, len(r));
    }
    slices[s] = make_int4(32 * mx, mx, (int)mask, 0);
  }
  __syncthreads();
  const int total = block_scan(reinterpret_cast<int*>(slices), 4, nsl, sm);
  for (int r = threadIdx.x; r < 32 * nsl; r += kThreads) {
    const int4 d = slices[r >> 5];
    const size_t base = (size_t)d.x + (r & 31);
    int k = 0;
    if (r < rows) k = entry(r, col + base, val + base);
    for (; k < d.y; k++) { col[base + 32 * (size_t)k] = 0; val[base + 32 * (size_t)k] = 0.0; }
  }
  for (int q = threadIdx.x; q < 32; q += kThreads) { col[(size_t)total + q] = 0; val[(size_t)total + q] = 0.0; }
}

// the ordered sliced-ELL bodies of the form (build_layout, identity orderings, no long rows): A's rows in the row-major
// index's order; A' row j = column j sorted by row, stably (build_col_major)
__device__ __forceinline__ void form_layouts(const BatchPrep& P, int m, int n, int* sm) {
  sell_body(m, P.a_slices, P.a_col, P.a_val, sm, [&](int r) { return P.rptr[r + 1] - P.rptr[r]; },
            [&](int r, int* c, double* v) {
              const int q0 = P.rptr[r], len = P.rptr[r + 1] - q0;
              for (int k = 0; k < len; k++) { const int p = P.rpos[q0 + k]; c[32 * k] = P.pcol[p]; v[32 * k] = P.cval[p]; }
              return len;
            });
  __syncthreads();
  sell_body(n, P.at_slices, P.at_col, P.at_val, sm, [&](int j) { return P.cbeg[j + 1] - P.cbeg[j]; },
            [&](int j, int* c, double* v) {
              const int p0 = P.cbeg[j], len = P.cbeg[j + 1] - p0;
              bool sorted = true;
              for (int k = 0; k < len; k++) {
                c[32 * k] = P.cidx[p0 + k]; v[32 * k] = P.cval[p0 + k];
                if (k > 0 && P.cidx[p0 + k] < P.cidx[p0 + k - 1]) sorted = false;
              }
              if (!sorted)   // stable insertion sort by row
                for (int k = 1; k < len; k++) {
                  const int ck = c[32 * k];
                  const double vk = v[32 * k];
                  int h = k - 1;
                  for (; h >= 0 && c[32 * h] > ck; h--) { c[32 * (h + 1)] = c[32 * h]; v[32 * (h + 1)] = v[32 * h]; }
                  c[32 * (h + 1)] = ck; v[32 * (h + 1)] = vk;
                }
              return len;
            });
}

__global__ void __launch_bounds__(kThreads) batch_prep_kernel(const BatchPrep* __restrict__ prep, int do_scale) {
  __shared__ int sm[kThreads + 1];
  __shared__ double smd[kThreads / 32];
  const BatchPrep& P = prep[blockIdx.x];
  const int t = threadIdx.x, wid = t >> 5;
  const int n0 = P.n0, m = P.m, n = P.n, nnz = P.nnz;
  const int nnz0 = nnz - (n - n0);
  const double sense = P.sense;
  using V = BatchVec;
  double* cost = V::col(P.vec, n, V::kCost);
  double* lower = V::col(P.vec, n, V::kLower);
  double* upper = V::col(P.vec, n, V::kUpper);
  double* colscale = V::col(P.vec, n, V::kColscale);
  double* x0 = V::col(P.vec, n, V::kX0);
  double* xsum = V::col(P.vec, n, V::kXsum);
  double* rhs = V::row(P.vec, n, m, V::kRhs);
  double* rowscale = V::row(P.vec, n, m, V::kRowscale);
  double* y0 = V::row(P.vec, n, m, V::kY0);
  const int* rni = P.row_new_idx;
  const int* rcl = P.row_class;

  // ---- formulate: within a structural column EQ / BOUND entries first, then LEQ (negated) / GEQ; one -1 slack column per
  // BOUND row; c *= sense; bounds beyond +-1e20 -> +-inf (host_prep.cpp formulate)
  for (int j = t; j < n0; j += kThreads) {
    int k = P.a_start[j];
    P.cbeg[j] = k;
    for (int p = P.a_start[j]; p < P.a_start[j + 1]; p++) {
      const int i = P.a_index[p], c = rcl[i];
      if (c == kEq || c == kBound) { P.cidx[k] = rni[i]; P.cval[k] = P.a_value[p]; P.pcol[k] = j; k++; }
    }
    for (int p = P.a_start[j]; p < P.a_start[j + 1]; p++) {
      const int i = P.a_index[p], c = rcl[i];
      if (c == kLeq) { P.cidx[k] = rni[i]; P.cval[k] = -P.a_value[p]; P.pcol[k] = j; k++; }
      else if (c == kGeq) { P.cidx[k] = rni[i]; P.cval[k] = P.a_value[p]; P.pcol[k] = j; k++; }
    }
    cost[j] = P.col_cost[j] * sense;
    lower[j] = lower_inf(P.col_lower[j]);
    upper[j] = upper_inf(P.col_upper[j]);
    colscale[j] = 1.0;
  }
  for (int i = t; i < m; i += kThreads) {
    const int r = rni[i], c = rcl[i];
    rhs[r] = c == kEq ? P.row_lower[i] : c == kBound ? 0.0 : c == kLeq ? -P.row_upper[i] : P.row_lower[i];
    rowscale[r] = 1.0;
    if (c == kBound) {
      const int j = n0 + P.slack[i], q = nnz0 + P.slack[i];
      P.cbeg[j] = q; P.cidx[q] = r; P.cval[q] = -1.0; P.pcol[q] = j;
      cost[j] = 0.0;
      lower[j] = lower_inf(P.row_lower[i]);
      upper[j] = upper_inf(P.row_upper[i]);
      colscale[j] = 1.0;
    }
  }
  if (t == 0) P.cbeg[n] = nnz;
  // ---- the row-major index (build_row_index): positions p ascending (= columns ascending) within each row
  const int rtotal = block_scan(P.rptr, 1, m, sm);   // (its first barrier also orders the formulate writes above)
  if (t == 0) P.rptr[m] = rtotal;
  for (int i = t; i < m; i += kThreads) P.rwork[i] = P.rptr[i];
  __syncthreads();
  if (wid == 0) {
    row_walk(nnz, P.cidx, P.rwork, P.rpos);
  } else if (t == 32 || t == 64) {   // |c|^2 and |b|^2 of the unscaled form, index order (formulate's norms, squared)
    const double* v = t == 32 ? cost : rhs;
    const int len = t == 32 ? n : m;
    double s = 0.0;
    for (int q = 0; q < len; q++) s += v[q] * v[q];
    P.rec[t == 32 ? kRecCostSq : kRecRhsSq] = s;
  }
  __syncthreads();

  // ---- scale: 10 Ruiz passes, then Pock-Chambolle (host_prep.cpp scale)
  double am = 0.0;
  if (do_scale) {
    for (int j = t; j < n; j += kThreads) {
      double mx = 0.0;
      for (int p = P.cbeg[j]; p < P.cbeg[j + 1]; p++) { const double a = fabs(P.cval[p]); if (a > mx) mx = a; }
      P.cs[j] = mx;
    }
    for (int i = t; i < m; i += kThreads) {
      double r = 0.0;
      for (int q = P.rptr[i]; q < P.rptr[i + 1]; q++) { const double a = fabs(P.cval[P.rpos[q]]); if (r < a) r = a; }
      P.rs[i] = r;
    }
    __syncthreads();
    double* cs = P.cs;
    double* cs_next = P.cs_next;
    const int kRuiz = 10;
    for (int it = 0; it <= kRuiz; it++) {
      for (int j = t; j < n; j += kThreads) {
        const double v = sqrt(cs[j]);
        const double c = (v == 0.0) ? 1.0 : v;
        cs[j] = c;
        cost[j] /= c; lower[j] *= c; upper[j] *= c; colscale[j] *= c;
      }
      for (int i = t; i < m; i += kThreads) {
        const double r = (P.rs[i] == 0.0) ? 1.0 : sqrt(P.rs[i]);
        P.rs[i] = r;
        rhs[i] /= r; rowscale[i] *= r;
      }
      __syncthreads();
      const bool next_is_pc = it == kRuiz - 1, last = it == kRuiz;
      for (int j = t; j < n; j += kThreads) {
        double acc = 0.0;
        const double cj = cs[j];
        for (int p = P.cbeg[j]; p < P.cbeg[j + 1]; p++) {
          double v = P.cval[p] / P.rs[P.cidx[p]];   // row division first, then column division
          v /= cj;
          P.cval[p] = v;
          const double a = fabs(v);
          if (last) { if (a > am) am = a; }
          else if (next_is_pc) { acc += a; }
          else { if (a > acc) acc = a; }
        }
        cs_next[j] = acc;
      }
      __syncthreads();
      if (last) break;
      for (int i = t; i < m; i += kThreads) {
        double r = 0.0;
        for (int q = P.rptr[i]; q < P.rptr[i + 1]; q++) {
          const double a = fabs(P.cval[P.rpos[q]]);
          if (next_is_pc) r += a;
          else if (r < a) r = a;
        }
        P.rs[i] = r;
      }
      double* sw = cs; cs = cs_next; cs_next = sw;
      __syncthreads();
    }
  } else {
    for (int p = t; p < nnz; p += kThreads) { const double a = fabs(P.cval[p]); am = (am < a) ? a : am; }
  }
  const double amax = block_max(am, smd);

  // ---- the ordered sliced-ELL bodies
  form_layouts(P, m, n, sm);

  // ---- the start point (engine.cu host_start_point) and xSum = proj(0)
  const bool warm = P.warm_x && P.warm_rv && P.warm_rd;
  if (warm) {
    for (int j = t; j < n0; j += kThreads) x0[j] = P.warm_x[j];
    for (int i = t; i < m; i += kThreads) {
      const double mu = rcl[i] == kLeq ? -1 : 1;
      y0[rni[i]] = sense * mu * P.warm_rd[i];
      if (rcl[i] == kBound) x0[n0 + P.slack[i]] = P.warm_rv[i];
    }
    __syncthreads();
  }
  for (int j = t; j < n; j += kThreads) {
    const double v = warm ? x0[j] * colscale[j] : 0.0;
    x0[j] = project(v, lower[j], upper[j]);
    xsum[j] = project(0.0, lower[j], upper[j]);
  }
  for (int i = t; i < m; i += kThreads) y0[i] = warm ? y0[i] * rowscale[i] : 0.0;
  // ---- |c|^2 and |b|^2 of the scaled form in index order (what sets beta), amax
  if (t == 0 || t == 32) {
    const double* v = t == 0 ? cost : rhs;
    const int len = t == 0 ? n : m;
    double s = 0.0;
    for (int q = 0; q < len; q++) s += v[q] * v[q];
    P.rec[t == 0 ? kRecScaledCostSq : kRecScaledRhsSq] = s;
    if (t == 0) P.rec[kRecAmax] = amax;
  }
}

__global__ void __launch_bounds__(kThreads) batch_post_kernel(const BatchPrep* __restrict__ prep, const BatchPost* __restrict__ post) {
  const BatchPrep& P = prep[blockIdx.x];
  const BatchPost& Q = post[blockIdx.x];
  if (!(Q.col_value && Q.col_dual && Q.row_value && Q.row_dual)) return;
  const int n0 = P.n0, m = P.m, n = P.n;
  using V = BatchVec;
  const double* v = P.vec;
  const bool avg = Q.sel == 2;
  const double* dx = V::col(v, n, avg ? V::kXavg : V::kX0 + Q.sel);
  const double* daty = V::col(v, n, avg ? V::kAtyavg : V::kAty0 + Q.sel);
  const double* dy = V::row(v, n, m, avg ? V::kYavg : V::kY0 + Q.sel);
  const double* dax = V::row(v, n, m, avg ? V::kAxavg : V::kAx0 + Q.sel);
  const double *cost = V::col(v, n, V::kCost), *lower = V::col(v, n, V::kLower), *upper = V::col(v, n, V::kUpper);
  const double *colscale = V::col(v, n, V::kColscale), *rowscale = V::row(v, n, m, V::kRowscale);
  const double sense = P.sense;
  for (int j = threadIdx.x; j < n0; j += kThreads) {
    double sp = 0.0, sn = 0.0;
    if (Q.have_check) {   // dSlackPos / dSlackNeg of the returned iterate
      double rc = daty[j] * -1.0;
      rc = rc + 1.0 * cost[j];
      double a = rc > 0.0 ? rc : 0.0;
      a = a * (lower[j] > -kInf ? 1.0 : 0.0);
      double b = rc < 0.0 ? rc : 0.0;
      b = b * -1.0;
      b = b * (upper[j] < kInf ? 1.0 : 0.0);
      sp = a; sn = b;
    }
    const double c = colscale[j];
    const double x = dx[j] / c;
    sp *= c; sn *= c;
    Q.col_value[j] = x;
    const double d = sp - sn;
    Q.col_dual[j] = d * sense;
  }
  for (int i = threadIdx.x; i < m; i += kThreads) {
    const int r = P.row_new_idx[i], c = P.row_class[i];
    double val = dax[r] * rowscale[r];
    if (c == kLeq) val = -val;
    else if (c == kBound) { const int j = n0 + P.slack[i]; val = val + dx[j] / colscale[j]; }
    Q.row_value[i] = val;
    double d = dy[r] / rowscale[r] * sense;
    if (c == kLeq) d = -d;
    Q.row_dual[i] = d;
  }
}

// formulate_hipdlp, the row-major indexes and scale_hipdlp (hip_form.cuh hip_form; every listed column ranked whole), then the
// ordered sliced-ELL bodies (every column is already sorted by row)
__global__ void __launch_bounds__(kThreads, 3)
hip_batch_prep_kernel(const BatchPrep* __restrict__ prep, const HipBatchPrep* __restrict__ hprep, int scaling_mode,
                      int ruiz_iterations) {
  __shared__ int sm[kThreads + 1];
  const BatchPrep& P = prep[blockIdx.x];
  const int m = P.m, n = P.n;
  using V = HipBatchVec;
  HipFormVecs F;
  F.cost = V::col(P.vec, n, V::kCost); F.lower = V::col(P.vec, n, V::kLower); F.upper = V::col(P.vec, n, V::kUpper);
  F.colscale = V::col(P.vec, n, V::kColscale);
  F.rlo = V::row(P.vec, n, m, V::kRlo); F.rup = V::row(P.vec, n, m, V::kRup); F.rowscale = V::row(P.vec, n, m, V::kRowscale);
  hip_form(P, hprep[blockIdx.x], F, scaling_mode, ruiz_iterations, sm, [](auto&&...) { return false; });
  form_layouts(P, m, n, sm);
}

__global__ void __launch_bounds__(kThreads)
hip_batch_post_kernel(const BatchPrep* __restrict__ prep, const HipBatchPrep* __restrict__ hprep,
                      const HipBatchPost* __restrict__ post, int scaled) {
  const auto same = [](int k) { return k; };
  hip_postsolve(prep[blockIdx.x], hprep[blockIdx.x], post[blockIdx.x], scaled, same, same);
}

}  // namespace

void launch_hip_batch_size(cudaStream_t s, int count, const BatchPrep* prep, BatchSize* sizes) {
  if (count > 0) hip_batch_size_kernel<<<count, kThreads, 0, s>>>(prep, sizes);
}
void launch_hip_batch_prep(cudaStream_t s, int count, const BatchPrep* prep, const HipBatchPrep* hprep, int scaling_mode,
                           int ruiz_iterations) {
  if (count > 0) hip_batch_prep_kernel<<<count, kThreads, 0, s>>>(prep, hprep, scaling_mode, ruiz_iterations);
}
void launch_hip_batch_post(cudaStream_t s, int count, const BatchPrep* prep, const HipBatchPrep* hprep,
                           const HipBatchPost* post, int scaled) {
  if (count > 0) hip_batch_post_kernel<<<count, kThreads, 0, s>>>(prep, hprep, post, scaled);
}

void launch_batch_size(cudaStream_t s, int count, const BatchPrep* prep, BatchSize* sizes) {
  if (count > 0) batch_size_kernel<<<count, kThreads, 0, s>>>(prep, sizes);
}
void launch_lp_size(cudaStream_t s, const BatchPrep& lp, bool hip, LpSize* out) {
  for (int pass = 0; pass < 2; pass++) {
    if (hip) lp_size_kernel<HipRows><<<kLpSizeBlocks, kThreads, 0, s>>>(lp, pass, out);
    else lp_size_kernel<PdlpRows><<<kLpSizeBlocks, kThreads, 0, s>>>(lp, pass, out);
  }
}
void launch_batch_prep(cudaStream_t s, int count, const BatchPrep* prep, int do_scale) {
  if (count > 0) batch_prep_kernel<<<count, kThreads, 0, s>>>(prep, do_scale);
}
void launch_batch_post(cudaStream_t s, int count, const BatchPrep* prep, const BatchPost* post) {
  if (count > 0) batch_post_kernel<<<count, kThreads, 0, s>>>(prep, post);
}

}  // namespace b200
