// highs_b200/csrc/batch_tree_prep.cu -- the device prologue and postsolve of the tree members of
// b200pdlp_solve_hipdlp_batch_mixed_device (engine_batch.cu solve_hipdlp_batch_device): one CTA of kThreads threads
// per member, and no CTA waits on another, so any number of members runs.  After hip_batch_size_kernel (batch_prep.cu):
//
//   hip_tree_plan_kernel   make_perm of the form's rows and columns (stable sorts by descending length in windows of
//                          kSortWindow that never straddle neq), their inverses, and plan_sell of A and A' (slice
//                          descriptors, long rows, segments): what the host needs to lay out the bodies and the scratch
//   hip_tree_form_kernel   formulate_hipdlp, the row-major indexes, scale_hipdlp (hip_form.cuh hip_form), in standard-form
//                          order
//   hip_tree_fill_kernel   the seven data vectors gathered into device order, and the tree sliced-ELL bodies and long-row
//                          arrays of A and A'
//   hip_tree_post_kernel   hip_host_postsolve of the returned iterate, its device-order vectors read through cinv / rinv
//
// Bits: every value is that of build_layout(f, 0, 1, -1) (host_prep.cpp make_perm / plan_sell / build_sell) after
// formulate_hipdlp / scale_hipdlp, packed as solve_hipdlp_batch packs a tree member.  The orderings and plans are integer
// work; the formulate and scale steps are hip_batch_prep_kernel's (hip_form.cuh hip_form), in standard-form order.  An
// unsorted column is ordered by (new row, value key, stored index) as there; one longer than kTreeSortTile entries in
// O(len log len): tiles of kTreeSortTile entries ranked in shared memory, then merged.
#include <cub/block/block_radix_sort.cuh>

#include "hip_form.cuh"

namespace b200 {
namespace {

constexpr int kSortItems = kSortWindow / kThreads;   // keys per thread of one window's radix sort
static_assert(kSortItems * kThreads == kSortWindow, "one window per CTA-wide sort");

// make_perm over [b, e): windows of kSortWindow from b, each stably sorted by descending len(); writes perm[b, e) and inv
template <class Len, class Sort>
__device__ void window_sort(int b, int e, int bits, Len len, int* perm, int* inv, typename Sort::TempStorage& tmp) {
  for (int w0 = b; w0 < e; w0 += kSortWindow) {
    const int we = min(w0 + kSortWindow, e);
    unsigned keys[kSortItems];
    int vals[kSortItems];
#pragma unroll
    for (int u = 0; u < kSortItems; u++) {   // blocked: thread t holds positions t * kSortItems + u, so ties keep their order
      const int r = w0 + threadIdx.x * kSortItems + u;
      keys[u] = r < we ? (unsigned)len(r) + 1u : 0u;   // 0: past the window, sorted last
      vals[u] = r;
    }
    Sort(tmp).SortDescending(keys, vals, 0, bits);
#pragma unroll
    for (int u = 0; u < kSortItems; u++) {
      const int k = w0 + threadIdx.x * kSortItems + u;
      if (k < we) { perm[k] = vals[u]; inv[vals[u]] = k; }
    }
    __syncthreads();
  }
}

// plan_sell of one matrix with `rows` rows taken in perm order (len(form row)), rows longer than kTreeLongRow masked and cut
// into segments.  Writes the slice descriptors {ptr, len, skipmask, 0} and the long rows' descriptors (at most cap each);
// returns through the last arguments the padded total, the counts and lcount (sm: kThreads + 1 ints, sl: 3 (kThreads + 1)
// long longs of shared memory).
template <class Len>
__device__ void plan_tree(int rows, const int* perm, Len len, int4* slices, int4* segs, int4* longs, int cap, int* sm,
                          long long* sl, int* pad, int* nseg, int* nlong, long long* lcount) {
  const int t = threadIdx.x;
  const int nsl = (rows + 31) / 32;
  for (int s = t; s < nsl; s += kThreads) {
    int mx = 0;
    unsigned mask = 0;
    for (int l = 0; l < 32; l++) {
      const int r = 32 * s + l;
      if (r >= rows) { mask |= 1u << l; continue; }
      const int ln = len(perm[r]);
      if (ln > kTreeLongRow) { mask |= 1u << l; continue; }
      mx = max(mx, ln);
    }
    slices[s] = make_int4(32 * mx, mx, (int)mask, 0);
  }
  __syncthreads();
  *pad = block_scan(reinterpret_cast<int*>(slices), 4, nsl, sm);   // (a slice holds at most 32 kTreeLongRow entries)
  // the long rows in device order: per thread a contiguous chunk of rows, then a scan of (rows, segments, entries)
  const int chunk = (rows + kThreads - 1) / kThreads;
  const int b = min(t * chunk, rows), e = min(b + chunk, rows);
  long long c[3] = {0, 0, 0};
  for (int r = b; r < e; r++) {
    const int ln = len(perm[r]);
    if (ln <= kTreeLongRow) continue;
    c[0] += 1; c[1] += (ln + kNnzPerBlock - 1) / kNnzPerBlock; c[2] += (ln + 3) / 4 * 4;
  }
  for (int k = 0; k < 3; k++) sl[k * (kThreads + 1) + t] = c[k];
  __syncthreads();
  if (t < 3) {
    long long run = 0;
    for (int q = 0; q < kThreads; q++) { const long long v = sl[t * (kThreads + 1) + q]; sl[t * (kThreads + 1) + q] = run; run += v; }
    sl[t * (kThreads + 1) + kThreads] = run;
  }
  __syncthreads();
  int id = (int)sl[t], sg = (int)sl[(kThreads + 1) + t];
  long long base = sl[2 * (kThreads + 1) + t];
  for (int r = b; r < e; r++) {
    const int ln = len(perm[r]);
    if (ln <= kTreeLongRow) continue;
    const int ns = (ln + kNnzPerBlock - 1) / kNnzPerBlock;
    if (id < cap) longs[id] = make_int4(r, sg, ns, sg);
    for (int q = 0; q < ns; q++)
      if (sg + q < cap)
        segs[sg + q] = make_int4(r, (int)base + q * kNnzPerBlock, (int)min(base + (long long)(q + 1) * kNnzPerBlock, base + ln), id);
    id++; sg += ns; base += (ln + 3) / 4 * 4;
  }
  *nlong = (int)sl[kThreads];
  *nseg = (int)sl[(kThreads + 1) + kThreads];
  *lcount = sl[2 * (kThreads + 1) + kThreads] + 8;
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads)
hip_tree_plan_kernel(const BatchPrep* __restrict__ prep, const HipTreePrep* __restrict__ tprep, HipTreePlan* __restrict__ plans) {
  using Sort = cub::BlockRadixSort<unsigned, kThreads, kSortItems, int>;
  __shared__ typename Sort::TempStorage tmp;
  __shared__ int sm[kThreads + 1];
  __shared__ long long sl[3 * (kThreads + 1)];
  __shared__ int maxcol;
  const BatchPrep& P = prep[blockIdx.x];
  const HipTreePrep& T = tprep[blockIdx.x];
  const int t = threadIdx.x, n0 = P.n0, n = P.n, m = P.m, neq = P.neq;
  if (t == 0) maxcol = 0;
  __syncthreads();
  // the form's row lengths (P.rptr from the sizing, before any scan) and column lengths (a slack column has one entry)
  const auto rlen = [&](int r) { return P.rptr[r]; };
  const auto clen = [&](int j) { return j < n0 ? P.a_start[j + 1] - P.a_start[j] : 1; };
  int mc = 0;
  for (int j = t; j < n0; j += kThreads) mc = max(mc, clen(j));
  atomicMax(&maxcol, mc);
  const int bits = 32 - __clz(max(n, m) + 1);   // every key is at most max(n, m) + 1
  window_sort<decltype(rlen), Sort>(0, neq, bits, rlen, T.rperm, T.rinv, tmp);
  window_sort<decltype(rlen), Sort>(neq, m, bits, rlen, T.rperm, T.rinv, tmp);
  window_sort<decltype(clen), Sort>(0, n, bits, clen, T.cperm, T.cinv, tmp);
  HipTreePlan rec;
  plan_tree(m, T.rperm, rlen, P.a_slices, T.a_segs, T.a_long, T.cap, sm, sl, &rec.pad_a, &rec.nseg_a, &rec.nlong_a, &rec.lcount_a);
  plan_tree(n, T.cperm, clen, P.at_slices, T.at_segs, T.at_long, T.cap, sm, sl, &rec.pad_at, &rec.nseg_at, &rec.nlong_at,
            &rec.lcount_at);
  if (t == 0) {
    const bool big = rec.pad_a < 0 || rec.pad_a > 2000000000 || rec.pad_at < 0 || rec.pad_at > 2000000000 ||
                     rec.lcount_a > 2000000008ll || rec.lcount_at > 2000000008ll;
    const bool over = rec.nseg_a > T.cap || rec.nlong_a > T.cap || rec.nseg_at > T.cap || rec.nlong_at > T.cap;
    rec.err = big || over ? 1 : 0;
    rec.maxcol = maxcol;
    plans[blockIdx.x] = rec;
  }
}

// a value_key back to its double
__device__ __forceinline__ double key_value(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

__device__ __forceinline__ bool rec_less(const HipSortRec& a, const HipSortRec& b) {
  return a.row < b.row || (a.row == b.row && (a.key < b.key || (a.key == b.key && a.idx < b.idx)));
}

// Column j (len > kTreeSortTile entries, stored at p0 = a_start[j]) sorted into the form by (new row, value key, stored
// index): tiles ranked by hip_rank_entries into srt[0, len), then pairwise merges of sorted runs between srt[0, len) and
// srt[len, 2 len).  Every key is distinct (the stored index is part of it), so an entry's place in a merged run is its
// place in its own run plus the number of smaller entries in the other run.
__device__ __forceinline__ void sort_long_column(const BatchPrep& P, const HipTreePrep& T, int j, int* s_row, unsigned long long* s_key) {
  const int p0 = P.a_start[j], len = P.a_start[j + 1] - p0;
  HipSortRec* src = T.srt;
  HipSortRec* dst = T.srt + len;
  for (int k0 = 0; k0 < len; k0 += kTreeSortTile)
    hip_rank_entries(P, j, k0, min(k0 + kTreeSortTile, len), s_row, s_key,
                     [&](int rank, int k, int row, double, unsigned long long key) {
                       HipSortRec r;
                       r.row = row; r.idx = k; r.key = key;
                       src[k0 + rank] = r;
                     });
  __syncthreads();
  for (int width = kTreeSortTile; width < len; width *= 2) {
    for (int e = threadIdx.x; e < len; e += kThreads) {
      const int run = e / width, own = run * width;
      const int pb = (run ^ 1) * width, pe = min(pb + width, len);
      const HipSortRec r = src[e];
      int cnt = 0;
      if (pb < len) {   // entries of the other run below r: a binary search
        int lo = pb, hi = pe;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (rec_less(src[mid], r)) lo = mid + 1; else hi = mid;
        }
        cnt = lo - pb;
      }
      dst[(run & ~1) * width + (e - own) + cnt] = r;
    }
    __syncthreads();
    HipSortRec* sw = src; src = dst; dst = sw;
  }
  for (int e = threadIdx.x; e < len; e += kThreads) {
    const HipSortRec r = src[e];
    P.cidx[p0 + e] = r.row; P.cval[p0 + e] = key_value(r.key); P.pcol[p0 + e] = j;
  }
  __syncthreads();
}

// One tree sliced-ELL body (fill_sell_host with the plan's descriptors): device row r is the form's row perm[r], its entries
// entry(form row, k) for k < len(form row) -> (column id, value); masked lanes and padding (0, 0); 32 zeros after the last
// slice.  Then each long row's entries at its first segment's nnz_begin in lcol / lval (the rest zeroed by the host).
template <class Len, class Entry>
__device__ __forceinline__ void tree_body(int rows, const int* perm, const int4* slices, int* col, double* val, int pad, int nlong,
                          const int4* longs, const int4* segs, int* lcol, double* lval, Len len, Entry entry) {
  const int nsl = (rows + 31) / 32;
  for (int r = threadIdx.x; r < 32 * nsl; r += kThreads) {
    const int4 d = slices[r >> 5];
    const size_t base = (size_t)d.x + (r & 31);
    int k = 0;
    if (!(((unsigned)d.z >> (r & 31)) & 1u)) {
      const int fr = perm[r], ln = len(fr);
      for (; k < ln; k++) entry(fr, k, col + base + 32 * (size_t)k, val + base + 32 * (size_t)k);
    }
    for (; k < d.y; k++) { col[base + 32 * (size_t)k] = 0; val[base + 32 * (size_t)k] = 0.0; }
  }
  for (int q = threadIdx.x; q < 32; q += kThreads) { col[(size_t)pad + q] = 0; val[(size_t)pad + q] = 0.0; }
  for (int id = 0; id < nlong; id++) {
    const int4 lr = longs[id];
    const int fr = perm[lr.x], ln = len(fr);
    const size_t b = (size_t)segs[lr.y].y;
    for (int k = threadIdx.x; k < ln; k += kThreads) entry(fr, k, lcol + b + k, lval + b + k);
  }
}

// the form's data vectors in standard-form order: built in slots the rounds start from zero, then gathered into device order
__device__ __forceinline__ HipFormVecs std_order_vecs(const BatchPrep& P) {
  using V = HipBatchVec;
  const int n = P.n, m = P.m;
  double* v = P.vec;
  HipFormVecs F;
  F.cost = V::col(v, n, V::kX); F.lower = V::col(v, n, V::kXa); F.upper = V::col(v, n, V::kXn); F.colscale = V::col(v, n, V::kRx);
  F.rlo = V::row(v, n, m, V::kY); F.rup = V::row(v, n, m, V::kYa); F.rowscale = V::row(v, n, m, V::kYn);
  return F;
}

// formulate_hipdlp, the row-major indexes and scale_hipdlp (hip_form.cuh hip_form), in standard-form order; a listed column
// longer than kTreeSortTile is sorted by sort_long_column.
// (__maxnreg__ instead of __launch_bounds__: under the latter ptxas keeps this kernel at 64 registers and spills.)
__global__ void __maxnreg__(96)
hip_tree_form_kernel(const BatchPrep* __restrict__ prep, const HipBatchPrep* __restrict__ hprep,
                     const HipTreePrep* __restrict__ tprep, int scaling_mode, int ruiz_iterations) {
  __shared__ int sm[kThreads + 1];
  const BatchPrep& P = prep[blockIdx.x];
  const HipTreePrep& T = tprep[blockIdx.x];
  hip_form(P, hprep[blockIdx.x], std_order_vecs(P), scaling_mode, ruiz_iterations, sm,
           [&](int j, int len, int* s_row, unsigned long long* s_key) {
             if (len <= kTreeSortTile) return false;
             sort_long_column(P, T, j, s_row, s_key);
             return true;
           });
}

// the seven data vectors gathered into device order, and the tree layouts of A and A'
__global__ void __launch_bounds__(kThreads)
hip_tree_fill_kernel(const BatchPrep* __restrict__ prep, const HipTreePrep* __restrict__ tprep,
                     const HipTreePlan* __restrict__ plans) {
  const BatchPrep& P = prep[blockIdx.x];
  const HipTreePrep& T = tprep[blockIdx.x];
  const HipTreePlan& Z = plans[blockIdx.x];
  const int t = threadIdx.x, n = P.n, m = P.m;
  using V = HipBatchVec;
  double* v = P.vec;
  const HipFormVecs F = std_order_vecs(P);
  // ---- the seven data vectors in device order (upload_pools' packing), the standard-order slots zeroed again
  for (int k = t; k < n; k += kThreads) {
    const int c = T.cperm[k];
    V::col(v, n, V::kCost)[k] = F.cost[c];
    V::col(v, n, V::kLower)[k] = F.lower[c];
    V::col(v, n, V::kUpper)[k] = F.upper[c];
    V::col(v, n, V::kColscale)[k] = F.colscale[c];
  }
  for (int k = t; k < m; k += kThreads) {
    const int r = T.rperm[k];
    V::row(v, n, m, V::kRlo)[k] = F.rlo[r];
    V::row(v, n, m, V::kRup)[k] = F.rup[r];
    V::row(v, n, m, V::kRowscale)[k] = F.rowscale[r];
  }
  __syncthreads();
  for (int k = t; k < n; k += kThreads) { F.cost[k] = 0.0; F.lower[k] = 0.0; F.upper[k] = 0.0; F.colscale[k] = 0.0; }
  for (int k = t; k < m; k += kThreads) { F.rlo[k] = 0.0; F.rup[k] = 0.0; F.rowscale[k] = 0.0; }

  // ---- the tree layouts (build_sell): A's device rows are form rows rperm[.], entries in row-major order, columns through
  // cinv; A''s device rows are columns cperm[.], entries in cbeg order (sorted by row), rows through rinv
  tree_body(m, T.rperm, P.a_slices, P.a_col, P.a_val, Z.pad_a, Z.nlong_a, T.a_long, T.a_segs, T.a_lcol, T.a_lval,
            [&](int r) { return P.rptr[r + 1] - P.rptr[r]; },
            [&](int r, int k, int* c, double* x) { const int p = P.rpos[P.rptr[r] + k]; *c = T.cinv[P.pcol[p]]; *x = P.cval[p]; });
  tree_body(n, T.cperm, P.at_slices, P.at_col, P.at_val, Z.pad_at, Z.nlong_at, T.at_long, T.at_segs, T.at_lcol, T.at_lval,
            [&](int j) { return P.cbeg[j + 1] - P.cbeg[j]; },
            [&](int j, int k, int* c, double* x) { const int p = P.cbeg[j] + k; *c = T.rinv[P.cidx[p]]; *x = P.cval[p]; });
}

__global__ void __launch_bounds__(kThreads)
hip_tree_post_kernel(const BatchPrep* __restrict__ prep, const HipBatchPrep* __restrict__ hprep,
                     const HipTreePrep* __restrict__ tprep, const HipBatchPost* __restrict__ post, int scaled) {
  const HipTreePrep& T = tprep[blockIdx.x];
  hip_postsolve(prep[blockIdx.x], hprep[blockIdx.x], post[blockIdx.x], scaled, [&](int j) { return T.cinv[j]; },
                [&](int r) { return T.rinv[r]; });
}

}  // namespace

void launch_hip_tree_plan(cudaStream_t s, int count, const BatchPrep* prep, const HipTreePrep* tprep, HipTreePlan* plans) {
  if (count > 0) hip_tree_plan_kernel<<<count, kThreads, 0, s>>>(prep, tprep, plans);
}
void launch_hip_tree_prep(cudaStream_t s, int count, const BatchPrep* prep, const HipBatchPrep* hprep, const HipTreePrep* tprep,
                          const HipTreePlan* plans, int scaling_mode, int ruiz_iterations) {
  if (count <= 0) return;
  hip_tree_form_kernel<<<count, kThreads, 0, s>>>(prep, hprep, tprep, scaling_mode, ruiz_iterations);
  hip_tree_fill_kernel<<<count, kThreads, 0, s>>>(prep, tprep, plans);
}
void launch_hip_tree_post(cudaStream_t s, int count, const BatchPrep* prep, const HipBatchPrep* hprep, const HipTreePrep* tprep,
                          const HipBatchPost* post, int scaled) {
  if (count > 0) hip_tree_post_kernel<<<count, kThreads, 0, s>>>(prep, hprep, tprep, post, scaled);
}

}  // namespace b200
