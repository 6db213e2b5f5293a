// highs_b200/csrc/device_prep.cu -- see device_prep.cuh.  Every stage has a host twin in host_prep.cpp that produces the
// same bits (tests/test_gpu_device_prep.py compares them array by array).
#include "device_prep.hpp"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <climits>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "setup_kernels.hpp"

namespace b200 {

// ===================================================================================== block cache
namespace {
struct Block { void* p; size_t bytes; int device; };
struct Cache {
  std::mutex mu;
  std::vector<Block> free_blocks;     // cached, not in use
  std::vector<Block> live;            // handed out
  size_t cached_bytes = 0;
  size_t cap_bytes = [] {
    if (const char* e = getenv("B200PDLP_CACHE_MB")) return (size_t)std::max(0L, atol(e)) << 20;
    return (size_t)16 << 30;
  }();
};
Cache& dcache() { static Cache* c = new Cache; return *c; }
Cache& hcache() { static Cache* c = new Cache; return *c; }
}  // namespace

void* dev_cache_alloc(size_t bytes) {
  bytes = std::max<size_t>((bytes + 511) & ~(size_t)511, 512);
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) throw std::runtime_error("cudaGetDevice failed");
  Cache& c = dcache();
  {
    std::lock_guard<std::mutex> lk(c.mu);
    int best = -1;
    for (int i = 0; i < (int)c.free_blocks.size(); i++) {
      const Block& b = c.free_blocks[i];
      if (b.device != dev || b.bytes < bytes || b.bytes > bytes + bytes / 4 + (1 << 16)) continue;
      if (best < 0 || b.bytes < c.free_blocks[best].bytes) best = i;
    }
    if (best >= 0) {
      Block b = c.free_blocks[best];
      c.free_blocks.erase(c.free_blocks.begin() + best);
      c.cached_bytes -= b.bytes;
      c.live.push_back(b);
      return b.p;
    }
  }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {   // out of memory with blocks parked in the cache: give them back and try once more
    cudaGetLastError();
    dev_cache_release();
    e = cudaMalloc(&p, bytes);
  }
  if (e != cudaSuccess) throw std::runtime_error(std::string("cudaMalloc(") + std::to_string(bytes) + "): " + cudaGetErrorString(e));
  std::lock_guard<std::mutex> lk(c.mu);
  c.live.push_back({p, bytes, dev});
  return p;
}

void dev_cache_free(void* p) {
  if (!p) return;
  Cache& c = dcache();
  Block b{nullptr, 0, 0};
  {
    std::lock_guard<std::mutex> lk(c.mu);
    for (size_t i = 0; i < c.live.size(); i++)
      if (c.live[i].p == p) { b = c.live[i]; c.live[i] = c.live.back(); c.live.pop_back(); break; }
    if (b.p && c.cached_bytes + b.bytes <= c.cap_bytes) {
      c.free_blocks.push_back(b);
      c.cached_bytes += b.bytes;
      return;
    }
  }
  cudaFree(p);   // not ours (or the cache is full)
}

void dev_cache_release() {
  Cache& c = dcache();
  std::vector<Block> blocks;
  {
    std::lock_guard<std::mutex> lk(c.mu);
    blocks.swap(c.free_blocks);
    c.cached_bytes = 0;
  }
  int cur = -1;
  cudaGetDevice(&cur);
  for (const Block& b : blocks) { cudaSetDevice(b.device); cudaFree(b.p); }
  if (cur >= 0) cudaSetDevice(cur);
}

void* pinned_cache_alloc(size_t bytes, bool mapped) {
  bytes = std::max<size_t>((bytes + 4095) & ~(size_t)4095, 4096);
  Cache& c = hcache();
  const int tag = mapped ? 1 : 0;
  {
    std::lock_guard<std::mutex> lk(c.mu);
    for (size_t i = 0; i < c.free_blocks.size(); i++)
      if (c.free_blocks[i].device == tag && c.free_blocks[i].bytes >= bytes && c.free_blocks[i].bytes <= 2 * bytes) {
        Block b = c.free_blocks[i];
        c.free_blocks.erase(c.free_blocks.begin() + i);
        c.live.push_back(b);
        return b.p;
      }
  }
  void* p = nullptr;
  const cudaError_t e = cudaHostAlloc(&p, bytes, mapped ? cudaHostAllocMapped : cudaHostAllocDefault);
  if (e != cudaSuccess) throw std::runtime_error(std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
  std::lock_guard<std::mutex> lk(c.mu);
  c.live.push_back({p, bytes, tag});
  return p;
}
void pinned_cache_free(void* p) {
  if (!p) return;
  Cache& c = hcache();
  std::lock_guard<std::mutex> lk(c.mu);
  for (size_t i = 0; i < c.live.size(); i++)
    if (c.live[i].p == p) { c.free_blocks.push_back(c.live[i]); c.live[i] = c.live.back(); c.live.pop_back(); return; }
  cudaFreeHost(p);
}

// ===================================================================================== kernels
namespace {
constexpr int kTpb = 256;
inline int grid_for(long long work) {
  long long g = (work + kTpb - 1) / kTpb;
  if (g < 1) g = 1;
  return (int)(g > kGridUnit * 32LL ? kGridUnit * 32LL : g);
}
inline int warp_grid(long long rows) { return (int)std::max<long long>(1, (rows * 32 + kTpb - 1) / kTpb); }

// ---- formulateLP_highs, CupdlpWrapper.cpp:280-448 (host twin: host_prep.cpp::formulate)
// row classes with the +-1e20 thresholds (:316-317); eq-like = EQ or BOUND (they come first in the new order).
// hip (HiPDLP mode, pdhg.cc:175-198; host twin formulate_hipdlp): thresholds +-infinity, so a bound of 1e25 is finite, and
// free rows are a class of their own (kFreeRow = 4, eq-like, with a slack column like BOUND rows)
__global__ void __launch_bounds__(kTpb)
classify_rows_kernel(int m, int hip, const double* __restrict__ rl, const double* __restrict__ ru, int* __restrict__ cls,
                     int* __restrict__ eqlike, int* __restrict__ isbound) {
  const int stride = gridDim.x * kTpb;
  const double thr = hip ? INFINITY : 1e20;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < m; i += stride) {
    const bool lo = rl[i] > -thr, up = ru[i] < thr;
    int c;
    if (lo && up && rl[i] == ru[i]) c = 0;      // kEq
    else if (lo && !up) c = 2;                   // kGeq
    else if (!lo && up) c = 1;                   // kLeq
    else if (hip && !lo && !up) c = 4;           // kFreeRow
    else c = 3;                                  // kBound (ranged rows; free rows too outside HiPDLP mode)
    cls[i] = c;
    eqlike[i] = (c == 0 || c >= 3) ? 1 : 0;
    isbound[i] = c >= 3 ? 1 : 0;
  }
}

// new row order: EQ/BOUND rows first (original order), then LEQ/GEQ (:380-404); rhs; slack column of a BOUND row
// (:328-331,367-373,439-445): A x - z = 0, lo <= z <= up
// hip: rup != nullptr receives the row upper bounds (EQ [b, b], GEQ / LEQ [b, inf], BOUND / FREE [0, 0], pdhg.cc:247-270) and
// the slack columns keep the row's bounds unclamped (:235-244)
__global__ void __launch_bounds__(kTpb)
row_maps_kernel(int m, int n0, int nnz0, int neq, const double* __restrict__ rl, const double* __restrict__ ru,
                const int* __restrict__ cls, const int* __restrict__ eq_ex, const int* __restrict__ bd_ex,
                int* __restrict__ new_idx, int* __restrict__ row_old, int* __restrict__ slack_row, double* __restrict__ rhs,
                double* __restrict__ cost, double* __restrict__ lower, double* __restrict__ upper, int* __restrict__ cbeg,
                int* __restrict__ cidx, double* __restrict__ cval, int* __restrict__ colof, double* __restrict__ rup) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < m; i += stride) {
    const int c = cls[i];
    const bool eql = c == 0 || c >= 3;
    const int ni = eql ? eq_ex[i] : neq + (i - eq_ex[i]);
    new_idx[i] = ni;
    row_old[ni] = i;
    double b;
    if (c == 0) b = rl[i];
    else if (c >= 3) b = 0.0;
    else if (c == 1) b = -ru[i];
    else b = rl[i];
    rhs[ni] = b;
    if (rup) rup[ni] = c == 0 ? ru[i] : (c >= 3 ? 0.0 : INFINITY);
    if (c >= 3) {
      const int k = bd_ex[i], j = n0 + k;
      slack_row[k] = i;
      cost[j] = 0.0;
      double l = rl[i], u = ru[i];
      if (!rup && l < -1e20) l = -INFINITY;     // :375-378
      if (!rup && u > 1e20) u = INFINITY;
      lower[j] = l;
      upper[j] = u;
      cbeg[j] = nnz0 + k;
      cidx[nnz0 + k] = ni;
      cval[nnz0 + k] = -1.0;
      colof[nnz0 + k] = j;
    }
  }
}

__global__ void __launch_bounds__(kTpb)
col_vectors_kernel(int n0, int n, int nnz, double sense, const int* __restrict__ a_start, const double* __restrict__ cc,
                   const double* __restrict__ cl, const double* __restrict__ cu, double* __restrict__ cost,
                   double* __restrict__ lower, double* __restrict__ upper, int* __restrict__ cbeg, int what) {
  // what & 1: the column starts (structure);  what & 2: cost and bounds (values, which arrive on the second copy stream);
  // what & 4: HiPDLP mode -- the cost is not multiplied by the sense and the bounds are not clamped (pdhg.cc:280-297)
  const int stride = gridDim.x * kTpb;
  for (int j = blockIdx.x * kTpb + threadIdx.x; j < n0; j += stride) {
    if (what & 4) {
      cost[j] = cc[j];
      lower[j] = cl[j];
      upper[j] = cu[j];
    } else if (what & 2) {
      cost[j] = cc[j] * sense;
      double l = cl[j], u = cu[j];
      if (l < -1e20) l = -INFINITY;
      if (u > 1e20) u = INFINITY;
      lower[j] = l;
      upper[j] = u;
    }
    if (what & 1) cbeg[j] = a_start[j];
  }
  if ((what & 1) && blockIdx.x == 0 && threadIdx.x == 0) cbeg[n] = nnz;
}

// per nonzero: is its row eq-like (for the stable partition of every column), is its row index in range, does the
// column's storage order ascend (flags[0] |= bad index, flags[1] |= a descent inside a column)
__global__ void __launch_bounds__(kTpb)
nnz_flags_kernel(int nnz0, int m, const int* __restrict__ a_index, const int* __restrict__ colof,
                 const int* __restrict__ eqlike, int* __restrict__ fl, int* __restrict__ flags) {
  const int stride = gridDim.x * kTpb;
  int bad = 0, desc = 0;
  for (int p = blockIdx.x * kTpb + threadIdx.x; p < nnz0; p += stride) {
    const int r = a_index[p];
    if ((unsigned)r >= (unsigned)m) { bad = 1; fl[p] = 0; continue; }
    fl[p] = eqlike[r];
    if (p > 0 && colof[p - 1] == colof[p] && a_index[p - 1] >= r) desc |= a_index[p - 1] > r ? 1 : 2;   // 2: a repeated row
  }
  if (bad) atomicOr(&flags[0], 1);
  if (desc) atomicOr(&flags[1], desc);
}

// structural columns: within a column EQ/BOUND entries first, then LEQ (negated) / GEQ, each group in storage order
// (:410-433) = a stable partition; the exclusive scan of the eq-like flags gives every entry its place
__global__ void __launch_bounds__(kTpb)
scatter_entries_kernel(int nnz0, const int* __restrict__ a_start, const int* __restrict__ a_index,
                       const int* __restrict__ colof, const int* __restrict__ fl_ex,
                       const int* __restrict__ cls, const int* __restrict__ new_idx, int* __restrict__ cidx,
                       unsigned* __restrict__ dest) {
  // structure only: the new row index goes to its place; dest[p] = the place (bit 31: a LEQ row, the value is negated) for
  // scatter_values_kernel, which runs once the coefficient array has arrived
  const int stride = gridDim.x * kTpb;
  for (int p = blockIdx.x * kTpb + threadIdx.x; p < nnz0; p += stride) {
    const int j = colof[p];
    const int s = a_start[j], e = a_start[j + 1];
    const int ne = fl_ex[e] - fl_ex[s];          // eq-like entries of the column
    const int k = fl_ex[p] - fl_ex[s];           // eq-like entries before p
    const int r = a_index[p];
    const int c = cls[r];
    const bool eql = c == 0 || c >= 3;
    const int q = eql ? s + k : s + ne + (p - s - k);
    cidx[q] = new_idx[r];
    dest[p] = (unsigned)q | (c == 1 ? 0x80000000u : 0u);
  }
}

__global__ void __launch_bounds__(kTpb)
scatter_values_kernel(int nnz0, const double* __restrict__ a_value, const unsigned* __restrict__ dest, double* __restrict__ cval) {
  const int stride = gridDim.x * kTpb;
  for (int p = blockIdx.x * kTpb + threadIdx.x; p < nnz0; p += stride) {
    const unsigned d = dest[p];
    const double v = a_value[p];
    cval[d & 0x7fffffffu] = (d >> 31) ? -v : v;
  }
}

// colof[p] = column of nonzero p (one warp per column; a dense column is written 32 entries at a time).  Also validates the
// caller's a_start on the way (flags[3] |= not non-decreasing / outside [0, nnz]); ranges are clamped so that a malformed
// a_start cannot make this kernel write out of bounds before the host has seen the flag.
__global__ void __launch_bounds__(kTpb) colof2_kernel(int n, int nnz, const int* __restrict__ cbeg, int* __restrict__ colof, int* __restrict__ flags) {
  const int j = (blockIdx.x * kTpb + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (j >= n) return;
  int b = cbeg[j], e = cbeg[j + 1];
  if (b > e || b < 0 || e > nnz) { if (lane == 0) atomicOr(&flags[3], 1); b = b < 0 ? 0 : b; e = e > nnz ? nnz : e; }
  for (int p = b + lane; p < e; p += 32) colof[p] = j;
}

// deterministic sums of squares: block partials, then one block (fixed tree)
__global__ void __launch_bounds__(kTpb) sumsq_partial_kernel(int len, const double* __restrict__ v, double* __restrict__ part) {
  __shared__ double sm[kTpb / 32];
  double s = 0.0;
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) s += v[i] * v[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kTpb / 32; w++) t += sm[w];
    part[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(kTpb) sum_final_kernel(int nb, const double* __restrict__ part, double* __restrict__ out) {
  __shared__ double sm[kTpb / 32];
  double s = 0.0;
  for (int i = threadIdx.x; i < nb; i += kTpb) s += part[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kTpb / 32; w++) t += sm[w];
    *out = t;
  }
}

__global__ void __launch_bounds__(kTpb) fill_d_kernel(int len, double* __restrict__ v, double w) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) v[i] = w;
}
__global__ void __launch_bounds__(kTpb) iota_kernel(int len, int* __restrict__ v) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) v[i] = i;
}
__global__ void __launch_bounds__(kTpb) hist_kernel(int nnz, const int* __restrict__ idx, int* __restrict__ cnt) {
  const int stride = gridDim.x * kTpb;
  for (int p = blockIdx.x * kTpb + threadIdx.x; p < nnz; p += stride) atomicAdd(&cnt[idx[p]], 1);
}
__global__ void __launch_bounds__(kTpb) gather_i_kernel(int len, const int* __restrict__ src, const int* __restrict__ idx, int* __restrict__ dst) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) dst[i] = src[idx[i]];
}
__global__ void __launch_bounds__(kTpb) gather_d_kernel(int len, const double* __restrict__ src, const int* __restrict__ idx, double* __restrict__ dst) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) dst[i] = src[idx[i]];
}
__global__ void __launch_bounds__(kTpb) invert_perm_kernel(int len, const int* __restrict__ perm, int* __restrict__ inv) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) inv[perm[i]] = i;
}

// make_perm (host_prep.cpp): rows sorted by DESCENDING length inside windows of kSortWindow rows that do not straddle
// `boundary`, ties in ascending index (stable).  key = window id << 32 | (INT_MAX - length); a stable radix sort of
// (key, index) pairs whose input is in ascending index order gives exactly that order.
constexpr int kWindow = 8192;
__global__ void __launch_bounds__(kTpb)
perm_keys_kernel(int len, int boundary, const int* __restrict__ ptr, unsigned long long* __restrict__ keys) {
  const int stride = gridDim.x * kTpb;
  const int w0 = (boundary + kWindow - 1) / kWindow;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) {
    const int ln = ptr[i + 1] - ptr[i];
    const int wid = i < boundary ? i / kWindow : w0 + (i - boundary) / kWindow;
    keys[i] = ((unsigned long long)wid << 32) | (unsigned long long)(0x7fffffff - ln);
  }
}

// plan_sell (host_prep.cpp), per slice of 32 device rows: longest body row and the mask of lanes that are beyond the
// last row or hold a long row
__global__ void __launch_bounds__(kTpb)
slice_plan_kernel(int nrows, int nslices, const int* __restrict__ perm, const int* __restrict__ ptr, int long_threshold,
                  int* __restrict__ slice_len, unsigned* __restrict__ slice_mask, long long* __restrict__ slice_slots,
                  int* __restrict__ long_flag) {
  const int s = (blockIdx.x * kTpb + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (s >= nslices) return;
  const int nr = s * 32 + lane;
  int ln = 0;
  bool masked = true;
  if (nr < nrows) {
    const int r = perm[nr];
    ln = ptr[r + 1] - ptr[r];
    const bool is_long = ln > long_threshold;
    long_flag[nr] = is_long ? 1 : 0;
    masked = is_long;
  }
  int body = masked ? 0 : ln;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const int t = __shfl_xor_sync(0xffffffffu, body, o); body = t > body ? t : body; }
  const unsigned mask = __ballot_sync(0xffffffffu, masked);
  if (lane == 0) { slice_len[s] = body; slice_mask[s] = mask; slice_slots[s] = 32LL * body; }
}
__global__ void __launch_bounds__(kTpb)
slice_desc_kernel(int nslices, const int* __restrict__ slice_len, const unsigned* __restrict__ slice_mask,
                  const long long* __restrict__ slot_ex, int4* __restrict__ slices, int* __restrict__ too_big) {
  const int stride = gridDim.x * kTpb;
  for (int s = blockIdx.x * kTpb + threadIdx.x; s < nslices; s += stride) {
    const long long off = slot_ex[s];
    if (off + 32LL * slice_len[s] > 2000000000LL) *too_big = 1;
    slices[s] = make_int4((int)off, slice_len[s], (int)slice_mask[s], 0);
  }
}
// How much do a warp's gathers share 32-byte sectors?  One warp per sampled slice looks at the slice's first column ids.
__global__ void __launch_bounds__(kTpb)
sector_sharing_kernel(int nslices, int step, const int4* __restrict__ slices, const int* __restrict__ col, int* __restrict__ out) {
  const int w = (blockIdx.x * kTpb + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const long long sl = (long long)w * step;
  if (sl >= nslices) return;
  const int4 d = slices[sl];
  if (d.y < 1) return;
  const bool live = !((unsigned)d.z >> lane & 1u);
  const unsigned act = __ballot_sync(0xffffffffu, live);
  bool leader = false;
  if (live) {
    const int sector = col[d.x + lane] >> 2;
    const unsigned same = __match_any_sync(act, sector);
    leader = lane == __ffs(same) - 1;
  }
  const unsigned leaders = __ballot_sync(0xffffffffu, leader);
  if (lane == 0) { atomicAdd(out, __popc(leaders)); atomicAdd(out + 1, __popc(act)); }
}
// Window of the input vector touched by one tile of kTileSlices slices (DevSell::tiled): [lo, lo + w), lo even, w even (16-byte
// granules for the bulk copy); w = 0 if it does not fit the staging buffer or would run past the vector.  Padding entries of
// the layout (column 0, value 0) are not entries.  One CTA per tile; counts the tiles that fit in fit[0].
__global__ void __launch_bounds__(kTpb)
tile_window_kernel(int nslices, int ncols, const int4* __restrict__ slices, const int* __restrict__ col,
                   const double* __restrict__ val, int* __restrict__ lo_out, int* __restrict__ w_out, int* __restrict__ fit) {
  __shared__ int smin[kTpb / 32], smax[kTpb / 32];
  const int tile = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int s0 = tile * kTileSlices, s1 = min(s0 + kTileSlices, nslices);
  int mn = INT_MAX, mx = -1;
  for (int sl = s0 + wid; sl < s1; sl += kTpb / 32) {
    const int4 d = slices[sl];
    for (int k = 0; k < d.y; k++) {
      const size_t o = (size_t)d.x + 32 * (size_t)k + lane;
      const int c = col[o];
      if (c != 0 || val[o] != 0.0) { mn = min(mn, c); mx = max(mx, c); }
    }
  }
  for (int off = 16; off > 0; off >>= 1) {
    mn = min(mn, __shfl_down_sync(0xffffffffu, mn, off));
    mx = max(mx, __shfl_down_sync(0xffffffffu, mx, off));
  }
  if (lane == 0) { smin[wid] = mn; smax[wid] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 1; q < kTpb / 32; q++) { mn = min(mn, smin[q]); mx = max(mx, smax[q]); }
    int lo = 0, w = 0;
    if (mx >= 0) {
      lo = mn & ~1;
      w = (mx - lo + 2) & ~1;
      if (lo + w > ncols) w = (ncols & 1) ? 0 : ncols - lo;
      if (w > kTileMaxWindow || w <= 0) { w = 0; lo = 0; }
    }
    lo_out[tile] = lo;
    w_out[tile] = w;
    if (w > 0) atomicAdd(fit, 1);
  }
}
// long rows -> descriptors and segments of kNnzBlk entries (plan_sell's second loop).  `list` holds the device-row ids of
// the long rows in ascending order; one thread walks them (they are few).  totals: [0] n_partials (= segments),
// [1] lcount (entries of lcol / lval incl. the tail of 8)
__global__ void long_plan_kernel(int nlong, const int* __restrict__ list, const int* __restrict__ perm, const int* __restrict__ ptr,
                                 int4* __restrict__ long_rows, int4* __restrict__ segs, long long* __restrict__ totals,
                                 int write) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  long long lpos = 0;
  int nsegs = 0;
  for (int q = 0; q < nlong; q++) {
    const int nr = list[q];
    const int r = perm[nr];
    const int ln = ptr[r + 1] - ptr[r];
    const int nseg = (ln + kNnzBlk - 1) / kNnzBlk;
    const int base = (int)lpos;
    if (write) {
      long_rows[q] = make_int4(nr, nsegs, nseg, nsegs);
      for (int sg = 0; sg < nseg; sg++) {
        const int b = base + sg * kNnzBlk;
        const int e = min(base + (sg + 1) * kNnzBlk, base + ln);
        segs[nsegs + sg] = make_int4(nr, b, e, q);
      }
    }
    nsegs += nseg;
    lpos += ln;
    lpos = (lpos + 3) / 4 * 4;
  }
  totals[0] = nsegs;
  totals[1] = lpos + 8;
}

// ---- HiPDLP mode on several GPUs: nnz-balanced contiguous blocks of a device order (host twin: balanced_blocks).
// w[i] = length of the i-th row in `perm` order + 5 (a per-row cost, as partition_rows charges), w[count] = 0; its exclusive
// scan is the host's prefix array pre[0 .. count].
__global__ void __launch_bounds__(kTpb)
block_weight_kernel(int count, const int* __restrict__ perm, const int* __restrict__ ptr, long long* __restrict__ w) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i <= count; i += stride)
    w[i] = i < count ? (long long)(ptr[perm[i] + 1] - ptr[perm[i]]) + 5 : 0;
}
// b[0] = 0, b[world] = count, b[g] = min(lower_bound(pre[0 .. count], pre[count] g / world), count): one thread per g.  The
// host searches from b[g-1]; every pre[i] before it is < the previous target <= this one, so the whole range gives the same.
__global__ void block_bounds_kernel(int count, int world, const long long* __restrict__ pre, int* __restrict__ b) {
  const int g = threadIdx.x;
  if (g > world) return;
  if (g == 0 || g == world) { b[g] = g == 0 ? 0 : count; return; }
  const long long target = pre[count] * g / world;
  int lo = 0, hi = count + 1;   // first i in [0, count] with pre[i] >= target (count + 1 if none)
  while (lo < hi) {
    const int mid = lo + (hi - lo) / 2;
    if (pre[mid] < target) lo = mid + 1; else hi = mid;
  }
  b[g] = lo < count ? lo : count;
}

// ---- HiPDLP mode: entries of a column ordered by (new row, value), as std::sort of (row, value) pairs (pdhg.cc:300-333).
// Columns stored with strictly ascending rows need nothing beyond the stable eq-like partition (the renumbering is
// monotone inside each group); otherwise an LSD radix sort: first by value, then (stably) by (column, new row).
// Doubles as radix keys: flip all bits of a negative value, the sign bit of a non-negative one (ascending numeric order;
// -0.0 sorts before +0.0, which std::sort leaves in either order -- both orders give the same sums)
__global__ void __launch_bounds__(kTpb) value_key_kernel(int len, const double* __restrict__ v, unsigned long long* __restrict__ key) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(v[i]);
    key[i] = (u >> 63) ? ~u : (u | 0x8000000000000000ull);
  }
}
__global__ void __launch_bounds__(kTpb)
colrow_key_kernel(int len, const int* __restrict__ perm, const int* __restrict__ colof, const int* __restrict__ cidx,
                  unsigned long long* __restrict__ key) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) {
    const int q = perm[i];
    key[i] = ((unsigned long long)colof[q] << 32) | (unsigned)cidx[q];
  }
}
// |c|_2^2 and |b|_2^2 of the UNSCALED HiPDLP data, added in index order like the host's loops (pdhg.cc:353-354): warp 0
// sums the cost, warp 1 the rhs; every lane adds all terms in index order (shuffle broadcast).  The terms come in batches of
// kNormBatch x 32, the next batch's loads in flight while the current one is added, so that the chain of dependent
// additions, not the load latency, sets the time.
constexpr int kNormBatch = 8;
__global__ void __launch_bounds__(64)
ordered_norms_kernel(int n, const double* __restrict__ cost, int m, const double* __restrict__ rhs, double* __restrict__ out) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int len = w == 0 ? n : m;
  const double* v = w == 0 ? cost : rhs;
  auto load = [&](int base, double* t) {
#pragma unroll
    for (int u = 0; u < kNormBatch; u++) {
      const int i = base + 32 * u + lane;
      t[u] = i < len ? v[i] * v[i] : 0.0;
    }
  };
  double cur[kNormBatch], nxt[kNormBatch];
  load(0, cur);
  double sum = 0.0;
  for (int base = 0; base < len; base += 32 * kNormBatch) {
    load(base + 32 * kNormBatch, nxt);
#pragma unroll
    for (int u = 0; u < kNormBatch; u++) {
      const int cb = base + 32 * u;
      if (cb + 32 <= len) {
#pragma unroll
        for (int k = 0; k < 32; k++) sum = sum + __shfl_sync(0xffffffffu, cur[u], k);
      } else if (cb < len) {
        for (int k = 0; k < len - cb; k++) sum = sum + __shfl_sync(0xffffffffu, cur[u], k);
      }
    }
#pragma unroll
    for (int u = 0; u < kNormBatch; u++) cur[u] = nxt[u];
  }
  if (lane == 0) out[w] = sum;
}
}  // namespace

// ===================================================================================== the prologue
namespace {
struct Tmp {   // temporaries of the prologue, returned to the block cache when it ends
  cudaStream_t stream = nullptr;
  std::vector<void*> blocks;
  template <class T> T* get(size_t count) {
    void* p = dev_cache_alloc(std::max<size_t>(count, 1) * sizeof(T));
    blocks.push_back(p);
    return static_cast<T*>(p);
  }
  ~Tmp() { cudaStreamSynchronize(stream); for (void* p : blocks) dev_cache_free(p); }   // (error paths: kernels may still be running)
};
#define PREP_OK(call)                                                                                         \
  do {                                                                                                        \
    cudaError_t e_ = (call);                                                                                  \
    if (e_ != cudaSuccess)                                                                                    \
      throw std::runtime_error(std::string(#call) + ": " + cudaGetErrorString(e_) + " at device_prep.cu:" + \
                               std::to_string(__LINE__));                                                     \
  } while (0)

template <class T> T* keep(size_t count) { return static_cast<T*>(dev_cache_alloc(std::max<size_t>(count, 1) * sizeof(T))); }

void exclusive_scan_i(cudaStream_t s, Tmp& tmp, const int* in, int* out, int count) {
  size_t bytes = 0;
  PREP_OK(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, count, s));
  void* w = tmp.get<char>(bytes);
  PREP_OK(cub::DeviceScan::ExclusiveSum(w, bytes, in, out, count, s));
}
void exclusive_scan_ll(cudaStream_t s, Tmp& tmp, const long long* in, long long* out, int count) {
  size_t bytes = 0;
  PREP_OK(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, count, s));
  void* w = tmp.get<char>(bytes);
  PREP_OK(cub::DeviceScan::ExclusiveSum(w, bytes, in, out, count, s));
}
int bits_for(long long maxval) {
  int b = 1;
  while ((1LL << b) <= maxval && b < 62) b++;
  return b;
}

// one sliced-ELL matrix: perm (length sort), plan, allocation, fill
struct MatrixSource {
  int nrows, ncols;
  const int* ptr;        // [nrows + 1] row pointer of the source rows (rptr for A, cbeg for A')
  int boundary;          // windows of the length sort do not straddle it
  SellSource src;        // where the fill reads entries from (colmap is set after the OTHER perm exists)
};

void make_perm_device(cudaStream_t s, Tmp& tmp, int len, int boundary, const int* ptr, int* perm, int* inv) {
  if (len <= 0) return;
  unsigned long long* k_in = tmp.get<unsigned long long>(len);
  unsigned long long* k_out = tmp.get<unsigned long long>(len);
  int* v_in = tmp.get<int>(len);
  perm_keys_kernel<<<grid_for(len), kTpb, 0, s>>>(len, boundary, ptr, k_in);
  iota_kernel<<<grid_for(len), kTpb, 0, s>>>(len, v_in);
  const int nwin = (boundary + kWindow - 1) / kWindow + (len - boundary + kWindow - 1) / kWindow + 1;
  const int end_bit = 32 + bits_for(nwin);
  size_t bytes = 0;
  PREP_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, k_in, k_out, v_in, perm, len, 0, end_bit, s));
  void* w = tmp.get<char>(bytes);
  PREP_OK(cub::DeviceRadixSort::SortPairs(w, bytes, k_in, k_out, v_in, perm, len, 0, end_bit, s));
  invert_perm_kernel<<<grid_for(len), kTpb, 0, s>>>(len, perm, inv);
}
}  // namespace

void DevicePrologue::run(cudaStream_t s, const b200pdlp_lp& lp, bool do_scale, int long_threshold) {
  NvtxRange nvtx("b200pdlp: device prologue");
  nvtxRangePushA("H2D of the HighsLp arrays + formulate");
  const bool hip = hipdlp;
  Tmp tmp;
  tmp.stream = s;
  const int n0 = lp.num_col, m = lp.num_row, nnz0 = inputs_on_device ? device_nnz : lp.a_start[n0];
  // ---- the caller's arrays in HBM: where they are, or copied there (pinned sources stream at PCIe speed; pageable ones are
  // staged by the driver)
  const int *a_start = lp.a_start, *a_index = lp.a_index;
  const double *a_value = lp.a_value, *cc = lp.col_cost, *cl = lp.col_lower, *cu = lp.col_upper, *rl = lp.row_lower,
               *ru = lp.row_upper;
  // Two copy streams: the STRUCTURE (column starts, row indices, row bounds: 4 n + 4 nnz + 16 m bytes) goes first on `s`; the
  // VALUES (coefficients, cost, column bounds: 8 nnz + 24 n bytes, two thirds of the traffic) follow on a second stream, and
  // everything that depends on the sparsity pattern alone -- classification, the stable partition, the row-major index
  // (radix sort), both length orderings, the slice plans and the three size read-backs -- runs underneath that copy.
  struct Side {
    cudaStream_t st = nullptr; cudaEvent_t structure_up = nullptr, values_up = nullptr;
    cudaEvent_t norms_in = nullptr, norms_t0 = nullptr, norms_t1 = nullptr;   // HiPDLP: the ordered norms on this stream
    Side() {
      PREP_OK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
      PREP_OK(cudaEventCreateWithFlags(&structure_up, cudaEventDisableTiming));
      PREP_OK(cudaEventCreateWithFlags(&values_up, cudaEventDisableTiming));
      PREP_OK(cudaEventCreateWithFlags(&norms_in, cudaEventDisableTiming));
      PREP_OK(cudaEventCreate(&norms_t0));
      PREP_OK(cudaEventCreate(&norms_t1));
    }
    ~Side() {   // before `tmp` hands the staging buffers back: no copy may still be writing them (exception paths)
      if (st) { cudaStreamSynchronize(st); cudaStreamDestroy(st); }
      for (cudaEvent_t e : {structure_up, values_up, norms_in, norms_t0, norms_t1}) if (e) cudaEventDestroy(e);
    }
  } side;
  if (inputs_on_device) {
    PREP_OK(cudaEventRecord(side.values_up, s));   // (the values are there already)
    h2d_bytes = 0;
  } else {
    int* d_start = tmp.get<int>(n0 + 1);
    int* d_index = tmp.get<int>(nnz0);
    double* d_value = tmp.get<double>(nnz0);
    double* d_cc = tmp.get<double>(n0);
    double* d_cl = tmp.get<double>(n0);
    double* d_cu = tmp.get<double>(n0);
    double* d_rl = tmp.get<double>(m);
    double* d_ru = tmp.get<double>(m);
    auto up = [&](cudaStream_t q, void* d, const void* h, size_t bytes) { if (bytes) PREP_OK(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, q)); };
    up(s, d_start, lp.a_start, (size_t)(n0 + 1) * 4);
    up(s, d_index, lp.a_index, (size_t)nnz0 * 4);
    up(s, d_rl, lp.row_lower, (size_t)m * 8); up(s, d_ru, lp.row_upper, (size_t)m * 8);
    PREP_OK(cudaEventRecord(side.structure_up, s));
    PREP_OK(cudaStreamWaitEvent(side.st, side.structure_up, 0));   // the structure first: the copy engine is shared
    up(side.st, d_value, lp.a_value, (size_t)nnz0 * 8);
    up(side.st, d_cc, lp.col_cost, (size_t)n0 * 8); up(side.st, d_cl, lp.col_lower, (size_t)n0 * 8); up(side.st, d_cu, lp.col_upper, (size_t)n0 * 8);
    PREP_OK(cudaEventRecord(side.values_up, side.st));
    h2d_bytes = (size_t)(n0 + 1) * 4 + (size_t)nnz0 * 12 + (size_t)n0 * 24 + (size_t)m * 16;
    a_start = d_start; a_index = d_index; a_value = d_value; cc = d_cc; cl = d_cl; cu = d_cu; rl = d_rl; ru = d_ru;
  }

  // ---- classification, row order
  int* cls = arr.row_class = keep<int>(m);
  int* eqlike = tmp.get<int>(m + 1);
  int* isbound = tmp.get<int>(m + 1);
  int* eq_ex = tmp.get<int>(m + 1);
  int* bd_ex = arr.bound_ord = keep<int>(m + 1);
  int* flags = tmp.get<int>(4);
  PREP_OK(cudaMemsetAsync(flags, 0, 4 * sizeof(int), s));
  PREP_OK(cudaMemsetAsync(eqlike + m, 0, sizeof(int), s));
  PREP_OK(cudaMemsetAsync(isbound + m, 0, sizeof(int), s));
  if (m > 0) classify_rows_kernel<<<grid_for(m), kTpb, 0, s>>>(m, hip ? 1 : 0, rl, ru, cls, eqlike, isbound);
  exclusive_scan_i(s, tmp, eqlike, eq_ex, m + 1);     // eq_ex[m] = number of eq-like rows
  exclusive_scan_i(s, tmp, isbound, bd_ex, m + 1);    // bd_ex[m] = number of BOUND rows
  int* colof0 = tmp.get<int>(nnz0);
  if (n0 > 0) colof2_kernel<<<warp_grid(n0), kTpb, 0, s>>>(n0, nnz0, a_start, colof0, flags);
  int* fl = tmp.get<int>(nnz0 + 1);
  int* fl_ex = tmp.get<int>(nnz0 + 1);
  PREP_OK(cudaMemsetAsync(fl + nnz0, 0, sizeof(int), s));
  if (nnz0 > 0) nnz_flags_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, m, a_index, colof0, eqlike, fl, flags);
  exclusive_scan_i(s, tmp, fl, fl_ex, nnz0 + 1);
  // read-back 1: sizes of the standard form
  int h4[4] = {0, 0, 0, 0}, hflags[4] = {0, 0, 0, 0};
  PREP_OK(cudaMemcpyAsync(&h4[0], eq_ex + m, sizeof(int), cudaMemcpyDeviceToHost, s));
  PREP_OK(cudaMemcpyAsync(&h4[1], bd_ex + m, sizeof(int), cudaMemcpyDeviceToHost, s));
  PREP_OK(cudaMemcpyAsync(hflags, flags, 4 * sizeof(int), cudaMemcpyDeviceToHost, s));
  PREP_OK(cudaStreamSynchronize(s));
  sc.neq = h4[0]; sc.nbound = h4[1]; sc.bad_index = hflags[0]; sc.cols_sorted = (hflags[1] & 1) ? 0 : 1;
  const bool hip_sort = hip && hflags[1] != 0;   // a descent or a repeated row inside a column: sort by (new row, value)
  if (hflags[3]) throw std::invalid_argument("b200pdlp: a_start must be non-decreasing and within [0, nnz]");
  if (sc.bad_index) throw std::invalid_argument("b200pdlp: a_index entry outside [0, num_row)");
  const int neq = sc.neq, nbound = sc.nbound;
  const int n = n0 + nbound, nnz = nnz0 + nbound;
  arr.n = n; arr.m = m; arr.nnz = nnz; arr.neq = neq; arr.n0 = n0; arr.nbound = nbound;
  arr.row_new_idx = keep<int>(m);
  arr.row_old = keep<int>(m);
  arr.slack_row = keep<int>(nbound);

  // ---- standard form (column-major), standard-form order
  int* cbeg = tmp.get<int>(n + 1);
  int* cidx = tmp.get<int>(nnz);
  double* cval = tmp.get<double>(nnz);
  int* colof = tmp.get<int>(nnz);
  double* cost = tmp.get<double>(n);
  double* lower = tmp.get<double>(n);
  double* upper = tmp.get<double>(n);
  double* colscale = tmp.get<double>(n);
  double* rhs = tmp.get<double>(m);
  double* rowscale = tmp.get<double>(m);
  double* rup = hip ? tmp.get<double>(m) : nullptr;   // HiPDLP: row upper bounds, standard-form order
  col_vectors_kernel<<<grid_for(std::max(n0, 1)), kTpb, 0, s>>>(n0, n, nnz, lp.sense, a_start, cc, cl, cu, cost, lower, upper, cbeg, 1);
  if (m > 0)
    row_maps_kernel<<<grid_for(m), kTpb, 0, s>>>(m, n0, nnz0, neq, rl, ru, cls, eq_ex, bd_ex, arr.row_new_idx, arr.row_old,
                                                 arr.slack_row, rhs, cost, lower, upper, cbeg, cidx, cval, colof, rup);
  unsigned* dest = tmp.get<unsigned>(nnz0);
  if (nnz0 > 0) {
    scatter_entries_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, a_start, a_index, colof0, fl_ex, cls, arr.row_new_idx, cidx, dest);
    PREP_OK(cudaMemcpyAsync(colof, colof0, (size_t)nnz0 * sizeof(int), cudaMemcpyDeviceToDevice, s));
  }
  if (hip_sort && nnz0 > 0) {
    // the values are needed for the order: wait for them here (only inputs whose columns are not strictly ascending)
    PREP_OK(cudaStreamWaitEvent(s, side.values_up, 0));
    scatter_values_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, a_value, dest, cval);
    unsigned long long* k_in = tmp.get<unsigned long long>(nnz0);
    unsigned long long* k_out = tmp.get<unsigned long long>(nnz0);
    int* v_in = tmp.get<int>(nnz0);
    int* perm1 = tmp.get<int>(nnz0);
    int* perm2 = tmp.get<int>(nnz0);
    value_key_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, cval, k_in);
    iota_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, v_in);
    size_t bytes = 0;
    PREP_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, k_in, k_out, v_in, perm1, nnz0, 0, 64, s));
    void* w = tmp.get<char>(bytes);
    PREP_OK(cub::DeviceRadixSort::SortPairs(w, bytes, k_in, k_out, v_in, perm1, nnz0, 0, 64, s));
    colrow_key_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, perm1, colof0, cidx, k_in);
    const int end_bit = 32 + bits_for(std::max(n0 - 1, 1));
    bytes = 0;
    PREP_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, k_in, k_out, perm1, perm2, nnz0, 0, end_bit, s));
    w = tmp.get<char>(bytes);
    PREP_OK(cub::DeviceRadixSort::SortPairs(w, bytes, k_in, k_out, perm1, perm2, nnz0, 0, end_bit, s));
    int* ci = tmp.get<int>(nnz0);
    double* cv = tmp.get<double>(nnz0);
    gather_i_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, cidx, perm2, ci);
    gather_d_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, cval, perm2, cv);
    PREP_OK(cudaMemcpyAsync(cidx, ci, (size_t)nnz0 * sizeof(int), cudaMemcpyDeviceToDevice, s));
    PREP_OK(cudaMemcpyAsync(cval, cv, (size_t)nnz0 * sizeof(double), cudaMemcpyDeviceToDevice, s));
  }
  // HiPDLP: row-major index of the CALLER's matrix for the postsolve's row_value = A x (stable sort of the original
  // positions by row: a row's entries in column order, the order of the host's column loop)
  int* orpos = nullptr;
  if (hip) {
    arr.orow_ptr = keep<int>(m + 1);
    arr.orow_col = keep<int>(nnz0);
    arr.orow_val = keep<double>(nnz0);
    int* cnt = tmp.get<int>(m + 1);
    PREP_OK(cudaMemsetAsync(cnt, 0, (size_t)(m + 1) * sizeof(int), s));
    if (nnz0 > 0) hist_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, a_index, cnt);
    exclusive_scan_i(s, tmp, cnt, arr.orow_ptr, m + 1);
    if (nnz0 > 0) {
      orpos = tmp.get<int>(nnz0);
      int* k_out = tmp.get<int>(nnz0);
      int* v_in = tmp.get<int>(nnz0);
      iota_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, v_in);
      size_t bytes = 0;
      const int end_bit = bits_for(std::max(m - 1, 1));
      PREP_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, a_index, k_out, v_in, orpos, nnz0, 0, end_bit, s));
      void* w = tmp.get<char>(bytes);
      PREP_OK(cub::DeviceRadixSort::SortPairs(w, bytes, a_index, k_out, v_in, orpos, nnz0, 0, end_bit, s));
      gather_i_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, colof0, orpos, arr.orow_col);
    }
  }
  double* part = tmp.get<double>(4 * 4736);
  double* dsc = tmp.get<double>(16);
  PREP_OK(cudaMemsetAsync(dsc, 0, 16 * sizeof(double), s));
  auto sumsq = [&](const double* v, int len, double* out, int slot) {
    if (len <= 0) return;
    const int g = grid_for(len);
    sumsq_partial_kernel<<<g, kTpb, 0, s>>>(len, v, part + (size_t)slot * 4736);
    sum_final_kernel<<<1, kTpb, 0, s>>>(g, part + (size_t)slot * 4736, out);
  };

  nvtxRangePop();
  nvtxRangePushA("row-major index (radix sort)");
  // ---- row-major index of the nonzeros: stable radix sort of the positions by row (csc2csr, cupdlp_utils.c:1222-1254)
  int* rptr = tmp.get<int>(m + 2);
  int* rpos = tmp.get<int>(nnz);
  {
    int* cnt = tmp.get<int>(m + 2);
    PREP_OK(cudaMemsetAsync(cnt, 0, (size_t)(m + 2) * sizeof(int), s));
    if (nnz > 0) hist_kernel<<<grid_for(nnz), kTpb, 0, s>>>(nnz, cidx, cnt);
    exclusive_scan_i(s, tmp, cnt, rptr, m + 1);
    if (nnz > 0) {
      int* k_out = tmp.get<int>(nnz);
      int* v_in = tmp.get<int>(nnz);
      iota_kernel<<<grid_for(nnz), kTpb, 0, s>>>(nnz, v_in);
      size_t bytes = 0;
      const int end_bit = bits_for(std::max(m - 1, 1));
      PREP_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, cidx, k_out, v_in, rpos, nnz, 0, end_bit, s));
      void* w = tmp.get<char>(bytes);
      PREP_OK(cub::DeviceRadixSort::SortPairs(w, bytes, cidx, k_out, v_in, rpos, nnz, 0, end_bit, s));
    }
  }
  // columns not stored with ascending rows: positions ordered by (column, row) for A' (second, stable LSD pass)
  int* cpos = nullptr;
  if (!hip && !sc.cols_sorted && nnz > 0) {
    int* k_in = tmp.get<int>(nnz);
    int* k_out = tmp.get<int>(nnz);
    cpos = tmp.get<int>(nnz);
    gather_i_kernel<<<grid_for(nnz), kTpb, 0, s>>>(nnz, colof, rpos, k_in);   // note: slack entries need colof too
    size_t bytes = 0;
    const int end_bit = bits_for(std::max(n - 1, 1));
    PREP_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, k_in, k_out, rpos, cpos, nnz, 0, end_bit, s));
    void* w = tmp.get<char>(bytes);
    PREP_OK(cub::DeviceRadixSort::SortPairs(w, bytes, k_in, k_out, rpos, cpos, nnz, 0, end_bit, s));
  }

  auto values_and_scaling = [&]() {
    NvtxRange r2("values: formulate + Ruiz + Pock-Chambolle scaling");
    // ---- the values have arrived (or the stream waits for them here)
    PREP_OK(cudaStreamWaitEvent(s, side.values_up, 0));
    col_vectors_kernel<<<grid_for(std::max(n0, 1)), kTpb, 0, s>>>(n0, n, nnz, lp.sense, a_start, cc, cl, cu, cost, lower, upper, cbeg, 2);
    if (nnz0 > 0) scatter_values_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, a_value, dest, cval);
    if (n > 0) fill_d_kernel<<<grid_for(n), kTpb, 0, s>>>(n, colscale, 1.0);
    if (m > 0) fill_d_kernel<<<grid_for(m), kTpb, 0, s>>>(m, rowscale, 1.0);
    // Init_Scaling (cupdlp_scaling.c:395-425): 2-norms of the unscaled cost and rhs
    sumsq(cost, n, dsc + 0, 0);
    sumsq(rhs, m, dsc + 1, 1);
    // ---- PDHG_Scale_Data (setup_kernels.cu): 10 Ruiz passes + Pock-Chambolle, bit-identical to host_prep.cpp::scale
    double* cs = tmp.get<double>(n);
    double* cnorm = tmp.get<double>(n);
    double* rs = tmp.get<double>(m);
    double* rnorm = tmp.get<double>(m);
    double* amax = dsc + 4;
    DevForm F{n, m, nnz, cbeg, cidx, colof, cval, cost, lower, upper, colscale, rhs, rowscale};
    DevScaleScratch w{cs, cnorm, rs, rnorm, amax};
    if (do_scale && nnz > 0) {
      device_scale_ruiz(s, F, w);
      device_scale_pock_chambolle(s, F, w, rptr, rpos);
    } else if (nnz > 0) {
      device_abs_max(s, nnz, cval, amax);
    }
    PREP_OK(cudaGetLastError());
    // PDHG_Init_Step_Sizes: |c|^2, |b|^2 of the scaled data
    sumsq(cost, n, dsc + 2, 2);
    sumsq(rhs, m, dsc + 3, 3);

  };
  // HiPDLP mode (PDLPSolver::preprocessLp + Scaling::scaleProblem; host twin host_prep_hipdlp.cpp)
  double* unscaled = hip ? tmp.get<double>((size_t)n + m) : nullptr;
  auto values_and_scaling_hip = [&]() {
    NvtxRange r2("values: HiPDLP formulate + scaling");
    PREP_OK(cudaStreamWaitEvent(s, side.values_up, 0));
    col_vectors_kernel<<<grid_for(std::max(n0, 1)), kTpb, 0, s>>>(n0, n, nnz, 1.0, a_start, cc, cl, cu, cost, lower, upper, cbeg, 4);
    if (nnz0 > 0 && !hip_sort) scatter_values_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, a_value, dest, cval);
    if (nnz0 > 0) gather_d_kernel<<<grid_for(nnz0), kTpb, 0, s>>>(nnz0, a_value, orpos, arr.orow_val);
    if (n > 0) fill_d_kernel<<<grid_for(n), kTpb, 0, s>>>(n, colscale, 1.0);
    if (m > 0) fill_d_kernel<<<grid_for(m), kTpb, 0, s>>>(m, rowscale, 1.0);
    // |c|^2 and |b|^2 of the unscaled data in index order: one warp each, on the side stream under the scaling and the layouts
    if (n > 0) PREP_OK(cudaMemcpyAsync(unscaled, cost, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s));
    if (m > 0) PREP_OK(cudaMemcpyAsync(unscaled + n, rhs, (size_t)m * sizeof(double), cudaMemcpyDeviceToDevice, s));
    PREP_OK(cudaEventRecord(side.norms_in, s));
    PREP_OK(cudaStreamWaitEvent(side.st, side.norms_in, 0));
    PREP_OK(cudaEventRecord(side.norms_t0, side.st));
    ordered_norms_kernel<<<1, 64, 0, side.st>>>(n, unscaled, m, unscaled + n, dsc);
    PREP_OK(cudaEventRecord(side.norms_t1, side.st));
    double* cs = tmp.get<double>(n);
    double* rs = tmp.get<double>(m);
    DevForm F{n, m, nnz, cbeg, cidx, colof, cval, cost, lower, upper, colscale, rhs, rowscale};
    DevScaleScratch w{cs, nullptr, rs, nullptr, dsc + 4};
    sc.scaled = device_scale_hipdlp(s, F, w, rptr, rpos, rup, scaling_mode, ruiz_iterations) ? 1 : 0;
    PREP_OK(cudaGetLastError());
  };
  auto keep_the_form = [&]() {
    // the standard form in standard-form order survives the prologue (tests: b200pdlp_problem_get_*; several GPUs: the host
    // builds every rank's layouts from it)
    auto dup_i = [&](const int* src, size_t cnt) { int* d = keep<int>(cnt); PREP_OK(cudaMemcpyAsync(d, src, cnt * sizeof(int), cudaMemcpyDeviceToDevice, s)); return d; };
    auto dup_d = [&](const double* src, size_t cnt) { double* d = keep<double>(cnt); PREP_OK(cudaMemcpyAsync(d, src, cnt * sizeof(double), cudaMemcpyDeviceToDevice, s)); return d; };
    form.cbeg = dup_i(cbeg, n + 1); form.cidx = dup_i(cidx, nnz); form.cval = dup_d(cval, nnz);
    form.cost = dup_d(cost, n); form.lower = dup_d(lower, n); form.upper = dup_d(upper, n); form.colscale = dup_d(colscale, n);
    form.rhs = dup_d(rhs, m); form.rowscale = dup_d(rowscale, m);
    form.rptr = dup_i(rptr, m + 1); form.rpos = dup_i(rpos, nnz);
    if (hip) form.row_upper = dup_d(rup, m);
    form.rcol = keep<int>(nnz);
    if (nnz > 0) gather_i_kernel<<<grid_for(nnz), kTpb, 0, s>>>(nnz, colof, rpos, form.rcol);
  };
  if (stop_after_scaling) {
    values_and_scaling();
    keep_the_form();
    double hd[5] = {0, 0, 0, 0, 0};
    PREP_OK(cudaMemcpyAsync(hd, dsc, 5 * sizeof(double), cudaMemcpyDeviceToHost, s));
    PREP_OK(cudaStreamSynchronize(s));
    sc.norm_cost_sq = hd[0]; sc.norm_rhs_sq = hd[1]; sc.beta_cost_sq = hd[2]; sc.beta_rhs_sq = hd[3]; sc.amax = hd[4];
    nvtxRangePop();
    return;
  }
  nvtxRangePop();
  nvtxRangePushA("orderings + sliced-ELL layouts");
  // ---- device orderings and sliced-ELL plans
  arr.rperm = keep<int>(m); arr.rinv = keep<int>(m);
  arr.cperm = keep<int>(n); arr.cinv = keep<int>(n);
  make_perm_device(s, tmp, m, neq, rptr, arr.rperm, arr.rinv);
  make_perm_device(s, tmp, n, n, cbeg, arr.cperm, arr.cinv);
  // HiPDLP mode on several GPUs: the partition of both device orders into `world` blocks (read-back 1b)
  const bool blocks = world > 1;
  if (blocks) {
    int* bnd = tmp.get<int>(2 * (world + 1));
    auto partition = [&](int count, const int* perm, const int* ptr, int* b) {
      long long* w = tmp.get<long long>(count + 1);
      long long* pre = tmp.get<long long>(count + 1);
      block_weight_kernel<<<grid_for(count + 1), kTpb, 0, s>>>(count, perm, ptr, w);
      exclusive_scan_ll(s, tmp, w, pre, count + 1);
      block_bounds_kernel<<<1, 32, 0, s>>>(count, world, pre, b);
    };
    partition(m, arr.rperm, rptr, bnd);
    partition(n, arr.cperm, cbeg, bnd + world + 1);
    std::vector<int> hb((size_t)2 * (world + 1));
    PREP_OK(cudaMemcpyAsync(hb.data(), bnd, hb.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    PREP_OK(cudaStreamSynchronize(s));
    rb.assign(hb.begin(), hb.begin() + world + 1);
    cb.assign(hb.begin() + world + 1, hb.end());
  }
  struct Plan {
    int nrows = 0, nslices = 0;
    int *slice_len = nullptr; unsigned* slice_mask = nullptr; long long *slots = nullptr, *slot_ex = nullptr;
    int *long_flag = nullptr, *long_list = nullptr, *nlong_dev = nullptr;
    long long* totals = nullptr;
  };
  int* too_big = flags + 2;
  auto plan1 = [&](Plan& P, int nrows, const int* perm, const int* ptr) {
    P.nrows = nrows; P.nslices = (nrows + 31) / 32;
    P.slice_len = tmp.get<int>(P.nslices); P.slice_mask = tmp.get<unsigned>(P.nslices);
    P.slots = tmp.get<long long>(P.nslices + 1); P.slot_ex = tmp.get<long long>(P.nslices + 1);
    P.long_flag = tmp.get<int>(nrows); P.long_list = tmp.get<int>(nrows); P.nlong_dev = tmp.get<int>(1);
    P.totals = tmp.get<long long>(2);
    PREP_OK(cudaMemsetAsync(P.slots + P.nslices, 0, sizeof(long long), s));
    PREP_OK(cudaMemsetAsync(P.nlong_dev, 0, sizeof(int), s));
    if (P.nslices > 0) {
      slice_plan_kernel<<<warp_grid(P.nslices), kTpb, 0, s>>>(nrows, P.nslices, perm, ptr, long_threshold, P.slice_len,
                                                             P.slice_mask, P.slots, P.long_flag);
      exclusive_scan_ll(s, tmp, P.slots, P.slot_ex, P.nslices + 1);
      size_t bytes = 0;
      cub::CountingInputIterator<int> ids(0);
      PREP_OK(cub::DeviceSelect::Flagged(nullptr, bytes, ids, P.long_flag, P.long_list, P.nlong_dev, nrows, s));
      void* wsp = tmp.get<char>(bytes);
      PREP_OK(cub::DeviceSelect::Flagged(wsp, bytes, ids, P.long_flag, P.long_list, P.nlong_dev, nrows, s));
    } else {
      PREP_OK(cudaMemsetAsync(P.slot_ex, 0, sizeof(long long), s));
    }
  };
  // One job per sliced-ELL matrix: rows perm[0 .. nrows) of a device order (perm = the order + the block's first row), their
  // entries read from `src`.  One GPU: A and A'.  Block mode: A_g and A_g' of every rank on this device.
  SellSource SA{rptr, rptr + 1, rpos, colof, cval, 0, arr.cinv};
  SellSource SAT{cbeg, cbeg + 1, cpos, cidx, cval, 0, arr.rinv};
  if (cpos) {
    // cpos lists ALL positions ordered by (column, row): column j's entries are cpos[cbeg[j] .. cbeg[j+1]) since every
    // column keeps its range
    SAT.pos = cpos;
  }
  struct Job {
    DevSellOwned* M; int nrows, ncols; const int* perm; const int* ptr; const SellSource* src;
    Plan P; long long padded = 0, lcount = 8; int nlong = 0, nsegs = 0;
  };
  std::vector<Job> jobs;
  if (blocks) {
    block_A.assign(ranks.size(), DevSellOwned());
    block_AT.assign(ranks.size(), DevSellOwned());
    for (size_t k = 0; k < ranks.size(); k++) {
      const int g = ranks[k];
      jobs.push_back(Job{&block_A[k], rb[g + 1] - rb[g], n, arr.rperm + rb[g], rptr, &SA});
      jobs.push_back(Job{&block_AT[k], cb[g + 1] - cb[g], m, arr.cperm + cb[g], cbeg, &SAT});
    }
  } else {
    jobs.push_back(Job{&A, m, n, arr.rperm, rptr, &SA});
    jobs.push_back(Job{&AT, n, m, arr.cperm, cbeg, &SAT});
  }
  for (Job& J : jobs) plan1(J.P, J.nrows, J.perm, J.ptr);
  // read-back 2: sizes of the layouts (padded slots, long rows)
  std::vector<long long> hsz(2 * jobs.size(), 0);
  for (size_t k = 0; k < jobs.size(); k++) {
    PREP_OK(cudaMemcpyAsync(&hsz[2 * k], jobs[k].P.slot_ex + jobs[k].P.nslices, sizeof(long long), cudaMemcpyDeviceToHost, s));
    PREP_OK(cudaMemcpyAsync(&hsz[2 * k + 1], jobs[k].P.nlong_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
  }
  PREP_OK(cudaStreamSynchronize(s));
  for (size_t k = 0; k < jobs.size(); k++) {
    jobs[k].padded = hsz[2 * k];
    jobs[k].nlong = (int)hsz[2 * k + 1];
    if (jobs[k].padded > 2000000000LL) throw std::runtime_error("b200pdlp: matrix too large for 32-bit slice offsets");
  }
  // long rows: count the segments first (sizes), then write the descriptors
  auto long_sizes = [&](Plan& P, int nlong, const int* perm, const int* ptr) {
    long_plan_kernel<<<1, 32, 0, s>>>(nlong, P.long_list, perm, ptr, nullptr, nullptr, P.totals, 0);
  };
  for (Job& J : jobs) long_sizes(J.P, J.nlong, J.perm, J.ptr);
  for (size_t k = 0; k < jobs.size(); k++)
    PREP_OK(cudaMemcpyAsync(&hsz[2 * k], jobs[k].P.totals, 2 * sizeof(long long), cudaMemcpyDeviceToHost, s));
  PREP_OK(cudaStreamSynchronize(s));
  for (size_t k = 0; k < jobs.size(); k++) {
    jobs[k].nsegs = (int)hsz[2 * k];
    jobs[k].lcount = hsz[2 * k + 1];
    if (jobs[k].lcount > 2000000000LL) throw std::runtime_error("b200pdlp: long rows too large for 32-bit offsets");
  }
  if (!blocks) {
    sc.a_padded = jobs[0].padded; sc.a_nlong = jobs[0].nlong; sc.a_nsegs = jobs[0].nsegs; sc.a_lcount = jobs[0].lcount;
    sc.at_padded = jobs[1].padded; sc.at_nlong = jobs[1].nlong; sc.at_nsegs = jobs[1].nsegs; sc.at_lcount = jobs[1].lcount;
  }

  if (hip) values_and_scaling_hip();
  else values_and_scaling();

  // ---- allocate and fill the layouts
  auto build = [&](DevSellOwned& M, Plan& P, int nrows, int ncols, long long padded, int nlong, int nsegs, long long lcount,
                   const int* perm, const int* ptr, const SellSource& S) {
    M.nrows = nrows; M.ncols = ncols; M.nslices = P.nslices; M.padded = padded; M.nlong = nlong; M.nsegs = nsegs;
    M.lcount = lcount;
    M.slices = keep<int4>(P.nslices);
    M.col = keep<int>((size_t)padded + 32);
    M.val = keep<double>((size_t)padded + 32);
    M.segs = keep<int4>(nsegs);
    M.long_rows = keep<int4>(nlong);
    M.lcol = keep<int>((size_t)lcount);
    M.lval = keep<double>((size_t)lcount);
    M.long_partial = keep<double>(nsegs);
    M.long_counter = keep<unsigned>(nlong);
    PREP_OK(cudaMemsetAsync(M.lcol, 0, std::max<size_t>((size_t)lcount, 1) * sizeof(int), s));
    PREP_OK(cudaMemsetAsync(M.lval, 0, std::max<size_t>((size_t)lcount, 1) * sizeof(double), s));
    PREP_OK(cudaMemsetAsync(M.long_partial, 0, std::max<size_t>(nsegs, 1) * sizeof(double), s));
    PREP_OK(cudaMemsetAsync(M.long_counter, 0, std::max<size_t>(nlong, 1) * sizeof(unsigned), s));
    if (P.nslices > 0) slice_desc_kernel<<<grid_for(P.nslices), kTpb, 0, s>>>(P.nslices, P.slice_len, P.slice_mask, P.slot_ex, M.slices, too_big);
    if (nlong > 0) long_plan_kernel<<<1, 32, 0, s>>>(nlong, P.long_list, perm, ptr, M.long_rows, M.segs, P.totals, 1);
    device_fill_sell(s, nrows, P.nslices, M.slices, perm, S, M.col, M.val, padded, nlong, M.long_rows, M.segs, M.lcol, M.lval);
  };
  for (Job& J : jobs) build(*J.M, J.P, J.nrows, J.ncols, J.padded, J.nlong, J.nsegs, J.lcount, J.perm, J.ptr, *J.src);
  int* sect = tmp.get<int>(4);
  PREP_OK(cudaMemsetAsync(sect, 0, 4 * sizeof(int), s));
  auto sample = [&](const DevSellOwned& M, int* out) {
    if (M.nslices <= 0) return;
    const int step = std::max(1, M.nslices / 4096), nw = (M.nslices + step - 1) / step;
    sector_sharing_kernel<<<warp_grid(nw), kTpb, 0, s>>>(M.nslices, step, M.slices, M.col, out);
  };
  if (!blocks) {   // (the shards run one slice per warp: no sampling, no tile windows)
    sample(A, sect);
    sample(AT, sect + 2);
  }
  // tile windows for the shared-memory staged shape (decided by the engine from tiles_staged / ntiles)
  int* fit = tmp.get<int>(2);
  PREP_OK(cudaMemsetAsync(fit, 0, 2 * sizeof(int), s));
  auto windows = [&](DevSellOwned& M, int* fit_out) {
    M.ntiles = (M.nslices + kTileSlices - 1) / kTileSlices;
    if (M.ntiles <= 0) { M.ntiles = 0; return; }
    M.tile_lo = keep<int>(M.ntiles);
    M.tile_w = keep<int>(M.ntiles);
    tile_window_kernel<<<M.ntiles, kTpb, 0, s>>>(M.nslices, M.ncols, M.slices, M.col, M.val, M.tile_lo, M.tile_w, fit_out);
  };
  if (!blocks) {
    windows(A, fit);
    windows(AT, fit + 1);
  }

  // ---- vectors in device order
  arr.cost = keep<double>(n); arr.lower = keep<double>(n); arr.upper = keep<double>(n); arr.colscale = keep<double>(n);
  arr.rhs = keep<double>(m); arr.rowscale = keep<double>(m);
  if (n > 0) {
    gather_d_kernel<<<grid_for(n), kTpb, 0, s>>>(n, cost, arr.cperm, arr.cost);
    gather_d_kernel<<<grid_for(n), kTpb, 0, s>>>(n, lower, arr.cperm, arr.lower);
    gather_d_kernel<<<grid_for(n), kTpb, 0, s>>>(n, upper, arr.cperm, arr.upper);
    gather_d_kernel<<<grid_for(n), kTpb, 0, s>>>(n, colscale, arr.cperm, arr.colscale);
  }
  if (m > 0) {
    gather_d_kernel<<<grid_for(m), kTpb, 0, s>>>(m, rhs, arr.rperm, arr.rhs);
    gather_d_kernel<<<grid_for(m), kTpb, 0, s>>>(m, rowscale, arr.rperm, arr.rowscale);
  }
  if (hip) {
    arr.rup = keep<double>(m);
    if (m > 0) gather_d_kernel<<<grid_for(m), kTpb, 0, s>>>(m, rup, arr.rperm, arr.rup);
  }
  PREP_OK(cudaGetLastError());
  if (keep_form) keep_the_form();
  nvtxRangePop();
  struct { double d[5]; int tb; int sect[4]; int fit[2]; } hfin;
  memset(&hfin, 0, sizeof(hfin));
  if (hip) PREP_OK(cudaStreamWaitEvent(s, side.norms_t1, 0));   // the ordered norms (side stream)
  PREP_OK(cudaMemcpyAsync(hfin.d, dsc, 5 * sizeof(double), cudaMemcpyDeviceToHost, s));
  PREP_OK(cudaMemcpyAsync(hfin.sect, sect, 4 * sizeof(int), cudaMemcpyDeviceToHost, s));
  PREP_OK(cudaMemcpyAsync(hfin.fit, fit, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
  PREP_OK(cudaMemcpyAsync(&hfin.tb, too_big, sizeof(int), cudaMemcpyDeviceToHost, s));
  PREP_OK(cudaStreamSynchronize(s));   // the temporaries go back to the cache below: everything that reads them is done
  sc.norm_cost_sq = hfin.d[0]; sc.norm_rhs_sq = hfin.d[1]; sc.beta_cost_sq = hfin.d[2]; sc.beta_rhs_sq = hfin.d[3]; sc.amax = hfin.d[4];
  sc.a_sectors = hfin.sect[0]; sc.a_lanes = hfin.sect[1]; sc.at_sectors = hfin.sect[2]; sc.at_lanes = hfin.sect[3];
  A.tiles_staged = hfin.fit[0]; AT.tiles_staged = hfin.fit[1];
  if (hip) {
    float ms = 0.f;
    PREP_OK(cudaEventElapsedTime(&ms, side.norms_t0, side.norms_t1));
    sc.norms_ms = ms;
  }
  if (hfin.tb) throw std::runtime_error("b200pdlp: matrix too large for 32-bit slice offsets");
}

// ===================================================================================== solve boundary
// PDHG_PreSolve (hot start, cupdlp_solver.c:1217-1279) + PDHG_Init_Variables (:531-591) and PDHG_PostSolve (:1281-1435)
// for a problem whose maps live on the device (host twins: engine.cu solve_on_device).
namespace {
__global__ void __launch_bounds__(kTpb)
init_cols_kernel(int n, int n0, int warm, const int* __restrict__ cperm, const int* __restrict__ slack_row,
                 const double* __restrict__ wcol, const double* __restrict__ wrowval, const double* __restrict__ colscale,
                 const double* __restrict__ lower, const double* __restrict__ upper, double* __restrict__ x0,
                 double* __restrict__ xsum) {
  const int stride = gridDim.x * kTpb;
  for (int jd = blockIdx.x * kTpb + threadIdx.x; jd < n; jd += stride) {
    const double u = upper[jd], l = lower[jd];
    double v = 0.0;
    if (warm) {
      const int j = cperm[jd];
      v = j < n0 ? wcol[j] : wrowval[slack_row[j - n0]];
      v = v * colscale[jd];
    }
    v = v < u ? v : u;     // PDHG_Project_Bounds: upper first, then lower
    v = v > l ? v : l;
    x0[jd] = v;
    double z = 0.0;        // the sums start at proj(0) (PDHG_Init_Variables :577-583)
    z = z < u ? z : u;
    z = z > l ? z : l;
    xsum[jd] = z;
  }
}
__global__ void __launch_bounds__(kTpb)
init_rows_kernel(int m, int warm, double sense, const int* __restrict__ rperm, const int* __restrict__ row_old,
                 const int* __restrict__ cls, const double* __restrict__ wdual, const double* __restrict__ rowscale,
                 double* __restrict__ y0) {
  const int stride = gridDim.x * kTpb;
  for (int id = blockIdx.x * kTpb + threadIdx.x; id < m; id += stride) {
    double v = 0.0;
    if (warm) {
      const int o = row_old[rperm[id]];
      const double mu = cls[o] == 1 ? -1.0 : 1.0;
      v = sense * mu * wdual[o];
      v = v * rowscale[id];
    }
    y0[id] = v;
  }
}
__global__ void __launch_bounds__(kTpb)
post_cols_kernel(int n0, int have_check, double sense, const int* __restrict__ cinv, const double* __restrict__ x,
                 const double* __restrict__ aty, const double* __restrict__ cost, const double* __restrict__ lower,
                 const double* __restrict__ upper, const double* __restrict__ colscale, double* __restrict__ col_value,
                 double* __restrict__ col_dual) {
  const int stride = gridDim.x * kTpb;
  for (int j = blockIdx.x * kTpb + threadIdx.x; j < n0; j += stride) {
    const int jd = cinv[j];
    const double sc = colscale[jd];
    col_value[j] = x[jd] / sc;
    double sp = 0.0, sn = 0.0;
    if (have_check) {   // dSlackPos / dSlackNeg of the returned iterate (cupdlp_solver.c:150-176)
      double rc = aty[jd] * -1.0;
      rc = rc + 1.0 * cost[jd];
      double a = rc > 0.0 ? rc : 0.0;
      a = a * (lower[jd] > -INFINITY ? 1.0 : 0.0);
      double b = rc < 0.0 ? rc : 0.0;
      b = b * -1.0;
      b = b * (upper[jd] < INFINITY ? 1.0 : 0.0);
      sp = a; sn = b;
    }
    sp = sp * sc;
    sn = sn * sc;
    const double v = sp - sn;
    col_dual[j] = v * sense;
  }
}
__global__ void __launch_bounds__(kTpb)
post_rows_kernel(int m, int n0, double sense, const int* __restrict__ new_idx, const int* __restrict__ cls,
                 const int* __restrict__ bound_ord, const int* __restrict__ rinv, const int* __restrict__ cinv,
                 const double* __restrict__ x, const double* __restrict__ y, const double* __restrict__ ax,
                 const double* __restrict__ colscale, const double* __restrict__ rowscale, double* __restrict__ row_value,
                 double* __restrict__ row_dual) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < m; i += stride) {
    const int id = rinv[new_idx[i]];
    const int c = cls[i];
    const double rs = rowscale[id];
    double v = ax[id] * rs;
    if (c == 1) v = -v;
    else if (c == 3) {
      const int jd = cinv[n0 + bound_ord[i]];
      v = v + x[jd] / colscale[jd];
    }
    row_value[i] = v;
    double d = (y[id] / rs) * sense;
    if (c == 1) d = -d;
    row_dual[i] = d;
  }
}
}  // namespace

void launch_init_point(cudaStream_t s, const DevProblemArrays& a, double sense, const double* wcol, const double* wrowval,
                       const double* wdual, const double* colscale, const double* lower, const double* upper,
                       const double* rowscale, double* x0, double* xsum, double* y0) {
  const int warm = (wcol && wrowval && wdual) ? 1 : 0;
  if (a.n > 0)
    init_cols_kernel<<<grid_for(a.n), kTpb, 0, s>>>(a.n, a.n0, warm, a.cperm, a.slack_row, wcol, wrowval, colscale, lower, upper, x0, xsum);
  if (a.m > 0) init_rows_kernel<<<grid_for(a.m), kTpb, 0, s>>>(a.m, warm, sense, a.rperm, a.row_old, a.row_class, wdual, rowscale, y0);
}

void launch_postsolve(cudaStream_t s, const DevProblemArrays& a, double sense, int have_check, const double* x, const double* aty,
                      const double* y, const double* ax, const double* cost, const double* lower, const double* upper,
                      const double* colscale, const double* rowscale, double* col_value, double* col_dual, double* row_value,
                      double* row_dual) {
  if (a.n0 > 0)
    post_cols_kernel<<<grid_for(a.n0), kTpb, 0, s>>>(a.n0, have_check, sense, a.cinv, x, aty, cost, lower, upper, colscale, col_value, col_dual);
  if (a.m > 0)
    post_rows_kernel<<<grid_for(a.m), kTpb, 0, s>>>(a.m, a.n0, sense, a.row_new_idx, a.row_class, a.bound_ord, a.rinv, a.cinv, x, y, ax,
                                                    colscale, rowscale, row_value, row_dual);
}

namespace {
__global__ void __launch_bounds__(kTpb)
hip_init_kernel(int n, const double* __restrict__ lower, const double* __restrict__ upper, double* __restrict__ x,
                double* __restrict__ xa) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < n; i += stride) {
    double v = 0.0;
    if (v > upper[i]) v = upper[i];
    if (v < lower[i]) v = lower[i];
    x[i] = v;
    xa[i] = v;
  }
}
__global__ void __launch_bounds__(kTpb)
hip_post_cols_kernel(int n0, int converged, int scaled, double sense, const int* __restrict__ cinv, const double* __restrict__ x,
                     const double* __restrict__ sp, const double* __restrict__ sn, const double* __restrict__ colscale,
                     double* __restrict__ col_value, double* __restrict__ col_dual) {
  const int stride = gridDim.x * kTpb;
  for (int j = blockIdx.x * kTpb + threadIdx.x; j < n0; j += stride) {
    const int jd = cinv[j];
    const double cs = colscale[jd];
    double xv = converged ? x[jd] : 0.0;
    if (scaled) xv = xv / cs;
    col_value[j] = xv;
    const double a = sp[jd] * cs, b = sn[jd] * cs;
    double v = a - b;
    v = v * sense;
    col_dual[j] = v;
  }
}
// one thread per row (the postsolve runs once per solve; a long row is a few thousand dependent adds)
__global__ void __launch_bounds__(kTpb)
hip_post_rows_kernel(int m, int converged, int scaled, const int* __restrict__ new_idx, const int* __restrict__ cls,
                     const int* __restrict__ rinv, const double* __restrict__ y, const double* __restrict__ rowscale,
                     const int* __restrict__ optr, const int* __restrict__ ocol, const double* __restrict__ oval,
                     const double* __restrict__ col_value, double* __restrict__ row_value, double* __restrict__ row_dual) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < m; i += stride) {
    const int id = rinv[new_idx[i]];
    double d = converged ? y[id] : 0.0;
    if (scaled) d = d / rowscale[id];
    row_dual[i] = cls[i] == 1 ? -d : d;
    double v = 0.0;
    for (int q = optr[i]; q < optr[i + 1]; q++) v = v + oval[q] * col_value[ocol[q]];
    row_value[i] = v;
  }
}
}  // namespace

void launch_hip_init_point(cudaStream_t s, int n, const double* lower, const double* upper, double* x, double* xa) {
  if (n > 0) hip_init_kernel<<<grid_for(n), kTpb, 0, s>>>(n, lower, upper, x, xa);
}

void launch_hip_postsolve(cudaStream_t s, const DevProblemArrays& a, double sense, int converged, int scaled, const double* x,
                          const double* y, const double* sp, const double* sn, const double* colscale, const double* rowscale,
                          double* col_value, double* col_dual, double* row_value, double* row_dual) {
  if (a.n0 > 0)
    hip_post_cols_kernel<<<grid_for(a.n0), kTpb, 0, s>>>(a.n0, converged, scaled, sense, a.cinv, x, sp, sn, colscale, col_value, col_dual);
  if (a.m > 0)
    hip_post_rows_kernel<<<grid_for(a.m), kTpb, 0, s>>>(a.m, converged, scaled, a.row_new_idx, a.row_class, a.rinv, y, rowscale,
                                                        a.orow_ptr, a.orow_col, a.orow_val, col_value, row_value, row_dual);
}

void DevSellOwned::release() {
  dev_cache_free(slices); dev_cache_free(col); dev_cache_free(val); dev_cache_free(segs); dev_cache_free(long_rows);
  dev_cache_free(lcol); dev_cache_free(lval); dev_cache_free(long_partial); dev_cache_free(long_counter);
  dev_cache_free(tile_lo); dev_cache_free(tile_w);
  *this = DevSellOwned();
}

void DevicePrologue::release_form() {
  dev_cache_free(form.cbeg); dev_cache_free(form.cidx); dev_cache_free(form.cval); dev_cache_free(form.cost);
  dev_cache_free(form.lower); dev_cache_free(form.upper); dev_cache_free(form.colscale); dev_cache_free(form.rhs);
  dev_cache_free(form.rowscale); dev_cache_free(form.rptr); dev_cache_free(form.rpos); dev_cache_free(form.rcol);
  dev_cache_free(form.row_upper);
  form = DevStdForm();
}

void DevicePrologue::release_blocks() {
  for (DevSellOwned& M : block_A) M.release();
  for (DevSellOwned& M : block_AT) M.release();
  block_A.clear();
  block_AT.clear();
}

void DevicePrologue::release_arrays() {
  dev_cache_free(arr.row_new_idx); dev_cache_free(arr.row_class); dev_cache_free(arr.row_old); dev_cache_free(arr.slack_row);
  dev_cache_free(arr.bound_ord); dev_cache_free(arr.rperm); dev_cache_free(arr.rinv); dev_cache_free(arr.cperm);
  dev_cache_free(arr.cinv); dev_cache_free(arr.cost); dev_cache_free(arr.lower); dev_cache_free(arr.upper);
  dev_cache_free(arr.colscale); dev_cache_free(arr.rhs); dev_cache_free(arr.rowscale);
  dev_cache_free(arr.rup); dev_cache_free(arr.orow_ptr); dev_cache_free(arr.orow_col); dev_cache_free(arr.orow_val);
  arr = DevProblemArrays();
}

}  // namespace b200
