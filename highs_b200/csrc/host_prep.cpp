// highs_b200/csrc/host_prep.cpp -- see host_prep.hpp.
//
// The arithmetic (which quotient is taken when, in which order sums run) follows
// the reference so that the scaled data are bit-identical to what cuPDLP-C
// iterates on; the loop structure does not: the reference makes four sweeps over
// the nonzeros per Ruiz pass (column norms, row norms, row division, column
// division), here every pass is one sweep that applies pass k and gathers the
// norms of pass k+1 at the same time.
#include "host_prep.hpp"

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <mutex>
#include <pthread.h>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <exception>
#include <functional>
#include <limits>
#include <stdexcept>
#include <thread>

namespace b200 {

// ---- tiny fork-join helper: the O(nnz) prologue (formulate, 11 scaling sweeps, transposition, ELL build)
// is the dominant cost of a short solve once the iterations run at ~10^4/s, so it is spread over host cores.
// Every parallel loop below is arranged so that each output element is produced by exactly one thread with
// the same arithmetic, in the same order, as the sequential code: results do not depend on the thread count.
static int host_threads() {
  static int n = [] {
    if (const char* e = getenv("B200PDLP_HOST_THREADS")) return std::max(1, atoi(e));
    const unsigned hc = std::thread::hardware_concurrency();
    return (int)std::max(1u, std::min(16u, hc ? hc : 1u));
  }();
  return n;
}
// Persistent worker pool: run_tasks(k, fn) executes fn(0) .. fn(k-1), one task per thread (the caller takes part),
// and returns when all are done.  The prologue has ~60 short parallel regions; spawning threads for each would cost
// about as much as the smaller regions themselves.  Workers spin briefly for the next region before they sleep.
// One region at a time (regions of concurrent callers are serialised); tasks must not start regions themselves.
namespace {
class Pool {
 public:
  // never destroyed: the workers sleep on the condition variable and end with the process (no join at exit, and a
  // fork()ed child -- which inherits the object but not the threads -- simply runs its regions inline)
  static Pool& get() { static Pool* p = new Pool; return *p; }
  void run_tasks(int k, const std::function<void(int)>& fn) {
    if (k <= 1 || workers_.empty() || dead_.load(std::memory_order_relaxed)) { for (int t = 0; t < k; t++) fn(t); return; }
    std::lock_guard<std::mutex> region(region_);
    unsigned long long g;
    {
      std::lock_guard<std::mutex> lk(m_);
      g = ++gen_;
      job_ = &fn; ntasks_ = k;
      remaining_.store(k, std::memory_order_relaxed);
      ticket_.store(g << 32, std::memory_order_release);
      wake_.store(g, std::memory_order_release);
    }
    cv_.notify_all();
    work(fn, k, g);
    // wait for the stragglers (short: spin, then yield)
    for (int spins = 0; remaining_.load(std::memory_order_acquire) > 0; spins++)
      if (spins > 2000) std::this_thread::yield();
    std::exception_ptr err;
    {
      std::lock_guard<std::mutex> lk(m_);
      job_ = nullptr;
      err = error_;
      error_ = nullptr;
    }
    if (err) std::rethrow_exception(err);   // first exception of any task, on the calling thread, after ALL tasks ended
  }
 private:
  Pool() {
    const int T = host_threads();
    for (int t = 1; t < T; t++) workers_.emplace_back([this] { loop(); });
    pthread_atfork(nullptr, nullptr, [] { Pool::get().dead_.store(true); });
  }
  // claim tasks of generation g only: a straggler of an earlier region can never take (or miscount) a task of the next
  void work(const std::function<void(int)>& fn, int k, unsigned long long g) {
    for (;;) {
      unsigned long long tk = ticket_.load(std::memory_order_acquire);
      if ((tk >> 32) != (g & 0xffffffffull)) return;
      const unsigned t = (unsigned)(tk & 0xffffffffull);
      if ((int)t >= k) return;
      if (!ticket_.compare_exchange_weak(tk, tk + 1, std::memory_order_acq_rel)) continue;
      try {
        fn((int)t);
      } catch (...) {   // e.g. std::bad_alloc in a task: hand it to the caller instead of std::terminate on a worker
        std::lock_guard<std::mutex> lk(m_);
        if (!error_) error_ = std::current_exception();
      }
      remaining_.fetch_sub(1, std::memory_order_acq_rel);
    }
  }
  void loop() {
    unsigned long long seen = 0;
    for (;;) {
      // spin a little for the next region, then sleep on the condition variable
      bool got = false;
      for (int spins = 0; spins < 30000; spins++) {
        if (wake_.load(std::memory_order_acquire) != seen) { got = true; break; }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
      }
      const std::function<void(int)>* job = nullptr;
      int k = 0;
      {
        std::unique_lock<std::mutex> lk(m_);
        if (!got) cv_.wait(lk, [&] { return wake_.load(std::memory_order_acquire) != seen; });
        seen = gen_;
        job = job_; k = ntasks_;
      }
      if (job) work(*job, k, seen);
    }
  }
  std::vector<std::thread> workers_;
  std::mutex m_, region_;
  std::condition_variable cv_;
  const std::function<void(int)>* job_ = nullptr;   // guarded by m_ (with gen_, ntasks_)
  int ntasks_ = 0;
  unsigned long long gen_ = 0;
  std::atomic<unsigned long long> wake_{0}, ticket_{0};
  std::atomic<int> remaining_{0};
  std::atomic<bool> dead_{false};
  std::exception_ptr error_;   // guarded by m_
};
}  // namespace

// fn(chunk_index, begin, end) over [0, count) cut into host_threads() contiguous chunks
void parallel_chunks(long long count, const std::function<void(int, long long, long long)>& fn, long long min_per_thread) {
  int T = host_threads();
  if (count < 2 * min_per_thread) T = 1;
  T = (int)std::min<long long>(T, std::max<long long>(1, count / min_per_thread));
  if (T <= 1) { fn(0, 0, count); return; }
  Pool::get().run_tasks(T, [&](int t) { fn(t, count * t / T, count * (t + 1) / T); });
}
// column chunks balanced by nonzeros: boundaries[t] .. boundaries[t+1]
static std::vector<int> balanced_columns(const std::vector<int>& cbeg, int n, int T) {
  std::vector<int> b(T + 1, n);
  b[0] = 0;
  const long long nnz = cbeg[n];
  for (int t = 1; t < T; t++) {
    const long long target = nnz * t / T;
    b[t] = (int)(std::lower_bound(cbeg.begin(), cbeg.begin() + n + 1, (int)target) - cbeg.begin());
    b[t] = std::max(b[t], b[t - 1]);
    b[t] = std::min(b[t], n);
  }
  return b;
}

// formulateLP_highs, CupdlpWrapper.cpp:280-448
void formulate(const b200pdlp_lp& lp, StdForm& f) {
  const int n0 = lp.num_col, m = lp.num_row;
  const int nnz0 = lp.a_start[n0];
  f = StdForm();
  f.n_orig = n0;
  f.m = m;
  f.sense = lp.sense;
  f.offset = lp.offset;
  f.row_class.resize(m);
  f.row_new_idx.resize(m);
  int n_eq_like = 0, n_bound = 0;
  for (int i = 0; i < m; i++) {
    const bool lo = lp.row_lower[i] > -1e20, up = lp.row_upper[i] < 1e20;  // :316-317
    RowClass c;
    if (lo && up && lp.row_lower[i] == lp.row_upper[i]) c = kEq;
    else if (lo && !up) c = kGeq;
    else if (!lo && up) c = kLeq;
    else c = kBound;  // ranged rows and (with a warning in the reference) free rows, :328-345
    f.row_class[i] = c;
    if (c == kEq || c == kBound) n_eq_like++;
    if (c == kBound) n_bound++;
  }
  f.neq = n_eq_like;
  f.n = n0 + n_bound;
  f.nnz = nnz0 + n_bound;
  // new row order: EQ/BOUND rows (original order), then LEQ/GEQ rows (:380-404)
  f.rhs.assign(m, 0.0);
  {
    int head = 0, tail = f.neq;
    for (int i = 0; i < m; i++) {
      switch (f.row_class[i]) {
        case kEq: f.rhs[head] = lp.row_lower[i]; f.row_new_idx[i] = head++; break;
        case kBound: f.rhs[head] = 0.0; f.row_new_idx[i] = head++; break;
        case kLeq: f.rhs[tail] = -lp.row_upper[i]; f.row_new_idx[i] = tail++; break;
        case kGeq: f.rhs[tail] = lp.row_lower[i]; f.row_new_idx[i] = tail++; break;
      }
    }
  }
  f.cost.assign(f.n, 0.0);
  f.lower.resize(f.n);
  f.upper.resize(f.n);
  for (int j = 0; j < n0; j++) {
    f.cost[j] = lp.col_cost[j] * lp.sense;
    f.lower[j] = lp.col_lower[j];
    f.upper[j] = lp.col_upper[j];
  }
  f.cbeg.resize(f.n + 1);
  f.cidx.resize(f.nnz);
  f.cval.resize(f.nnz);
  // structural columns: within a column EQ/BOUND entries first, then LEQ (negated) / GEQ (:410-433).
  // A structural column keeps its entry count, so column j starts at a_start[j]: columns are independent.
  parallel_chunks(n0, [&](int, long long j0, long long j1) {
    for (int j = (int)j0; j < (int)j1; j++) {
      int k = lp.a_start[j];
      f.cbeg[j] = k;
      for (int p = lp.a_start[j]; p < lp.a_start[j + 1]; p++) {
        const int c = f.row_class[lp.a_index[p]];
        if (c == kEq || c == kBound) { f.cidx[k] = f.row_new_idx[lp.a_index[p]]; f.cval[k] = lp.a_value[p]; k++; }
      }
      for (int p = lp.a_start[j]; p < lp.a_start[j + 1]; p++) {
        const int c = f.row_class[lp.a_index[p]];
        if (c == kLeq) { f.cidx[k] = f.row_new_idx[lp.a_index[p]]; f.cval[k] = -lp.a_value[p]; k++; }
        else if (c == kGeq) { f.cidx[k] = f.row_new_idx[lp.a_index[p]]; f.cval[k] = lp.a_value[p]; k++; }
      }
    }
  }, 4096);
  int k = nnz0;
  // one slack column per BOUND row: A x - z = 0, lo <= z <= up (:328-331,367-373,439-445)
  int j = n0;
  for (int i = 0; i < m; i++) {
    if (f.row_class[i] != kBound) continue;
    f.cbeg[j] = k;
    f.cidx[k] = f.row_new_idx[i];
    f.cval[k] = -1.0;
    k++;
    f.lower[j] = lp.row_lower[i];
    f.upper[j] = lp.row_upper[i];
    j++;
  }
  f.cbeg[f.n] = k;
  const double inf = std::numeric_limits<double>::infinity();
  for (int q = 0; q < f.n; q++) {  // :375-378
    if (f.lower[q] < -1e20) f.lower[q] = -inf;
    if (f.upper[q] > 1e20) f.upper[q] = inf;
  }
  // Init_Scaling (cupdlp_scaling.c:395-425): norms of the unscaled data, unit scales
  f.col_scale.assign(f.n, 1.0);
  f.row_scale.assign(f.m, 1.0);
  double s = 0.0;
  for (int q = 0; q < f.n; q++) s += f.cost[q] * f.cost[q];
  f.norm_cost = std::sqrt(s);
  s = 0.0;
  for (int i = 0; i < f.m; i++) s += f.rhs[i] * f.rhs[i];
  f.norm_rhs = std::sqrt(s);
}

// Counting-sort transposition of the nonzero pattern (what csc2csr / cupdlp_dcs_transpose do,
// cupdlp_cs.c:189-214), parallel: thread t histograms the rows of its column chunk, a prefix over
// (row, thread) gives every thread its private output range inside each row, and the scatter keeps
// the global column order.
void build_row_index(StdForm& f) {
  const int n = f.n, m = f.m;
  int T = (f.nnz < (1 << 18)) ? 1 : host_threads();
  while (T > 1 && (long long)T * m > (1LL << 27)) T /= 2;   // cap the T x m histogram at 512 MB
  const std::vector<int> cb = balanced_columns(f.cbeg, n, T);
  std::vector<std::vector<int>> hist(T);
  auto run = [&](const std::function<void(int)>& fn) { Pool::get().run_tasks(T, fn); };
  run([&](int t) {
    hist[t].assign(m, 0);
    for (int p = f.cbeg[cb[t]]; p < f.cbeg[cb[t + 1]]; p++) hist[t][f.cidx[p]]++;
  });
  f.rptr.assign(m + 1, 0);
  parallel_chunks(m, [&](int, long long b, long long e) {   // row totals (T x m reads) in parallel ...
    for (long long i = b; i < e; i++) {
      int c = 0;
      for (int t = 0; t < T; t++) c += hist[t][i];
      f.rptr[i + 1] = c;
    }
  });
  for (int i = 0; i < m; i++) f.rptr[i + 1] += f.rptr[i];   // ... then one short serial scan
  parallel_chunks(m, [&](int, long long b, long long e) {
    for (long long i = b; i < e; i++) {
      int off = f.rptr[i];
      for (int t = 0; t < T; t++) { const int c = hist[t][i]; hist[t][i] = off; off += c; }
    }
  });
  f.rpos.resize(f.nnz);
  f.rcol.resize(f.nnz);
  run([&](int t) {
    std::vector<int>& w = hist[t];
    for (int j = cb[t]; j < cb[t + 1]; j++)
      for (int p = f.cbeg[j]; p < f.cbeg[j + 1]; p++) {   // p ascending = columns ascending
        const int q = w[f.cidx[p]]++;
        f.rpos[q] = p;
        f.rcol[q] = j;
      }
  });
}

// PDHG_Scale_Data with Init_Scaling's fixed recipe: 10 inf-norm Ruiz passes, then
// Pock-Chambolle with alpha = 1 (cupdlp_scaling.c:47-120, 174-231, 395-409).
// Parallel layout: columns are cut into nnz-balanced chunks, one per thread.  Column norms are private to
// a chunk.  Row inf-norms (Ruiz) are gathered in per-thread arrays and merged with max (exact, order-free).
// The row 1-norms of the Pock-Chambolle pass must be added in the reference's order (columns ascending), so
// they are taken from a row-major index of the nonzeros (built once), one row per thread at a time.
void scale(StdForm& f, bool do_scale) {
  const int n = f.n, m = f.m;
  double amax = 0.0;
  if (!do_scale) {
    for (int p = 0; p < f.nnz; p++) amax = std::max(amax, std::fabs(f.cval[p]));
    f.amax = amax;
    return;
  }
  const bool timing = getenv("B200PDLP_TIMING") != nullptr;
  auto tprev = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) {
    if (!timing) return;
    const auto t1 = std::chrono::steady_clock::now();
    fprintf(stderr, "[b200pdlp scale] %-28s %8.1f ms\n", what, std::chrono::duration<double, std::milli>(t1 - tprev).count());
    tprev = t1;
  };
  const int T = (f.nnz < (1 << 18)) ? 1 : host_threads();
  const std::vector<int> cb = balanced_columns(f.cbeg, n, T);
  std::vector<double> cs(n), rs(m), cs_next(n);
  std::vector<std::vector<double>> rloc(T);           // per-thread row accumulators, first touched by their owner
  auto run_cols = [&](const std::function<void(int, int, int)>& fn) {   // fn(tid, col_begin, col_end)
    if (T == 1) { fn(0, 0, n); return; }
    Pool::get().run_tasks(T, [&](int t) { fn(t, cb[t], cb[t + 1]); });
  };
  auto merge_rows_max = [&](std::vector<double>& dst) {
    parallel_chunks(m, [&](int, long long b, long long e) {
      for (long long i = b; i < e; i++) {
        double v = rloc[0][i];
        for (int t = 1; t < T; t++) if (rloc[t][i] > v) v = rloc[t][i];
        dst[i] = v;
      }
    });
  };
  // row-major index of the nonzeros (position in cval), columns ascending within a row: for the exact row sums
  std::vector<int>& rptr = f.rptr;
  RawVec<int>& rpos = f.rpos;
  // norms for the first Ruiz pass
  run_cols([&](int t, int c0, int c1) {
    std::vector<double>& r = rloc[t];
    r.assign(m, 0.0);
    for (int j = c0; j < c1; j++) {
      double mx = 0.0;
      for (int p = f.cbeg[j]; p < f.cbeg[j + 1]; p++) {
        const double a = std::fabs(f.cval[p]);
        if (a > mx) mx = a;
        if (r[f.cidx[p]] < a) r[f.cidx[p]] = a;
      }
      cs[j] = mx;
    }
  });
  merge_rows_max(rs);
  lap("first norms");
  const int kRuiz = 10;
  std::vector<double> amax_t(T, 0.0);
  for (int it = 0; it <= kRuiz; it++) {
    // turn the gathered norms into this pass's factors (sqrt, with 0 -> 1) and apply them to the vectors
    parallel_chunks(n, [&](int, long long b, long long e) {
      for (long long j = b; j < e; j++) {
        const double v = std::sqrt(cs[j]);
        const double c = (v == 0.0) ? 1.0 : v;
        cs[j] = c;
        f.cost[j] /= c; f.lower[j] *= c; f.upper[j] *= c; f.col_scale[j] *= c;
      }
    });
    parallel_chunks(m, [&](int, long long b, long long e) {
      for (long long i = b; i < e; i++) {
        const double r = (rs[i] == 0.0) ? 1.0 : std::sqrt(rs[i]);
        rs[i] = r;
        f.rhs[i] /= r; f.row_scale[i] *= r;
      }
    });
    const bool next_is_pc = (it == kRuiz - 1);  // after the 10th Ruiz pass gather 1-norms
    const bool last = (it == kRuiz);            // the Pock-Chambolle pass itself
    run_cols([&](int t, int c0, int c1) {
      std::vector<double>& rn = rloc[t];
      if (!last && !next_is_pc) std::fill(rn.begin(), rn.end(), 0.0);
      double am = 0.0;
      for (int j = c0; j < c1; j++) {
        double acc = 0.0;
        const double cj = cs[j];
        for (int p = f.cbeg[j]; p < f.cbeg[j + 1]; p++) {
          const int i = f.cidx[p];
          double v = f.cval[p] / rs[i];   // row division first, then column division (:33-41)
          v /= cj;
          f.cval[p] = v;
          const double a = std::fabs(v);
          if (last) { if (a > am) am = a; }
          else if (next_is_pc) { acc += a; }
          else { if (a > acc) acc = a; if (rn[i] < a) rn[i] = a; }
        }
        cs_next[j] = acc;
      }
      amax_t[t] = am;
    });
    lap(last ? "final sweep" : "sweep");
    if (last) break;
    if (next_is_pc) {
      // exact row 1-norms in the reference's summation order
      if (rptr.empty()) { build_row_index(f); lap("row index"); }
      parallel_chunks(m, [&](int, long long b, long long e) {
        for (long long i = b; i < e; i++) {
          double sum = 0.0;
          for (int q = rptr[i]; q < rptr[i + 1]; q++) sum += std::fabs(f.cval[rpos[q]]);
          rs[i] = sum;
        }
      });
      lap("row 1-norms");
    } else {
      merge_rows_max(rs);
      lap("merge");
    }
    cs.swap(cs_next);
  }
  for (int t = 0; t < T; t++) amax = std::max(amax, amax_t[t]);
  f.amax = amax;
}

std::vector<int> partition_rows(const StdForm& f, int world) {
  std::vector<long long> cnt(f.m + 1, 0);
  for (int p = 0; p < f.nnz; p++) cnt[f.cidx[p] + 1]++;
  for (int i = 0; i < f.m; i++) cnt[i + 1] += cnt[i];
  std::vector<int> b(world + 1, 0);
  b[world] = f.m;
  // balance nnz + a per-row cost (vector traffic ~ 7 doubles per row ~ 5 nonzeros)
  const long long total = cnt[f.m] + 5LL * f.m;
  for (int g = 1; g < world; g++) {
    const long long target = total * g / world;
    int lo = b[g - 1], hi = f.m;
    while (lo < hi) {
      const int mid = (lo + hi) / 2;
      if (cnt[mid] + 5LL * mid < target) lo = mid + 1; else hi = mid;
    }
    b[g] = lo;
  }
  return b;
}

void build_row_major(const StdForm& f, int r0, int r1, Csr& a) {
  a = Csr();
  a.nrows = r1 - r0;
  a.ncols = f.n;
  if (!f.rptr.empty() && (int)f.rptr.size() == f.m + 1) {
    // gather the values through the row-major index (parallel); the columns were recorded when it was built
    a.rowptr.resize(a.nrows + 1);
    const int base = f.rptr[r0];
    for (int i = 0; i <= a.nrows; i++) a.rowptr[i] = f.rptr[r0 + i] - base;
    a.nnz = a.rowptr[a.nrows];
    a.col.resize(a.nnz);
    a.val.resize(a.nnz);
    parallel_chunks(a.nnz, [&](int, long long q0, long long q1) {
      for (long long q = q0; q < q1; q++) { a.col[q] = f.rcol[base + q]; a.val[q] = f.cval[f.rpos[base + q]]; }
    });
    return;
  }
  a.rowptr.assign(a.nrows + 1, 0);
  for (int p = 0; p < f.nnz; p++) { const int i = f.cidx[p]; if (i >= r0 && i < r1) a.rowptr[i - r0 + 1]++; }
  for (int i = 0; i < a.nrows; i++) a.rowptr[i + 1] += a.rowptr[i];
  a.nnz = a.rowptr[a.nrows];
  a.col.assign(a.nnz, 0);
  a.val.assign(a.nnz, 0.0);
  std::vector<int> w(a.rowptr.begin(), a.rowptr.end() - 1);
  for (int j = 0; j < f.n; j++)
    for (int p = f.cbeg[j]; p < f.cbeg[j + 1]; p++) {
      const int i = f.cidx[p];
      if (i < r0 || i >= r1) continue;
      const int q = w[i - r0]++;
      a.col[q] = j;
      a.val[q] = f.cval[p];
    }
}

void build_col_major(const StdForm& f, int r0, int r1, Csr& at) {
  // rows of A^T = columns of A restricted to rows [r0,r1), entries sorted by row
  // (the order in which the reference's row-scatter A^T y accumulates, cupdlp_linalg.c:73-109)
  at = Csr();
  at.nrows = f.n;
  at.ncols = r1 - r0;
  if (r0 == 0 && r1 == f.m) {
    at.rowptr.assign(f.cbeg.begin(), f.cbeg.begin() + f.n + 1);   // all rows: the column lengths themselves
  } else {
    std::vector<int> cnt(f.n, 0);
    parallel_chunks(f.n, [&](int, long long j0, long long j1) {
      for (int j = (int)j0; j < (int)j1; j++) {
        int c = 0;
        for (int p = f.cbeg[j]; p < f.cbeg[j + 1]; p++) c += (f.cidx[p] >= r0 && f.cidx[p] < r1);
        cnt[j] = c;
      }
    }, 4096);
    at.rowptr.assign(f.n + 1, 0);
    for (int j = 0; j < f.n; j++) at.rowptr[j + 1] = at.rowptr[j] + cnt[j];
  }
  at.nnz = at.rowptr[f.n];
  at.col.resize(at.nnz);   // uninitialised: every entry is written by the loop below
  at.val.resize(at.nnz);
  parallel_chunks(f.n, [&](int, long long j0, long long j1) {
  std::vector<std::pair<int, double>> tmp;
  for (int j = (int)j0; j < (int)j1; j++) {
    int q = at.rowptr[j];
    bool sorted = true;
    int prev = -1;
    for (int p = f.cbeg[j]; p < f.cbeg[j + 1]; p++) {
      const int i = f.cidx[p];
      if (i < r0 || i >= r1) continue;
      if (i < prev) sorted = false;
      prev = i;
      at.col[q] = i - r0;
      at.val[q] = f.cval[p];
      q++;
    }
    if (!sorted) {
      tmp.clear();
      for (int t = at.rowptr[j]; t < q; t++) tmp.emplace_back(at.col[t], at.val[t]);
      std::stable_sort(tmp.begin(), tmp.end(), [](const std::pair<int, double>& a, const std::pair<int, double>& b) { return a.first < b.first; });
      for (size_t t = 0; t < tmp.size(); t++) { at.col[at.rowptr[j] + t] = tmp[t].first; at.val[at.rowptr[j] + t] = tmp[t].second; }
    }
  }
  });
}

std::vector<int> make_perm(const std::vector<int>& rowptr, int boundary, bool sort) {
  const int n = (int)rowptr.size() - 1;
  std::vector<int> perm(n);
  for (int i = 0; i < n; i++) perm[i] = i;
  if (!sort) return perm;
  auto len = [&](int r) { return rowptr[r + 1] - rowptr[r]; };
  auto sort_range = [&](int b, int e) {
    const long long nwin = ((long long)(e - b) + kSortWindow - 1) / kSortWindow;
    parallel_chunks(nwin, [&](int, long long w0, long long w1) {
      for (long long wi = w0; wi < w1; wi++) {
        const int w = b + (int)wi * kSortWindow;
        const int we = std::min(w + kSortWindow, e);
        std::stable_sort(perm.begin() + w, perm.begin() + we, [&](int x, int y) { return len(x) > len(y); });
      }
    }, 4);
  };
  boundary = std::max(0, std::min(boundary, n));
  sort_range(0, boundary);
  sort_range(boundary, n);
  return perm;
}

std::vector<int> invert_perm(const std::vector<int>& perm) {
  std::vector<int> inv(perm.size());
  for (size_t i = 0; i < perm.size(); i++) inv[perm[i]] = (int)i;
  return inv;
}

// The PLAN of a sliced-ELL matrix depends only on the row lengths: slice offsets and lengths, masked lanes, long-row
// segments and their offsets in the long-row arrays.  The arrays themselves are filled afterwards -- by the host
// (fill_sell_host) or, given the plan, by a device kernel that reads the scaled matrix where it already lies in HBM.
void plan_sell(int nrows, int ncols, long long nnz, const std::vector<int>& perm, const std::function<int(int)>& old_row_len,
               int long_threshold, SellMatrix& out) {
  out = SellMatrix();
  out.nrows = nrows;
  out.ncols = ncols;
  out.nnz = nnz;
  const int nslices = (nrows + 31) / 32;
  out.slices.resize(nslices);
  auto len = [&](int newrow) { return old_row_len(perm[newrow]); };
  long long total = 0;
  for (int s = 0; s < nslices; s++) {
    int mx = 0;
    unsigned mask = 0;
    for (int l = 0; l < 32; l++) {
      const int nr = s * 32 + l;
      if (nr >= nrows) { mask |= 1u << l; continue; }
      const int ln = len(nr);
      if (ln > long_threshold) { mask |= 1u << l; continue; }
      mx = std::max(mx, ln);
    }
    if (total + 32LL * mx > 2000000000LL) throw std::runtime_error("b200pdlp: matrix too large for 32-bit slice offsets");
    out.slices[s] = {(int)total, mx, mask, 0};
    total += 32LL * mx;
  }
  out.padded = total;
  // long rows -> segments of kNnzPerBlock entries; a row's entries start 16-byte aligned in lcol / lval
  long long lpos = 0;
  for (int nr = 0; nr < nrows; nr++) {
    const int ln = len(nr);
    if (ln <= long_threshold) continue;
    const int nseg = (ln + kNnzPerBlock - 1) / kNnzPerBlock;
    const int base = (int)lpos;
    out.long_rows.push_back({nr, (int)out.segs.size(), nseg, out.n_partials});
    for (int sg = 0; sg < nseg; sg++)
      out.segs.push_back({nr, base + sg * kNnzPerBlock, std::min(base + (sg + 1) * kNnzPerBlock, base + ln), (int)out.long_rows.size() - 1});
    out.n_partials += nseg;
    lpos += ln;
    lpos = (lpos + 3) / 4 * 4;
    if (lpos > 2000000000LL) throw std::runtime_error("b200pdlp: long rows too large for 32-bit offsets");
  }
  out.lcount = lpos + 8;
}

void fill_sell_host(const Csr& a, const std::vector<int>& perm, const std::vector<int>& colmap, SellMatrix& out) {
  const long long total = out.padded;
  const int nslices = (int)out.slices.size();
  out.col.resize((size_t)total + 32);   // uninitialised: every slot is written below, by the thread that owns the slice
  out.val.resize((size_t)total + 32);
  for (int q = 0; q < 32; q++) { out.col[(size_t)total + q] = 0; out.val[(size_t)total + q] = 0.0; }
  parallel_chunks(nslices, [&](int, long long s0, long long s1) {
    for (long long s = s0; s < s1; s++) {
      const SellMatrix::Slice& sl = out.slices[s];
      for (int l = 0; l < 32; l++) {
        int k = 0;
        if (!((sl.skipmask >> l) & 1u)) {
          const int r = perm[s * 32 + l];
          for (int p = a.rowptr[r]; p < a.rowptr[r + 1]; p++, k++) {
            out.col[(size_t)sl.ptr + 32 * (size_t)k + l] = colmap[a.col[p]];
            out.val[(size_t)sl.ptr + 32 * (size_t)k + l] = a.val[p];
          }
        }
        for (; k < sl.len; k++) {   // padding
          out.col[(size_t)sl.ptr + 32 * (size_t)k + l] = 0;
          out.val[(size_t)sl.ptr + 32 * (size_t)k + l] = 0.0;
        }
      }
    }
  }, 256);
  out.lcol.assign((size_t)out.lcount, 0);
  out.lval.assign((size_t)out.lcount, 0.0);
  for (const SellMatrix::LongRow& lr : out.long_rows) {
    const int r = perm[lr.row];
    int q = out.segs[lr.first_seg].nnz_begin;
    for (int p = a.rowptr[r]; p < a.rowptr[r + 1]; p++, q++) { out.lcol[q] = colmap[a.col[p]]; out.lval[q] = a.val[p]; }
  }
}

void build_sell(const Csr& a, const std::vector<int>& perm, const std::vector<int>& colmap, int long_threshold,
                SellMatrix& out) {
  plan_sell(a.nrows, a.ncols, a.nnz, perm, [&](int r) { return a.rowptr[r + 1] - a.rowptr[r]; }, long_threshold, out);
  fill_sell_host(a, perm, colmap, out);
}

void build_layout(StdForm& f, int rank, int world, int ordered_max, HostLayout& L,
                  const std::function<void(const char*)>& lap, bool plan_only) {
  auto mark = [&](const char* what) { if (lap) lap(what); };
  L = HostLayout();
  L.rank = rank; L.world = world;
  L.bounds = partition_rows(f, world);
  L.r0 = L.bounds[rank]; L.r1 = L.bounds[rank + 1];
  L.ml = L.r1 - L.r0;
  const int n = f.n, ml = L.ml;
  {
    const int omax = ordered_max == 0 ? 4096 : ordered_max;
    L.ordered = world == 1 && omax > 0 && std::max(f.n, f.m) <= omax;
  }
  const bool sort = !L.ordered;
  const int long_threshold = L.ordered ? std::numeric_limits<int>::max() : 512;
  L.neq_local = std::max(0, std::min(f.neq - L.r0, ml));
  Csr at;
  if (f.rptr.empty()) build_row_index(f);
  if (plan_only) {
    if (world != 1) throw std::runtime_error("b200pdlp: plan-only layouts are single-GPU");
    L.rperm = make_perm(f.rptr, L.neq_local, sort);
    L.cperm = make_perm(f.cbeg, n, sort);
    L.rinv = invert_perm(L.rperm);
    L.cinv = invert_perm(L.cperm);
    mark("length sorts");
    L.nl = L.nl_real = n; L.c0 = 0; L.shard_len = n; L.seg_len = n;
    plan_sell(f.m, n, f.nnz, L.rperm, [&](int r) { return f.rptr[r + 1] - f.rptr[r]; }, long_threshold, L.A);
    plan_sell(n, f.m, f.nnz, L.cperm, [&](int j) { return f.cbeg[j + 1] - f.cbeg[j]; }, long_threshold, L.AT);
    L.csr_local.nrows = f.m; L.csr_local.ncols = n; L.csr_local.nnz = f.nnz;   // dimensions only
    mark("sliced-ELL plan");
    return;
  }
  build_row_major(f, L.r0, L.r1, L.csr_local);
  mark("row-major transpose");
  build_col_major(f, L.r0, L.r1, at);
  mark("col-major copy");
  L.rperm = make_perm(L.csr_local.rowptr, L.neq_local, sort);
  L.cperm = make_perm(f.cbeg, n, sort);   // GLOBAL column lengths: identical on every rank
  L.rinv = invert_perm(L.rperm);
  L.cinv = invert_perm(L.cperm);
  mark("length sorts");
  if (world == 1) {
    L.nl = L.nl_real = n; L.c0 = 0; L.shard_len = n; L.seg_len = n;
    build_sell(L.csr_local, L.rperm, L.cinv, long_threshold, L.A);
    build_sell(at, L.cperm, L.rinv, long_threshold, L.AT);
  } else {
    L.shard_len = ((n + world - 1) / world + 1) & ~1;          // even: 16-byte aligned segments
    L.seg_len = L.shard_len + 2;
    L.nl = L.shard_len;
    L.c0 = rank * L.shard_len;
    L.nl_real = std::max(0, std::min(L.shard_len, n - L.c0));
    std::vector<int> colpos(n);                                   // old column -> position in the segmented x
    for (int j = 0; j < n; j++) colpos[j] = (int)L.seg_pos(L.cinv[j]);
    build_sell(L.csr_local, L.rperm, colpos, long_threshold, L.A);
    L.A.ncols = world * L.seg_len;   // column ids are positions in the segmented x
    // rows of A_g^T in an order sorted by LOCAL length (windows of the global device order, so that
    // nearby outputs stay nearby); the kernel writes through at_outpos
    std::vector<int> ordered_rowptr(n + 1, 0);
    for (int j = 0; j < n; j++) ordered_rowptr[j + 1] = ordered_rowptr[j] + (at.rowptr[L.cperm[j] + 1] - at.rowptr[L.cperm[j]]);
    const std::vector<int> local = make_perm(ordered_rowptr, n, true);   // positions in device order
    std::vector<int> at_perm(n);
    L.at_outpos.resize(n);
    for (int r = 0; r < n; r++) { at_perm[r] = L.cperm[local[r]]; L.at_outpos[r] = (int)L.seg_pos(local[r]); }
    build_sell(at, at_perm, L.rinv, long_threshold, L.AT);
  }
  mark("sliced-ELL build");
}

// offsets of `world` contiguous blocks of perm[0..count) balancing entries + a per-row cost (as partition_rows does)
static std::vector<int> balanced_blocks(const std::vector<int>& ptr, const std::vector<int>& perm, int world) {
  const int count = (int)perm.size();
  std::vector<long long> pre(count + 1, 0);
  for (int i = 0; i < count; i++) pre[i + 1] = pre[i] + (ptr[perm[i] + 1] - ptr[perm[i]]) + 5;
  std::vector<int> b(world + 1, 0);
  b[world] = count;
  for (int g = 1; g < world; g++) {
    const long long target = pre[count] * g / world;
    b[g] = (int)(std::lower_bound(pre.begin() + b[g - 1], pre.end(), target) - pre.begin());
    b[g] = std::min(b[g], count);
  }
  return b;
}

void plan_hipdlp_shards(StdForm& f, int world, int ordered_max, HipShards& S) {
  S = HipShards();
  S.world = world;
  HostLayout L;   // the one-GPU orders (the plan-only build computes exactly the full build's orderings)
  build_layout(f, 0, 1, ordered_max, L, nullptr, /*plan_only=*/true);
  S.ordered = L.ordered;
  S.long_threshold = L.ordered ? std::numeric_limits<int>::max() : 512;
  S.rperm = std::move(L.rperm); S.rinv = std::move(L.rinv);
  S.cperm = std::move(L.cperm); S.cinv = std::move(L.cinv);
  build_row_major(f, 0, f.m, S.a);
  build_col_major(f, 0, f.m, S.at);
  S.rb = balanced_blocks(S.a.rowptr, S.rperm, world);
  S.cb = balanced_blocks(S.at.rowptr, S.cperm, world);
}

void build_hipdlp_shard(const HipShards& S, int rank, SellMatrix& A, SellMatrix& AT) {
  auto build = [&](const Csr& a, const std::vector<int>& order, int b0, int b1, const std::vector<int>& colmap, SellMatrix& out) {
    const std::vector<int> perm(order.begin() + b0, order.begin() + b1);
    long long nnz = 0;
    for (int r : perm) nnz += a.rowptr[r + 1] - a.rowptr[r];
    plan_sell(b1 - b0, a.ncols, nnz, perm, [&](int r) { return a.rowptr[r + 1] - a.rowptr[r]; }, S.long_threshold, out);
    fill_sell_host(a, perm, colmap, out);
  };
  build(S.a, S.rperm, S.rb[rank], S.rb[rank + 1], S.cinv, A);
  build(S.at, S.cperm, S.cb[rank], S.cb[rank + 1], S.rinv, AT);
}

void sell_apply_host(const SellMatrix& a, const double* xin, double* out) {
  // exactly what spmv_sell_kernel does: EVERY lane of a slice runs over the slice's full length (padding included),
  // so padding must be (col 0, val 0) and every column id must be a valid position of the input vector
  const int nslices = (int)a.slices.size();
  for (int s = 0; s < nslices; s++) {
    const SellMatrix::Slice& sl = a.slices[s];
    for (int l = 0; l < 32; l++) {
      const int row = s * 32 + l;
      const bool live = row < a.nrows && !((sl.skipmask >> l) & 1u);
      double acc = 0.0;
      for (int k = 0; k < sl.len; k++) {
        const size_t q = (size_t)sl.ptr + 32 * (size_t)k + l;
        if (q >= a.col.size() || a.col[q] < 0 || a.col[q] >= a.ncols)
          throw std::runtime_error("sliced ELL: column id outside the input vector");
        if (!live && (a.val[q] != 0.0 || a.col[q] != 0)) throw std::runtime_error("sliced ELL: padding is not (0, 0)");
        acc += a.val[q] * xin[a.col[q]];
      }
      if (live) out[row] = acc;
    }
  }
  for (const SellMatrix::LongRow& lr : a.long_rows) {
    double total = 0.0;
    for (int sg = 0; sg < lr.nseg; sg++) {
      const SellMatrix::Seg& g = a.segs[lr.first_seg + sg];
      double part = 0.0;
      for (int q = g.nnz_begin; q < g.nnz_end; q++) {
        if (a.lcol[q] < 0 || a.lcol[q] >= a.ncols) throw std::runtime_error("sliced ELL: long-row column id outside the input vector");
        part += a.lval[q] * xin[a.lcol[q]];
      }
      total += part;
    }
    out[lr.row] = total;
  }
}

}  // namespace b200
