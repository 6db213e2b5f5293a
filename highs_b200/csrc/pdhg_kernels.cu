// highs_b200/csrc/pdhg_kernels.cu -- kernel definitions + launchers (see kernels.cuh).
#include "pdhg_arith.cuh"
#include "pdhg_kernels.hpp"

namespace b200 {

// =============================================================== K1: primal step
// PDHG_primalGradientStep (CPU operation order, cupdlp_step.c:28-38):
//   x' = x; x' += (-tau) c; x' += tau aty; x' = min(x', u); x' = max(x', l)
// fused with |x - x'|^2 (cupdlp_linalg.c:790) and the deferred average update
// xSum += w x (PDHG_Update_Average, cupdlp_step.c:436) of the previous accepted step.
__global__ void __launch_bounds__(kThreads)
primal_step_kernel(int n, PdhgState* __restrict__ st, double* __restrict__ x0, double* __restrict__ x1,
                   const double* __restrict__ aty0, const double* __restrict__ aty1,
                   const double* __restrict__ c, const double* __restrict__ lo, const double* __restrict__ up,
                   double* __restrict__ xsum, ReduceScratch rs, unsigned* __restrict__ xnz) {
  if (st->iter >= st->stop_iter) return;
  const int cur = st->cur;
  const double tau = st->tau_try, ntau = -tau;
  const bool pend = st->pending != 0;
  const double w = st->w_pending;
  const double* __restrict__ x = cur ? x1 : x0;
  double* __restrict__ xn = cur ? x0 : x1;
  const double* __restrict__ aty = cur ? aty1 : aty0;
  double acc[1] = {0.0};
  auto one = [&](double xc, double ci, double ai, double u, double l, double& out) {
    return primal_update(xc, ci, ai, u, l, tau, ntau, out);
  };
  // pairs of elements with 128-bit loads/stores (all vectors are cudaMalloc-aligned); the loop runs warp-uniformly so that
  // a warp's 64 entries give two words of the nonzero bitmap (DevSell::nzmap) of x'
  const int npair = n >> 1, nq = (n + 1) >> 1;
  const int lane = threadIdx.x & 31;
  const int stride = gridDim.x * kThreads;
  for (int i0 = blockIdx.x * kThreads + (threadIdx.x & ~31); i0 < nq; i0 += stride) {
    const int i = i0 + lane;
    unsigned nz = 3u;   // two bits: entries 2i, 2i + 1 (1 = may be nonzero; past the end nothing reads them)
    if (i < npair) {
      const double2 xc = reinterpret_cast<const double2*>(x)[i];
      const double2 ci = reinterpret_cast<const double2*>(c)[i];
      const double2 ai = reinterpret_cast<const double2*>(aty)[i];
      const double2 u = reinterpret_cast<const double2*>(up)[i];
      const double2 l = reinterpret_cast<const double2*>(lo)[i];
      if (pend) {
        double2 sm = reinterpret_cast<double2*>(xsum)[i];
        sm.x = sm.x + w * xc.x;
        sm.y = sm.y + w * xc.y;
        reinterpret_cast<double2*>(xsum)[i] = sm;
      }
      double2 o;
      const double t0 = one(xc.x, ci.x, ai.x, u.x, l.x, o.x);
      const double t1 = one(xc.y, ci.y, ai.y, u.y, l.y, o.y);
      reinterpret_cast<double2*>(xn)[i] = o;
      add_term(acc[0], t0, rs, 0, 2 * i);
      add_term(acc[0], t1, rs, 0, 2 * i + 1);
      nz = (o.x != 0.0 ? 1u : 0u) | (o.y != 0.0 ? 2u : 0u);
    } else if (i < nq && xnz) {
      // odd n: x'[n - 1] is written (and summed) by block 0 below; the same arithmetic here gives its bit without a race
      // on the bitmap word
      double o;
      one(x[n - 1], c[n - 1], aty[n - 1], up[n - 1], lo[n - 1], o);
      nz = (o != 0.0 ? 1u : 0u) | 2u;
    }
    if (xnz) {
      const unsigned sh = nz << (2 * (lane & 15));
      const unsigned w_lo = __reduce_or_sync(0xffffffffu, lane < 16 ? sh : 0u);
      const unsigned w_hi = __reduce_or_sync(0xffffffffu, lane < 16 ? 0u : sh);
      const int wd = i0 >> 4;   // entries 2 i0 .. 2 i0 + 63
      if (lane == 0) xnz[wd] = w_lo;
      if (lane == 16 && 32 * (wd + 1) < n) xnz[wd + 1] = w_hi;
    }
  }
  if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
    const int i = n - 1;
    const double xc = x[i];
    if (pend) xsum[i] = xsum[i] + w * xc;
    double o;
    const double t = one(xc, c[i], aty[i], up[i], lo[i], o);
    xn[i] = o;
    add_term(acc[0], t, rs, 0, i);
  }
  block_partials<1>(acc, rs);
}

// where an epilogue's terms go: a plain array (registers) or one thread's column of a [NACC][kThreads] shared-memory
// array (consecutive threads -> consecutive doubles: conflict-free; a [kThreads][NACC] row per thread would put a warp's
// 32 stores NACC doubles apart, into the same banks)
struct StridedOut {
  double* p;
  __device__ __forceinline__ double& operator[](int a) const { return p[a * kThreads]; }
  __device__ __forceinline__ StridedOut operator+(int k) const { return StridedOut{p + k * kThreads}; }
};
// an epilogue that has slice_end(slice, live) gets it after every slice of the body, with the whole warp converged
template <class E, class = void> struct HasSliceEnd { static constexpr bool value = false; };
template <class E> struct HasSliceEnd<E, decltype(void(&E::slice_end))> { static constexpr bool value = true; };
template <class Epi>
__device__ __forceinline__ void slice_end(const Epi& e, int slice, bool live) {
  if constexpr (HasSliceEnd<Epi>::value) e.slice_end(slice, live);
}
// ===================================================================== SpMV
// Sliced-ELL body: one warp per slice of 32 rows, one lane per row.  A warp reads the slice's
// col / val arrays fully coalesced (k-major, lane-minor), every lane gathers its dense-vector
// entry through L2 and accumulates ITS row in a register, in the row's own entry order -- the
// order in which the reference's scatter SpMV adds into that output entry (cupdlp_linalg.c:17-33)
// -- then runs the fused epilogue on the finished row sum.  No shared memory, no shuffles: the
// L1TEX pipe only sees the coalesced streams and the (irreducible) one-line-per-lane gathers.
// Rows longer than the long-row threshold live outside the body as segments of kNnzBlk nonzeros
// (one CTA each, tree-summed); the last segment of a row to finish combines the partial sums in
// segment order and runs the epilogue, whose terms go to the partial-sum slot of the row's first segment.
// `due` != nullptr: speculative check-iteration launch -- run only if the check iteration has been reached
__device__ __forceinline__ bool check_not_due(const PdhgState* due) { return due && (due->done || due->iter < due->stop_iter); }

struct PlainEpilogue {
  static constexpr int NACC = 0;
  const double* __restrict__ in;
  double* __restrict__ out;
  const PdhgState* due;
  __device__ bool begin() { return !check_not_due(due); }
  __device__ const double* input() const { return in; }
  __device__ void prefetch(int) {}
  __device__ void row(int r, double s, double*) const { out[r] = s; }
};

// K2: PDHG_dualGradientStep (CPU order, cupdlp_step.c:55-67):
//   y' = y; y' += sigma b; y' += (-2 sigma) ax'; y' += sigma ax; y'[i>=nEqs] = max(y',0)
// + |y - y'|^2 + deferred ySum += w y.
template <int NACC_>
struct DualEpilogueT {
  static constexpr int NACC = NACC_;
  PdhgState* st;
  const double *x0, *x1;       // primal double buffer (input = the NEW x)
  double *y0, *y1, *ax0, *ax1;
  const double* b;
  double* ysum;
  int neq, row_offset;         // neq = number of LOCAL equality rows (they come first); row_offset unused
  double* axsum;               // A xSum, carried while the checks are dense (PdhgState::light_on); may be nullptr
  unsigned* ynz;               // nonzero bitmap of y' (DevSell::nzmap of A'), one word per slice; may be nullptr
  // cached from the state block by begin()
  const double *y, *ax;
  double *yn, *axn;
  double sigma, w;
  bool pend, accum;
  __device__ bool begin() {
    if (st->iter >= st->stop_iter) return false;
    const int cur = st->cur;
    y = cur ? y1 : y0; yn = cur ? y0 : y1;
    ax = cur ? ax1 : ax0; axn = cur ? ax0 : ax1;
    sigma = st->sigma_try; w = st->w_pending; pend = st->pending != 0;
    accum = pend && axsum != nullptr && st->light_on && st->iter < kDenseChecks;
    x0 = cur ? x0 : x1;   // x0 now = input vector (the NEW x)
    return true;
  }
  __device__ const double* input() const { return x0; }
  // the row's epilogue operands are requested BEFORE the gather loop so that they arrive under it
  double p_y, p_b, p_ax, p_ys, p_axs;
  __device__ void prefetch(int r) {
    p_y = y[r]; p_b = b[r]; p_ax = ax[r];
    p_ys = pend ? ysum[r] : 0.0;
    p_axs = accum ? axsum[r] : 0.0;
  }
  bool nz;
  __device__ void row(int r, double s, double* t) {
    axn[r] = s;
    const double yc = p_y;
    if (pend) ysum[r] = p_ys + w * yc;
    if (accum) axsum[r] = p_axs + w * p_ax;   // A xSum += w A x  (x = the iterate accepted by the previous pass)
    const double v = dual_update(yc, p_b, s, p_ax, sigma, r >= neq);
    yn[r] = v;
    nz = v != 0.0;
    const double d = yc - v;
    t[0] = d * d;
    if (NACC > 1) t[NACC - 1] = (p_ax - s) * d;   // row-side interaction (AΔx)·Δy, multi-GPU only
  }
  // after a slice's rows (the whole warp, lane = row of the slice): the slice's word of the bitmap.  Lanes without a live
  // row write 1 -- among them the long rows, whose y' the segment finisher writes later in this launch.
  __device__ void slice_end(int slice, bool live) const {
    if (!ynz) return;
    const unsigned bits = __ballot_sync(0xffffffffu, !live || nz);
    if ((threadIdx.x & 31) == 0) ynz[slice] = bits;
  }
};
using DualEpilogue = DualEpilogueT<1>;
using DualEpilogueMg = DualEpilogueT<2>;

// K3: aty' = A'y' fused with the interaction (x - x').(aty - aty')
// (cupdlp_compute_interaction_and_movement, cupdlp_linalg.c:772-801); K4 adds the block partials.
struct PrimalEpilogue {
  static constexpr int NACC = 1;
  PdhgState* st;
  const double *y0, *y1;       // dual double buffer (input = the NEW y)
  const double *x0, *x1;
  double *aty0, *aty1;
  double* atysum;              // A'ySum, carried while the checks are dense (PdhgState::light_on); may be nullptr
  const double *x, *xn, *aty;
  double* atyn;
  double w;
  bool accum;
  __device__ bool begin() {
    if (st->iter >= st->stop_iter) return false;
    const int cur = st->cur;
    x = cur ? x1 : x0; xn = cur ? x0 : x1;
    aty = cur ? aty1 : aty0; atyn = cur ? aty0 : aty1;
    y0 = cur ? y0 : y1;   // y0 now = input vector (the NEW y)
    w = st->w_pending;
    accum = st->pending != 0 && atysum != nullptr && st->light_on && st->iter < kDenseChecks;
    return true;
  }
  __device__ const double* input() const { return y0; }
  double p_x, p_xn, p_aty, p_as;
  __device__ void prefetch(int r) { p_x = x[r]; p_xn = xn[r]; p_aty = aty[r]; p_as = accum ? atysum[r] : 0.0; }
  __device__ void row(int r, double s, double* t) const {
    atyn[r] = s;
    if (accum) atysum[r] = p_as + w * p_aty;   // A'ySum += w A'y
    const double dx = p_x - p_xn;
    const double da = p_aty - s;
    t[0] = dx * da;
  }
};

// K4: one CTA adds the block partials of K1 (|dx|^2), K2 (|dy|^2) and K3 (interaction) in a fixed
// order -- or, in ordered mode, the per-element terms in index order -- and applies the step rule.
// dy2_override != nullptr (multi-GPU): |dy|^2 is the all-reduced scalar instead of local partials.
constexpr int kStepThreads = 1024;
__global__ void __launch_bounds__(kStepThreads)
step_rule_kernel(PdhgState* __restrict__ st, ReduceScratch r1, int nb1, ReduceScratch r2, int nb2, ReduceScratch r3,
                 int nb3, const double* __restrict__ dy2_override) {
  __shared__ double sm[3][kStepThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double tot[3];
  if (r1.terms) {
    // ordered mode: thread a adds accumulator a's terms sequentially
    if (st->iter >= st->stop_iter) return;
    double s = 0.0;
    if (threadIdx.x < 3) {
      // (selected field by field: taking the parameters' addresses would copy all three to the stack first)
      const double* t = threadIdx.x == 0 ? r1.terms : (threadIdx.x == 1 ? r2.terms : r3.terms);
      const int len = threadIdx.x == 0 ? r1.len : (threadIdx.x == 1 ? r2.len : r3.len);
      for (int i = 0; i < len; i++) s += t[i];
      sm[threadIdx.x][0] = s;
    }
    __syncthreads();
    tot[0] = sm[0][0]; tot[1] = sm[1][0]; tot[2] = sm[2][0];
  } else {
    // the three partial arrays in ONE loop: their loads are independent, so the three latencies overlap (same per-thread
    // order of additions as three separate loops: the sums are bit-identical)
    const double* __restrict__ p1 = r1.partials;
    const double* __restrict__ p2 = r2.partials;
    const double* __restrict__ p3 = r3.partials;
    const int nbmax = nb1 > nb2 ? (nb1 > nb3 ? nb1 : nb3) : (nb2 > nb3 ? nb2 : nb3);
    double s1 = 0.0, s2 = 0.0, s3 = 0.0;
    for (int i = threadIdx.x; i < nbmax; i += kStepThreads) {
      const double v1 = i < nb1 ? p1[i] : 0.0, v2 = i < nb2 ? p2[i] : 0.0, v3 = i < nb3 ? p3[i] : 0.0;
      if (i < nb1) s1 += v1;
      if (i < nb2) s2 += v2;
      if (i < nb3) s3 += v3;
    }
    // (the partial arrays are always valid memory: their loads are issued before the state block is looked at, so the two
    //  round trips overlap; a pass that turns out not to be due returns below without having written anything)
    if (st->iter >= st->stop_iter) return;
    s1 = warp_sum(s1); s2 = warp_sum(s2); s3 = warp_sum(s3);
    if (lane == 0) { sm[0][wid] = s1; sm[1][wid] = s2; sm[2][wid] = s3; }
    __syncthreads();
    if (wid == 0) {
#pragma unroll
      for (int a = 0; a < 3; a++) {
        double s = lane < kStepThreads / 32 ? sm[a][lane] : 0.0;
        tot[a] = warp_sum(s);
      }
    }
  }
  if (threadIdx.x == 0) {
    st->dx2 = tot[0];
    st->dy2 = dy2_override ? *dy2_override : tot[1];
    step_rule(st, tot[2]);
  }
}

// PIPE: persistent grid (DevSell::pipelined), slices walked in a software pipeline; !PIPE: one CTA per 8 slices
template <class Epi, bool PIPE = false>
__global__ void __launch_bounds__(kThreads) spmv_sell_kernel(DevSell A, Epi epi_arg, ReduceScratch rs) {
  Epi epi = epi_arg;
  if (!epi.begin()) return;
  const double* __restrict__ xin = epi.input();
  // Epilogues with many sums (CheckRowEpilogue, the multi-GPU check's 8): in the one-slice-per-warp shape every thread
  // finishes at most ONE row, so its terms go straight to a shared-memory row instead of living in 2 x NACC registers next
  // to the gather pipeline; the block tree is the same.
  constexpr bool kSmemAcc = (Epi::NACC > 4) && !PIPE;
  __shared__ double sacc[kSmemAcc ? Epi::NACC : 1][kSmemAcc ? kThreads : 1];
  double acc[(Epi::NACC > 0 && !kSmemAcc) ? Epi::NACC : 1] = {0.0};
  if constexpr (kSmemAcc) {
#pragma unroll
    for (int a = 0; a < Epi::NACC; a++) sacc[a][threadIdx.x] = 0.0;
  }
  if (PIPE && (int)blockIdx.x < A.nblocks_body) {
    // A warp walks the slices  w, w + W, w + 2W, ...  (W = warps of the body CTAs).  With one CTA per 8 slices (the default
    // grid) that is exactly one slice per warp; with a persistent grid (DevSell::nblocks_body = a few CTAs per SM) the walk
    // is software-pipelined: the descriptor is fetched two slices ahead and the first (up to) 8 column ids one slice ahead, so that
    // a slice's gathers issue at once instead of after two dependent round trips (descriptor -> column ids -> gathers).
    // Per-row arithmetic and its order are the same in both shapes.
    const int lane = threadIdx.x & 31;
    const int wstride = A.nblocks_body * (kThreads / 32);
    int slice = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
    int4 d = make_int4(0, 0, -1, 0), dn = make_int4(0, 0, -1, 0);
    int cpre[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (slice < A.nslices) {
      d = A.slices[slice];
      if (slice + wstride < A.nslices) dn = A.slices[slice + wstride];
#pragma unroll
      for (int u = 0; u < 8; u++) if (u < d.y) cpre[u] = A.col[d.x + lane + 32 * u];
    }
    while (slice < A.nslices) {
      int4 dnn = make_int4(0, 0, -1, 0);
      if (slice + 2 * wstride < A.nslices) dnn = A.slices[slice + 2 * wstride];
      int cnx[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (slice + wstride < A.nslices) {
#pragma unroll
        for (int u = 0; u < 8; u++) if (u < dn.y) cnx[u] = A.col[dn.x + lane + 32 * u];
      }
      const int row = slice * 32 + lane;
      const bool live = !((unsigned)d.z >> lane & 1u);
      if (live) epi.prefetch(row);
      const int* __restrict__ cp = A.col + d.x + lane;
      const double* __restrict__ vp = A.val + d.x + lane;
      double s = 0.0;
      int k = 0;
      {
        // the first min(len, 8) entries of every row: their column ids arrived one slice ago (u < d.y is warp-uniform)
        double v[8], g[8];
#pragma unroll
        for (int u = 0; u < 8; u++) g[u] = u < d.y ? xin[cpre[u]] : 0.0;
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = u < d.y ? vp[32 * u] : 0.0;
#pragma unroll
        for (int u = 0; u < 8; u++) if (u < d.y) s += v[u] * g[u];
        k = d.y < 8 ? d.y : 8;
      }
      for (; k + 8 <= d.y; k += 8) {
        int c[8];
        double v[8], g[8];
#pragma unroll
        for (int u = 0; u < 8; u++) c[u] = cp[32 * (k + u)];
#pragma unroll
        for (int u = 0; u < 8; u++) g[u] = xin[c[u]];
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = vp[32 * (k + u)];
#pragma unroll
        for (int u = 0; u < 8; u++) s += v[u] * g[u];
      }
      for (; k + 4 <= d.y; k += 4) {
        const int c0 = cp[32 * k], c1 = cp[32 * k + 32], c2 = cp[32 * k + 64], c3 = cp[32 * k + 96];
        const double g0 = xin[c0], g1 = xin[c1], g2 = xin[c2], g3 = xin[c3];
        const double v0 = vp[32 * k], v1 = vp[32 * k + 32], v2 = vp[32 * k + 64], v3 = vp[32 * k + 96];
        s += v0 * g0;
        s += v1 * g1;
        s += v2 * g2;
        s += v3 * g3;
      }
      for (; k < d.y; k++) s += vp[32 * k] * xin[cp[32 * k]];
      if (live) {
        if constexpr (kSmemAcc) {
          epi.row(row, s, StridedOut{&sacc[0][threadIdx.x]});
        } else {
          double t[Epi::NACC > 0 ? Epi::NACC : 1];
          epi.row(row, s, t);
          if constexpr (Epi::NACC > 0) {
#pragma unroll
            for (int a = 0; a < Epi::NACC; a++) add_term(acc[a], t[a], rs, a, row);
          }
        }
      }
      slice_end(epi, slice, live);
      d = dn;
      dn = dnn;
#pragma unroll
      for (int u = 0; u < 8; u++) cpre[u] = cnx[u];
      slice += wstride;
    }
  } else if ((int)blockIdx.x < A.nblocks_body) {
    const int slice = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (slice < A.nslices) {
      const int4 d = A.slices[slice];
      const int row = slice * 32 + lane;
      const bool live = !((unsigned)d.z >> lane & 1u);
      if (live) epi.prefetch(row);
      const int* __restrict__ cp = A.col + d.x + lane;
      const double* __restrict__ vp = A.val + d.x + lane;
      double s = 0.0;
      int k = 0;
      for (; k + 8 <= d.y; k += 8) {
        int c[8];
        double v[8], g[8];
#pragma unroll
        for (int u = 0; u < 8; u++) c[u] = cp[32 * (k + u)];
#pragma unroll
        for (int u = 0; u < 8; u++) g[u] = xin[c[u]];
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = vp[32 * (k + u)];
#pragma unroll
        for (int u = 0; u < 8; u++) s += v[u] * g[u];
      }
      for (; k + 4 <= d.y; k += 4) {
        const int c0 = cp[32 * k], c1 = cp[32 * k + 32], c2 = cp[32 * k + 64], c3 = cp[32 * k + 96];
        const double g0 = xin[c0], g1 = xin[c1], g2 = xin[c2], g3 = xin[c3];
        const double v0 = vp[32 * k], v1 = vp[32 * k + 32], v2 = vp[32 * k + 64], v3 = vp[32 * k + 96];
        s += v0 * g0;
        s += v1 * g1;
        s += v2 * g2;
        s += v3 * g3;
      }
      for (; k < d.y; k++) s += vp[32 * k] * xin[cp[32 * k]];
      if (live) {
        if constexpr (kSmemAcc) {
          epi.row(row, s, StridedOut{&sacc[0][threadIdx.x]});
        } else {
          double t[Epi::NACC > 0 ? Epi::NACC : 1];
          epi.row(row, s, t);
          if constexpr (Epi::NACC > 0) {
#pragma unroll
            for (int a = 0; a < Epi::NACC; a++) add_term(acc[a], t[a], rs, a, row);
          }
        }
      }
      slice_end(epi, slice, live);
    }
  } else {
    // one segment of a long row.  Its slot of the partial sums is +0.0, stored before the ticket (the fence after the
    // long_partial store orders it); the finisher stores the row's terms, 0.0 + term, into the slot of the row's FIRST segment.
    // So where a term lands does not depend on which segment finishes last, and K4's sums are the same run to run.
    __shared__ double sm[kThreads / 32];
    const int4 sg = A.segs[blockIdx.x - A.nblocks_body];
    double s = 0.0;
    for (int e = sg.y + threadIdx.x; e < sg.z; e += kThreads) s += A.lval[e] * xin[A.lcol[e]];
    s = block_sum(s, sm);
    if (threadIdx.x == 0) {
      const int4 lr = A.long_rows[sg.w];
      const int seg = (int)(blockIdx.x - A.nblocks_body) - lr.y;
      if constexpr (Epi::NACC > 0) {
#pragma unroll
        for (int a = 0; a < Epi::NACC; a++) rs.partials[(size_t)a * gridDim.x + blockIdx.x] = 0.0;
      }
      A.long_partial[lr.w + seg] = s;
      __threadfence();
      const unsigned t = atomicAdd(&A.long_counter[sg.w], 1u);
      if (t == (unsigned)lr.z - 1u) {
        __threadfence();
        const volatile double* p = A.long_partial + lr.w;
        double tot = 0.0;
        for (int q = 0; q < lr.z; q++) tot += p[q];
        A.long_counter[sg.w] = 0u;
        epi.prefetch(lr.x);
        const size_t first = (size_t)A.nblocks_body + lr.y;
        if constexpr (kSmemAcc) {
          epi.row(lr.x, tot, StridedOut{&sacc[0][threadIdx.x]});
#pragma unroll
          for (int a = 0; a < Epi::NACC; a++) rs.partials[(size_t)a * gridDim.x + first] = 0.0 + sacc[a][threadIdx.x];
        } else {
          double t[Epi::NACC > 0 ? Epi::NACC : 1];
          epi.row(lr.x, tot, t);
          if constexpr (Epi::NACC > 0) {
#pragma unroll
            for (int a = 0; a < Epi::NACC; a++) {
              rs.partials[(size_t)a * gridDim.x + first] = 0.0 + t[a];
              if (rs.terms) rs.terms[(size_t)a * rs.len + lr.x] = t[a];   // ordered mode: K4 adds these, in row order
            }
          }
        }
      }
    }
    return;   // (no block tree: the slot is written above)
  }
  if constexpr (kSmemAcc) {
    // same tree as block_partials: lanes, then the block's warps in order
    constexpr int kWarps = kThreads / 32;
    __shared__ double smp2[Epi::NACC][kWarps];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < Epi::NACC; a++) {
      const double v = warp_sum(sacc[a][threadIdx.x]);
      if (lane == 0) smp2[a][wid] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
      for (int a = 0; a < Epi::NACC; a++) {
        double v = 0.0;
#pragma unroll
        for (int w = 0; w < kWarps; w++) v += smp2[a][w];
        rs.partials[(size_t)a * gridDim.x + blockIdx.x] = v;
      }
    }
  } else if constexpr (Epi::NACC > 0) {
    block_partials<Epi::NACC>(acc, rs);
  }
}

// ============================================================ tiled SpMV (structured matrices)
// DevSell::tiled.  Same sliced-ELL arrays, same per-row arithmetic in the same order as spmv_sell_kernel, same epilogues; what
// changes is where the gathers go: a CTA owns kTileSlices consecutive slices (one length-sort window of 8192 rows), stages the
// window of the input vector that its rows touch in shared memory -- ONE bulk copy by the TMA unit (cp.async.bulk + mbarrier),
// 16-byte aligned, <= 192 KB -- and gathers from there: a gather then costs a shared-memory access (~4 bank-conflict cycles per
// warp) instead of 32 L1TEX wavefronts.  Sized in DESIGN.md section 8: staging pays only when one CTA covers a whole sort window
// (65 k gathers per staged window), which is why this is a separate kernel shape and not a variant of the 256-row CTA.
// Padding entries of the layout carry column 0 and value 0: a padded lane's index may fall outside the window, it then
// multiplies its 0 by 0 instead of by x[0] (the sum is unchanged; the sign of an all-zero row's zero may differ).
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

// `bytes` (a multiple of 16, from a 16-byte aligned address) into shared memory by the TMA unit: bulk copies of <= 32 KB
// completed on one mbarrier, which every thread of the CTA waits for (SASS: UBLKCP / SYNCS).  Contains a __syncthreads.
__device__ __forceinline__ void bulk_stage(void* dst, const void* src, unsigned bytes, unsigned long long* mbar) {
  const unsigned bar = smem_u32(mbar);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(1) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");   // the init, visible to the async proxy that completes on it
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    for (unsigned off = 0; off < bytes; off += 32768u) {   // chunks of 32 KB (each a multiple of 16 bytes)
      const unsigned n = bytes - off < 32768u ? bytes - off : 32768u;
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                       smem_u32(dst) + off),
                   "l"(reinterpret_cast<const char*>(src) + off), "r"(n), "r"(bar)
                   : "memory");
    }
  }
  unsigned done = 0;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done)
                 : "r"(bar), "r"(0)
                 : "memory");
  } while (!done);
}

template <class Epi>
__global__ void __launch_bounds__(kTileThreads, 1) spmv_sell_tile_kernel(DevSell A, Epi epi_arg, ReduceScratch rs) {
  extern __shared__ __align__(16) double xs[];
  __shared__ __align__(8) unsigned long long mbar;
  __shared__ double smp[Epi::NACC > 0 ? Epi::NACC : 1][kTileThreads / 32];
  Epi epi = epi_arg;
  if (!epi.begin()) return;
  const double* __restrict__ xin = epi.input();
  double acc[Epi::NACC > 0 ? Epi::NACC : 1] = {0.0};
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int tile = blockIdx.x;
  if (tile >= A.nblocks_body) {
    // one segment of a long row (same scheme as spmv_sell_kernel, on this kernel's 1024 threads, the same slots: +0.0 in
    // every segment's, the finisher's 0.0 + term in the first segment's): gathers from global memory
    const int4 sg = A.segs[tile - A.nblocks_body];
    double s = 0.0;
    for (int e = sg.y + threadIdx.x; e < sg.z; e += kTileThreads) s += A.lval[e] * xin[A.lcol[e]];
    s = warp_sum(s);
    if (lane == 0) smp[0][wid] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      double tot_seg = 0.0;
      for (int q = 0; q < kTileThreads / 32; q++) tot_seg += smp[0][q];
      const int4 lr = A.long_rows[sg.w];
      const int seg = (tile - A.nblocks_body) - lr.y;
      if constexpr (Epi::NACC > 0) {
#pragma unroll
        for (int a = 0; a < Epi::NACC; a++) rs.partials[(size_t)a * gridDim.x + blockIdx.x] = 0.0;
      }
      A.long_partial[lr.w + seg] = tot_seg;
      __threadfence();
      const unsigned t = atomicAdd(&A.long_counter[sg.w], 1u);
      if (t == (unsigned)lr.z - 1u) {
        __threadfence();
        const volatile double* pp = A.long_partial + lr.w;
        double tot = 0.0;
        for (int q = 0; q < lr.z; q++) tot += pp[q];
        A.long_counter[sg.w] = 0u;
        epi.prefetch(lr.x);
        double t2[Epi::NACC > 0 ? Epi::NACC : 1];
        epi.row(lr.x, tot, t2);
        if constexpr (Epi::NACC > 0) {
#pragma unroll
          for (int a = 0; a < Epi::NACC; a++) rs.partials[(size_t)a * gridDim.x + A.nblocks_body + lr.y] = 0.0 + t2[a];
        }
      }
    }
    return;
  }
  const int lo = A.tile_lo[tile], w = A.tile_w[tile];
  const bool staged = w > 0;
  if (staged) {
    if (A.tiled == 1) {
      bulk_stage(xs, xin + lo, (unsigned)w * 8u, &mbar);
    } else {
      for (int i = threadIdx.x; i < w; i += kTileThreads) xs[i] = xin[lo + i];
      __syncthreads();
    }
  }
  const int s0 = tile * kTileSlices;
  const int s1 = s0 + kTileSlices < A.nslices ? s0 + kTileSlices : A.nslices;
  const unsigned uw = (unsigned)w;
  for (int slice = s0 + wid; slice < s1; slice += kTileThreads / 32) {
    const int4 d = A.slices[slice];
    const int row = slice * 32 + lane;
    const bool live = !((unsigned)d.z >> lane & 1u);
    if (live) epi.prefetch(row);
    const int* __restrict__ cp = A.col + d.x + lane;
    const double* __restrict__ vp = A.val + d.x + lane;
    double s = 0.0;
    int k = 0;
    if (staged) {
      for (; k + 8 <= d.y; k += 8) {
        int c[8];
        double v[8], g[8];
#pragma unroll
        for (int u = 0; u < 8; u++) c[u] = cp[32 * (k + u)];
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = vp[32 * (k + u)];
#pragma unroll
        for (int u = 0; u < 8; u++) { const unsigned q = (unsigned)(c[u] - lo); g[u] = q < uw ? xs[q] : 0.0; }
#pragma unroll
        for (int u = 0; u < 8; u++) s += v[u] * g[u];
      }
      for (; k < d.y; k++) {
        const unsigned q = (unsigned)(cp[32 * k] - lo);
        s += vp[32 * k] * (q < uw ? xs[q] : 0.0);
      }
    } else {
      for (; k + 8 <= d.y; k += 8) {
        int c[8];
        double v[8], g[8];
#pragma unroll
        for (int u = 0; u < 8; u++) c[u] = cp[32 * (k + u)];
#pragma unroll
        for (int u = 0; u < 8; u++) g[u] = xin[c[u]];
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = vp[32 * (k + u)];
#pragma unroll
        for (int u = 0; u < 8; u++) s += v[u] * g[u];
      }
      for (; k < d.y; k++) s += vp[32 * k] * xin[cp[32 * k]];
    }
    if (live) {
      double t[Epi::NACC > 0 ? Epi::NACC : 1];
      epi.row(row, s, t);
      if constexpr (Epi::NACC > 0) {
#pragma unroll
        for (int a = 0; a < Epi::NACC; a++) acc[a] += t[a];
      }
    }
    slice_end(epi, slice, live);
  }
  if constexpr (Epi::NACC > 0) {
    // lanes, then the CTA's 32 warps in order: a fixed tree
#pragma unroll
    for (int a = 0; a < Epi::NACC; a++) {
      const double v = warp_sum(acc[a]);
      if (lane == 0) smp[a][wid] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
      for (int a = 0; a < Epi::NACC; a++) {
        double v = 0.0;
        for (int q = 0; q < kTileThreads / 32; q++) v += smp[a][q];
        rs.partials[(size_t)a * gridDim.x + blockIdx.x] = v;
      }
    }
  }
}

template <class Epi>
static void launch_tile(cudaStream_t s, const DevSell& A, const Epi& e, const ReduceScratch& rs) {
  static bool attr_set[64] = {false};   // per instantiation AND per device: the attribute belongs to the function in one context
  const size_t smem = (size_t)kTileMaxWindow * sizeof(double);
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    cudaFuncSetAttribute(spmv_sell_tile_kernel<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  spmv_sell_tile_kernel<Epi><<<A.nblocks_body + A.nsegs, kTileThreads, smem, s>>>(A, e, rs);
}

// ============================================================ zero-skip SpMV (the PDHG pass, one GPU)
// DevSell::zskip_grid.  K2 gathers x', K3 gathers y', and a PDLP iterate is full of exact zeros (x' = max(x', l) with
// l = 0, y' = max(y', 0) on inequality rows).  A term v * (+-0.0) is +-0.0, and s + (+-0.0) == s for every s that is not
// -0.0; a row sum starts at +0.0 and +0 + -0 = +0, so it never is.  Skipping those terms therefore leaves every row sum
// bit-identical, and it saves their gathers, which bound these kernels on random columns (one 32-byte sector per
// gathered double).  The producers of x' / y' write the nonzero bitmap (DevSell::nzmap); every CTA stages it in shared
// memory with one bulk copy and tests a bit before it gathers.
// The block partial sums are those of the shape described by nblocks_body / pipelined: a CTA is kZGroups groups of
// kThreads, and group q of the grid does the work of that shape's CTAs q, q + Q, q + 2Q, ... (Q = groups in the grid) --
// warp w of the group walks the slices 8c + w, 8c + w + W, ... (W = 8 nblocks_body) of CTA c, in the same order, and the
// group writes CTA c's partials with the same tree.  Then the long-row segments, one per group, likewise.
template <class Epi>
__global__ void __launch_bounds__(kZThreads, 1) spmv_sell_zskip_kernel(DevSell A, Epi epi_arg, ReduceScratch rs) {
  extern __shared__ __align__(16) unsigned nzs[];
  __shared__ __align__(8) unsigned long long mbar;
  __shared__ double smp[kZGroups][Epi::NACC][kThreads / 32];
  __shared__ double sseg[kZGroups][kThreads / 32];
  Epi epi = epi_arg;
  if (!epi.begin()) return;
  const double* __restrict__ xin = epi.input();
  bulk_stage(nzs, A.nzmap, (unsigned)A.nz_bytes, &mbar);
  auto bit = [&](int c) { return (nzs[c >> 5] >> (c & 31)) & 1u; };
  const int lane = threadIdx.x & 31, grp = threadIdx.x / kThreads, w = (threadIdx.x % kThreads) >> 5;
  const int ngroups = gridDim.x * kZGroups, gid = grp * gridDim.x + blockIdx.x;
  const int nb = A.nblocks_body, ns = A.nslices, W = nb * (kThreads / 32);
  const int nslots = A.nblocks_body + A.nsegs;
  // this warp's walk: descriptor and the first (up to) 8 column ids one slice ahead
  int s = gid * 8 + w;
  int4 d = make_int4(0, 0, -1, 0);
  int cpre[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (gid < nb && s < ns) {
    d = A.slices[s];
#pragma unroll
    for (int u = 0; u < 8; u++) if (u < d.y) cpre[u] = A.col[d.x + lane + 32 * u];
  }
  for (int c = gid; c < nb; c += ngroups) {   // group-uniform
    double acc[Epi::NACC] = {};
    bool more = s < ns;
    while (more) {
      int sn = s + W;
      more = sn < ns;
      if (!more) sn = c + ngroups < nb ? (c + ngroups) * 8 + w : ns;
      int4 dn = make_int4(0, 0, -1, 0);
      int cnx[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (sn < ns) {
        dn = A.slices[sn];
#pragma unroll
        for (int u = 0; u < 8; u++) if (u < dn.y) cnx[u] = A.col[dn.x + lane + 32 * u];
      }
      const int row = s * 32 + lane;
      const bool live = !((unsigned)d.z >> lane & 1u);
      if (live) epi.prefetch(row);
      const int* __restrict__ cp = A.col + d.x + lane;
      const double* __restrict__ vp = A.val + d.x + lane;
      double sum = 0.0;
      int k = 0;
      {
        double v[8], g[8];
#pragma unroll
        for (int u = 0; u < 8; u++) g[u] = (u < d.y && bit(cpre[u])) ? xin[cpre[u]] : 0.0;
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = u < d.y ? vp[32 * u] : 0.0;
#pragma unroll
        for (int u = 0; u < 8; u++) if (u < d.y) sum += v[u] * g[u];
        k = d.y < 8 ? d.y : 8;
      }
      for (; k + 8 <= d.y; k += 8) {
        int cc[8];
        double v[8], g[8];
#pragma unroll
        for (int u = 0; u < 8; u++) cc[u] = cp[32 * (k + u)];
#pragma unroll
        for (int u = 0; u < 8; u++) g[u] = bit(cc[u]) ? xin[cc[u]] : 0.0;
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = vp[32 * (k + u)];
#pragma unroll
        for (int u = 0; u < 8; u++) sum += v[u] * g[u];
      }
      for (; k < d.y; k++) {
        const int cc = cp[32 * k];
        sum += vp[32 * k] * (bit(cc) ? xin[cc] : 0.0);
      }
      if (live) {
        double t[Epi::NACC];
        epi.row(row, sum, t);
#pragma unroll
        for (int a = 0; a < Epi::NACC; a++) acc[a] += t[a];
      }
      slice_end(epi, s, live);
      d = dn;
#pragma unroll
      for (int u = 0; u < 8; u++) cpre[u] = cnx[u];
      s = sn;
    }
    group_partials<Epi::NACC>(acc, rs, c, nslots, smp);
  }
  // long-row segments: as one kThreads CTA of spmv_sell_kernel does them (block_sum's tree, the ticket, the slots: +0.0 in
  // every segment's, the finisher's 0.0 + term in the first segment's, nb + lr.y)
  const int t = threadIdx.x % kThreads;
  for (int q = gid; q < A.nsegs; q += ngroups) {
    const int4 sg = A.segs[q];
    double sv = 0.0;
    for (int e = sg.y + t; e < sg.z; e += kThreads) sv += A.lval[e] * xin[A.lcol[e]];
    sv = warp_sum(sv);
    if (lane == 0) sseg[grp][w] = sv;
    asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(kThreads) : "memory");
    if (w == 0) {
      double r = lane < kThreads / 32 ? sseg[grp][lane] : 0.0;
      r = warp_sum(r);
      if (lane == 0) {
        const int4 lr = A.long_rows[sg.w];
#pragma unroll
        for (int a = 0; a < Epi::NACC; a++) rs.partials[(size_t)a * nslots + nb + q] = 0.0;
        A.long_partial[lr.w + q - lr.y] = r;
        __threadfence();
        const unsigned tk = atomicAdd(&A.long_counter[sg.w], 1u);
        if (tk == (unsigned)lr.z - 1u) {
          __threadfence();
          const volatile double* pp = A.long_partial + lr.w;
          double tot = 0.0;
          for (int i = 0; i < lr.z; i++) tot += pp[i];
          A.long_counter[sg.w] = 0u;
          epi.prefetch(lr.x);
          double tt[Epi::NACC];
          epi.row(lr.x, tot, tt);
#pragma unroll
          for (int a = 0; a < Epi::NACC; a++) rs.partials[(size_t)a * nslots + nb + lr.y] = 0.0 + tt[a];
        }
      }
    }
    asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(kThreads) : "memory");   // warp 0 is done with sseg[grp]
  }
}

template <class Epi>
static void launch_zskip(cudaStream_t s, const DevSell& A, const Epi& e, const ReduceScratch& rs) {
  static bool attr_set[64] = {false};   // per instantiation AND per device (see launch_tile)
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr_set[dev]) {
    int cap = 0;
    cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaFuncAttributes fa;
    cudaFuncGetAttributes(&fa, spmv_sell_zskip_kernel<Epi>);
    cudaFuncSetAttribute(spmv_sell_zskip_kernel<Epi>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap - (int)fa.sharedSizeBytes);
    if (dev >= 0 && dev < 64) attr_set[dev] = true;
  }
  spmv_sell_zskip_kernel<Epi><<<A.zskip_grid, kZThreads, A.nz_bytes, s>>>(A, e, rs);
}

// ============================================================ multi-GPU kernels
// World > 1 (DESIGN.md section 5): rank g owns a row block (A_g, A_g^T, y, ax, b) AND a column shard
// of every n-vector (x, aty, c, l, u, xSum ...).  Full-length vectors exist only as the gather input
// of K2 (`xfull`) and as the partial A_g^T y (`part`), both laid out in G segments of
// seg_len = shard_len + 2 whose tail slots carry scalars.  One pass =
//   M1 primal_shard_kernel   finalize aty on the shard if the last pass was accepted, then the
//                            trial x' = proj(x - tau(c - aty)) on the shard -> send buffer (+ |dx|^2)
//   all-gather               x' shards (+ scalar tails) -> xfull on every rank
//   K2 spmv<DualEpilogueMg>  local rows; |dy|^2 and the ROW-side interaction (AΔx)·Δy
//   M2 stash_scalars_kernel  block partials of K2 -> the tail slots of every segment of `part`
//   K3a spmv<PartialAty>     part = A_g^T y'
//   reduce-scatter           part -> red (my shard of A^T y' + summed scalars)
//   M3 step_rule_mg_kernel   step rule from the gathered / reduced scalars
__global__ void __launch_bounds__(kThreads)
primal_shard_kernel(int len, PdhgState* __restrict__ st, double* __restrict__ xs0, double* __restrict__ xs1,
                    double* __restrict__ aty_s, const double* __restrict__ red, const double* __restrict__ c,
                    const double* __restrict__ lo, const double* __restrict__ up, double* __restrict__ xsum,
                    double* __restrict__ send, ReduceScratch rs) {
  if (st->iter >= st->stop_iter) return;
  const int cur = st->cur;
  const double tau = st->tau_try, ntau = -tau;
  const bool pend = st->pending != 0, take = st->accepted_last != 0;
  const double w = st->w_pending;
  const double* __restrict__ x = cur ? xs1 : xs0;
  double* __restrict__ xn = cur ? xs0 : xs1;
  double acc[1] = {0.0};
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) {
    double ai;
    if (take) { ai = red[i]; aty_s[i] = ai; } else ai = aty_s[i];
    const double xc = x[i];
    if (pend) xsum[i] = xsum[i] + w * xc;
    double v = xc + ntau * c[i];
    v = v + tau * ai;
    const double u = up[i], l = lo[i];
    v = v < u ? v : u;
    v = v > l ? v : l;
    xn[i] = v;
    send[i] = v;
    const double d = xc - v;
    acc[0] += d * d;
  }
  block_partials<1>(acc, rs);
}

// ------------------------------------------------------------ fused P2P variant
// Same algorithm, but the two collectives are folded into our own kernels over NVLink peer memory
// (buffers of all ranks mapped with CUDA IPC):
//   * reduce-scatter  -> the primal shard kernel adds the G partial A_h^T y' it needs straight from
//                        the peers' `part` buffers (fixed rank order = deterministic), and
//   * all-gather      -> writes its trial x' shard straight into every peer's `xfull`;
//   * two flag barriers (one tiny CTA each) order the phases and carry the scalars; the second one
//     also evaluates the step rule.
__device__ __forceinline__ double ld_sys(const double* p) {
  double v;
  asm volatile("ld.volatile.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(kThreads)
primal_shard_p2p_kernel(int len, PdhgState* __restrict__ st, double* __restrict__ xs0, double* __restrict__ xs1,
                        double* __restrict__ aty_s, PeerPtrs pp, int world, int rank, int seg_len,
                        const double* __restrict__ c, const double* __restrict__ lo, const double* __restrict__ up,
                        double* __restrict__ xsum, ReduceScratch rs, double* __restrict__ atysum) {
  if (st->iter >= st->stop_iter) return;
  const int cur = st->cur;
  const double tau = st->tau_try, ntau = -tau;
  const bool pend = st->pending != 0, take = st->accepted_last != 0;
  const bool accum = pend && atysum != nullptr && st->light_on && st->iter < kDenseChecks;   // dense-check phase: carry A'ySum
  const double w = st->w_pending;
  const double* __restrict__ x = cur ? xs1 : xs0;
  double* __restrict__ xn = cur ? xs0 : xs1;
  const size_t seg = (size_t)rank * seg_len;   // even: 16-byte aligned (shard_len and seg_len are even)
  double acc[1] = {0.0};
  auto one = [&](double xc, double ci, double ai, double u, double l, double& out) {
    double v = xc + ntau * ci;
    v = v + tau * ai;
    v = v < u ? v : u;
    v = v > l ? v : l;
    out = v;
    const double d = xc - v;
    return d * d;
  };
  const int npair = len >> 1;                  // len = shard_len is even
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < npair; i += stride) {
    double2 ai;
    if (take) {
      // reduce-scatter: my segment of the G partial A_h^T y', read from the peers' `part` buffers over NVLink and added
      // in rank order.  All G loads are issued before the first add (with the loads inside the summing loop a thread
      // would pay G NVLink round trips one after the other).  The address is formed whole per element: written as
      // (part[h] + seg) + i, the compiler keeps the 16 segment bases in registers (148 instead of 116)
      double2 q[kMaxPeers];
#pragma unroll
      for (int h = 0; h < kMaxPeers; h++)
        if (h < world) q[h] = __ldcg(reinterpret_cast<const double2*>(pp.part[h] + seg + 2 * (size_t)i));
      ai = make_double2(0.0, 0.0);
#pragma unroll
      for (int h = 0; h < kMaxPeers; h++) {
        if (h < world) { ai.x += q[h].x; ai.y += q[h].y; }
      }
      reinterpret_cast<double2*>(aty_s)[i] = ai;
    } else {
      ai = reinterpret_cast<const double2*>(aty_s)[i];
    }
    const double2 xc = reinterpret_cast<const double2*>(x)[i];
    const double2 ci = reinterpret_cast<const double2*>(c)[i];
    const double2 u = reinterpret_cast<const double2*>(up)[i];
    const double2 l = reinterpret_cast<const double2*>(lo)[i];
    if (pend) {
      double2 sm = reinterpret_cast<double2*>(xsum)[i];
      sm.x = sm.x + w * xc.x;
      sm.y = sm.y + w * xc.y;
      reinterpret_cast<double2*>(xsum)[i] = sm;
    }
    if (accum) {
      double2 sa = reinterpret_cast<double2*>(atysum)[i];
      sa.x = sa.x + w * ai.x;
      sa.y = sa.y + w * ai.y;
      reinterpret_cast<double2*>(atysum)[i] = sa;
    }
    double2 o;
    acc[0] += one(xc.x, ci.x, ai.x, u.x, l.x, o.x);
    acc[0] += one(xc.y, ci.y, ai.y, u.y, l.y, o.y);
    reinterpret_cast<double2*>(xn)[i] = o;
    for (int h = 0; h < world; h++) reinterpret_cast<double2*>(pp.xfull[h] + seg)[i] = o;   // all-gather, fused
  }
  // no per-thread system fence: the kernel boundary completes the peer stores, and the barrier
  // kernel that follows fences at system scope before it signals
  block_partials<1>(acc, rs);
}

// check-iteration collectives of the fused path ------------------------------------------------------
// all-gather of a column shard: store it into every peer's xfull segment
__global__ void __launch_bounds__(kThreads)
push_shard_kernel(const double* __restrict__ src, int len, PeerPtrs pp, int world, int rank, int seg_len,
                  const PdhgState* due) {
  if (check_not_due(due)) return;
  const size_t seg = (size_t)rank * seg_len;
  const int npair = len >> 1;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < npair; i += stride) {
    const double2 v = reinterpret_cast<const double2*>(src)[i];
    for (int h = 0; h < world; h++) reinterpret_cast<double2*>(pp.xfull[h] + seg)[i] = v;
  }
}

// solution assembly without NCCL: `len` (<= seg_len) doubles into slot `rank` of every peer's receive buffer
__global__ void __launch_bounds__(kThreads)
push_rows_kernel(const double* __restrict__ src, int len, PeerPtrs pp, int world, int rank, int seg_len) {
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) {
    const double v = src[i];
    for (int h = 0; h < world; h++) pp.recv[h][(size_t)rank * seg_len + i] = v;
  }
}

// Bounded wait of the cross-GPU barriers: a peer that has not arrived after kBarrierTimeoutNs raises the fault word (the host
// turns it into an error) instead of hanging the device.  The bound is wall-clock time (%globaltimer), not a spin count: how long a
// count of ld.acquire.sys on an L2-resident flag lasts depends on the part, and ranks' hosts may reach a barrier seconds apart.
constexpr unsigned long long kBarrierTimeoutNs = 60ull * 1000000000ull;
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ bool barrier_expired(long long& spins, unsigned long long t0) {
  return (++spins & 0xfff) == 0 && global_ns() - t0 > kBarrierTimeoutNs;
}

// barrier + all-reduce of k <= 32 scalars (k = 0: pure barrier): every rank writes its values into every
// peer's mailbox (double-buffered by epoch parity), signals, waits, then adds all ranks' values in rank order
constexpr int kBigBox = 32;
__global__ void p2p_exchange_kernel(double* vals, int k, PeerPtrs pp, int world, int rank, unsigned long long* epochs,
                                    int* fault, const PdhgState* due, const SolveCtl* only_if_restart) {
  if (check_not_due(due)) return;   // identical on every rank
  if (only_if_restart && only_if_restart->restart_choice == 0) return;   // (the choice is identical on every rank too)
  if (*reinterpret_cast<volatile int*>(fault)) return;   // a barrier already timed out: do not wait another minute per launch
  const int lane = threadIdx.x;
  unsigned long long e = 0;
  if (lane == 0) { e = epochs[10] + 1; epochs[10] = e; }
  e = __shfl_sync(0xffffffffu, e, 0);
  const size_t box = 3 * kMaxPeers + 2 * kMaxPeers + (size_t)(e & 1) * kMaxPeers * kBigBox;
  if (lane < world)
    for (int j = 0; j < k; j++) reinterpret_cast<double*>(pp.flags[lane] + box)[rank * kBigBox + j] = vals[j];
  __threadfence_system();
  if (lane < world) {
    const unsigned long long* mine = pp.flags[rank] + 2 * kMaxPeers + lane;
    unsigned long long* theirs = pp.flags[lane] + 2 * kMaxPeers + rank;
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(theirs), "l"(e) : "memory");
    long long spins = 0;
    const unsigned long long t0 = global_ns();
    unsigned long long seen = 0;
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(mine) : "memory");
      if (seen < e && barrier_expired(spins, t0)) { *fault = 1; break; }
    } while (seen < e);
  }
  __syncwarp();
  if (*reinterpret_cast<volatile int*>(fault)) return;   // a peer never arrived: leave the (stale) mailboxes alone
  if (lane < k) {
    const double* mb = reinterpret_cast<const double*>(pp.flags[rank] + box);
    double s = 0.0;
    for (int g = 0; g < world; g++) s += ld_sys(mb + g * kBigBox + lane);
    vals[lane] = s;
  }
}

// only the fused reduce (check iterations: make the accepted A^T y' current without a primal step)
__global__ void __launch_bounds__(kThreads)
reduce_part_p2p_kernel(int len, double* __restrict__ dst, PeerPtrs pp, int world, int rank, int seg_len, int pull,
                       const PdhgState* due, int only_if_accepted) {
  if (check_not_due(due)) return;
  if (only_if_accepted && !due->accepted_last) return;
  const size_t seg = (size_t)rank * seg_len;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) {
    // pull 1: read the peers' `part`; 2: read the peers' `recv` (check iterations park their partial A_g^T ybar there so
    // that `part` keeps the last pass's data).  Loads first, then the sum in rank order: see primal_shard_p2p_kernel
    double q[kMaxPeers];
#pragma unroll
    for (int h = 0; h < kMaxPeers; h++)
      if (h < world) q[h] = __ldcg((pull == 1 ? pp.part[h] : pp.recv[h]) + seg + i);
    double ai = 0.0;
#pragma unroll
    for (int h = 0; h < kMaxPeers; h++)
      if (h < world) ai += q[h];
    dst[i] = ai;
  }
}

// cross-GPU barrier: lane h signals peer h and waits for peer h.  mode 0 (after the primal shard
// kernel): first publishes this rank's |dx|^2 into every peer's xfull tail.  mode 1 (after the partial
// A^T y): first publishes |dy|^2 and the row-side interaction into the local `part` tails, and after
// the barrier adds all ranks' scalars in rank order and applies the step rule.
__global__ void __launch_bounds__(kStepThreads)
p2p_barrier_kernel(int mode, PdhgState* st, const double* __restrict__ partials, int nb, PeerPtrs pp, int world,
                   int rank, int seg_len, int shard_len, unsigned long long* epochs, int* fault) {
  __shared__ double sm[2][kStepThreads / 32];
  __shared__ double tot[2];
  if (st->iter >= st->stop_iter) return;   // identical on every rank: nobody enters
  if (*reinterpret_cast<volatile int*>(fault)) return;   // a barrier already timed out (the host raises the error)
  // device-side timeline (epochs[2..]): [2] last exit stamp, [3+3*mode] sum(entry - previous exit) = the
  // compute phase before this barrier, [4+3*mode] sum(time inside the barrier), [5+3*mode] sum(wait), [9] count
  unsigned long long t_entry = 0, t_sig = 0, t_done = 0;
  if (threadIdx.x == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_entry));
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nv = mode == 0 ? 1 : 2;
  for (int a = 0; a < nv; a++) {
    double s = 0.0;
    for (int i = threadIdx.x; i < nb; i += kStepThreads) s += partials[(size_t)a * nb + i];
    s = warp_sum(s);
    if (lane == 0) sm[a][wid] = s;
  }
  __syncthreads();
  if (wid == 0) {
    for (int a = 0; a < nv; a++) {
      double s = lane < kStepThreads / 32 ? sm[a][lane] : 0.0;
      s = warp_sum(s);
      if (lane == 0) tot[a] = s;
    }
    __syncwarp();
    unsigned long long e = 0;
    if (lane == 0) { e = epochs[mode] + 1; epochs[mode] = e; }
    e = __shfl_sync(0xffffffffu, e, 0);
    // |dx|^2 lives in one of the segment's two tail slots, chosen by the parity of the pass: a rank that has left
    // barrier 1 may already publish the NEXT pass's |dx|^2 while a slower peer is still adding up this pass's
    const size_t tail = (size_t)rank * seg_len + shard_len;
    // PUSH model: scalars are written into every peer's local memory before the flag, so that after
    // the barrier nobody has to read across NVLink (every remote scalar read is a round trip)
    if (mode == 0) {
      if (lane < world) pp.xfull[lane][tail + (e & 1)] = tot[0];
    } else {
      if (lane < world) {
        double* mb = reinterpret_cast<double*>(pp.flags[lane] + 3 * kMaxPeers) + 2 * rank;   // peer's mailbox slot of this rank
        mb[0] = tot[0];
        mb[1] = tot[1];
      }
    }
    // no fence needed: lane h wrote its scalars to peer h and now releases the flag at peer h (st.release.sys
    // orders the lane's own earlier stores); data written by earlier KERNELS is complete at the kernel boundary
    if (lane < world) {
      const unsigned long long* mine = pp.flags[rank] + mode * kMaxPeers + lane;
      unsigned long long* theirs = pp.flags[lane] + mode * kMaxPeers + rank;
      asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(theirs), "l"(e) : "memory");
      if (lane == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_sig));
      long long spins = 0;
      const unsigned long long t0 = global_ns();
      unsigned long long seen = 0;
      do {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(mine) : "memory");
        if (seen < e && barrier_expired(spins, t0)) { *fault = 1; break; }   // never hang the device
      } while (seen < e);
    }
    __syncwarp();
    if (*reinterpret_cast<volatile int*>(fault)) return;   // timed out: no reduce, no step rule on stale scalars (the host raises the error)
    if (lane == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_done));
    if (mode == 1 && lane == 0) {
      const double* mb = reinterpret_cast<const double*>(pp.flags[rank] + 3 * kMaxPeers);
      double dx2 = 0.0, dy2 = 0.0, inter = 0.0;
      const size_t slot = (size_t)shard_len + (epochs[0] & 1);   // barrier 0 of THIS pass bumped epochs[0] last
      for (int g = 0; g < world; g++) {   // local memory, fixed rank order
        dx2 += ld_sys(pp.xfull[rank] + (size_t)g * seg_len + slot);
        dy2 += ld_sys(mb + 2 * g);
        inter += ld_sys(mb + 2 * g + 1);
      }
      st->dx2 = dx2;
      st->dy2 = dy2;
      const int it0 = st->iter;
      step_rule(st, inter);
      st->accepted_last = st->iter != it0;
    }
    if (lane == 0) {
      unsigned long long t_exit;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_exit));
      if (epochs[2]) epochs[3 + 3 * mode] += t_entry - epochs[2];
      epochs[4 + 3 * mode] += t_exit - t_entry;
      epochs[5 + 3 * mode] += t_done - t_sig;
      epochs[2] = t_exit;
      if (mode == 1) epochs[9] += 1;
    }
  }
}

// sums block partials (fixed order) and writes them to dst[k * stride + slot] for k < copies
template <int NV>
__global__ void __launch_bounds__(kStepThreads)
stash_scalars_kernel(PdhgState* st, const double* __restrict__ partials, int nb, double* dst, int copies, int stride) {
  __shared__ double sm[NV][kStepThreads / 32];
  if (st && st->iter >= st->stop_iter) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int a = 0; a < NV; a++) {
    double s = 0.0;
    for (int i = threadIdx.x; i < nb; i += kStepThreads) s += partials[(size_t)a * nb + i];
    s = warp_sum(s);
    if (lane == 0) sm[a][wid] = s;
  }
  __syncthreads();
  if (wid == 0) {
#pragma unroll
    for (int a = 0; a < NV; a++) {
      double s = lane < kStepThreads / 32 ? sm[a][lane] : 0.0;
      s = warp_sum(s);
      s = __shfl_sync(0xffffffffu, s, 0);
      for (int k = lane; k < copies; k += 32) dst[(size_t)k * stride + a] = s;
    }
  }
}

__global__ void step_rule_mg_kernel(PdhgState* st, const double* __restrict__ xfull, int world, int seg_len,
                                    int shard_len, const double* __restrict__ red) {
  if (threadIdx.x != 0 || st->iter >= st->stop_iter) return;
  double dx2 = 0.0;
  for (int g = 0; g < world; g++) dx2 += xfull[(size_t)g * seg_len + shard_len];   // fixed rank order
  st->dx2 = dx2;
  st->dy2 = red[shard_len];
  const int it0 = st->iter;
  step_rule(st, red[shard_len + 1]);
  st->accepted_last = st->iter != it0;
}

// ===================================================== check-iteration kernels
// PDHG_Compute_Average_Iterate (cupdlp_step.c:377-420): flush the pending
// weighted iterate into the sum, then avg = sum * (1/sumStep).
__global__ void __launch_bounds__(kThreads)
average_kernel(int len, const double* __restrict__ v, double* __restrict__ sum, double* __restrict__ avg,
               int pending, double w, double scale) {
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) {
    double s = sum[i];
    if (pending) { s = s + w * v[i]; sum[i] = s; }
    avg[i] = s * scale;
  }
}

// Device-parametrised variants for the SPECULATIVE check: enqueued right behind the pass graph, before the host
// knows the state; they read buffer parity / pending weight / step sum from the state block and do nothing unless
// the check iteration has been reached.
__global__ void __launch_bounds__(kThreads)
average_dev_kernel(int len, const double* __restrict__ v0, const double* __restrict__ v1, double* __restrict__ sum,
                   double* __restrict__ avg, const PdhgState* __restrict__ st) {
  if (check_not_due(st)) return;
  const double* __restrict__ v = st->cur ? v1 : v0;
  const bool pending = st->pending != 0;
  const double w = st->w_pending;
  const double scale = st->sum_step > 0.0 ? 1.0 / st->sum_step : 1.0;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) {
    double s = sum[i];
    if (pending) { s = s + w * v[i]; sum[i] = s; }
    avg[i] = s * scale;
  }
}
// after both averages (and the multi-GPU A^T y materialisation) consumed them
__global__ void check_clear_kernel(PdhgState* st) {
  if (check_not_due(st)) return;
  st->pending = 0;
  st->accepted_last = 0;
}

// column-side pass A for up to two iterates (current, average):
// PDHG_Compute_Primal_Feasibility's objective (cupdlp_solver.c:23-24),
// PDHG_Compute_Dual_Feasibility (:69-204) and the norms needed by
// PDHG_Compute_{Primal,Dual}_Infeasibility (:255-262, :367).
// out per iterate: 0 c.x, 1 sp.lo_f, 2 sn.up_f, 3 |dual residual|^2, 4 |sp|^2, 5 |sn|^2, 6 |x|^2
__global__ void __launch_bounds__(kThreads)
col_check_a_kernel(int n, int nit, ColIter it0, ColIter it1, const double* __restrict__ c,
                   const double* __restrict__ lo, const double* __restrict__ up,
                   const double* __restrict__ cs, ReduceScratch rs, double* __restrict__ out) {
  double acc[14];
#pragma unroll
  for (int a = 0; a < 14; a++) acc[a] = 0.0;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    const double ci = c[i], l = lo[i], u = up[i], sc = cs[i];
    const bool hl = l > -INFINITY, hu = u < INFINITY;
    const double lf = hl ? l : 0.0, uf = hu ? u : 0.0;
#pragma unroll
    for (int t = 0; t < 2; t++) {
      if (t >= nit) break;
      const ColIter& it = t ? it1 : it0;
      double* a = acc + 7 * t;
      col_check_a_terms(it.x[i], it.aty[i], ci, hl, hu, lf, uf, sc,
                        [&](int k, double v) { add_term(a[k], v, rs, 7 * t + k, i); });
    }
  }
  double res[14];
  if (grid_reduce<14>(acc, rs, res) && threadIdx.x == 0)
    for (int a = 0; a < 14; a++) out[a] = res[a];
}

// Tree-mode (large problems) single-sweep variants: the ray residuals are homogeneous in the ray scale,
//   |(aty/s + sp/s - sn/s) colScale| = |(aty + sp - sn) colScale| / s,   likewise for the primal ray,
// so they are accumulated UNSCALED in the same sweep and divided by the scale on the host: one sweep, one
// read-back (and one all-reduce on several GPUs) per check instead of two.  Not bit-identical to the
// reference's scale-then-square order, which is why ordered mode keeps the two-sweep kernels above/below.
// out per iterate (10): 0..6 as col_check_a, 7 |(aty+sp-sn) colScale|^2, 8 |min(x,0) hasLower / colScale|^2,
// 9 |max(x,0) hasUpper / colScale|^2
__global__ void __launch_bounds__(kThreads)
col_check_fused_kernel(int n, ColIter it0, ColIter it1, const double* __restrict__ c, const double* __restrict__ lo,
                       const double* __restrict__ up, const double* __restrict__ cs, ReduceScratch rs,
                       double* __restrict__ out, const PdhgState* __restrict__ st, ColIter alt0) {
  // st != nullptr (speculative launch): skip unless due; the current iterate is it0 if cur == 0, alt0 otherwise
  if (st) {
    if (check_not_due(st)) return;
    if (st->cur) it0 = alt0;
  }
  double acc[20];
#pragma unroll
  for (int a = 0; a < 20; a++) acc[a] = 0.0;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    const double ci = c[i], l = lo[i], u = up[i], sc = cs[i];
    const bool hl = l > -INFINITY, hu = u < INFINITY;
    const double lf = hl ? l : 0.0, uf = hu ? u : 0.0;
    const double isc = 1.0 / sc;
#pragma unroll
    for (int t = 0; t < 2; t++) {
      const ColIter& it = t ? it1 : it0;
      const double x = it.x[i], aty = it.aty[i];
      const double rc = ci - aty;
      const double sp = hl ? (rc > 0.0 ? rc : 0.0) : 0.0;
      const double sn = hu ? (rc < 0.0 ? -rc : 0.0) : 0.0;
      const double rr = (rc - sp + sn) * sc;
      const double k = (aty + sp - sn) * sc;
      const double bl = hl ? (x < 0.0 ? x : 0.0) * isc : 0.0;
      const double bu = hu ? (x > 0.0 ? x : 0.0) * isc : 0.0;
      double* a = acc + 10 * t;
      a[0] += x * ci; a[1] += sp * lf; a[2] += sn * uf; a[3] += rr * rr; a[4] += sp * sp; a[5] += sn * sn;
      a[6] += x * x; a[7] += k * k; a[8] += bl * bl; a[9] += bu * bu;
    }
  }
  double res[20];
  if (grid_reduce<20>(acc, rs, res) && threadIdx.x == 0)
    for (int a = 0; a < 20; a++) out[a] = res[a];
}

// out per iterate (4): 0 y.b, 1 |primal residual|^2, 2 |y|^2, 3 |[ax]_eq, min([ax]_ineq,0) rowScale|^2
__global__ void __launch_bounds__(kThreads)
row_check_fused_kernel(int m, RowIter it0, RowIter it1, const double* __restrict__ b, const double* __restrict__ rsca,
                       int neq, ReduceScratch rs, double* __restrict__ out, const PdhgState* __restrict__ st, RowIter alt0) {
  if (st) {
    if (check_not_due(st)) return;
    if (st->cur) it0 = alt0;
  }
  double acc[8];
#pragma unroll
  for (int a = 0; a < 8; a++) acc[a] = 0.0;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < m; i += stride) {
    const double bi = b[i], sc = rsca[i];
    const bool ineq = i >= neq;
#pragma unroll
    for (int t = 0; t < 2; t++) {
      const RowIter& it = t ? it1 : it0;
      const double y = it.y[i], ax = it.ax[i];
      double r = ax - bi;
      if (ineq) r = r < 0.0 ? r : 0.0;
      r = r * sc;
      double k = ax;
      if (ineq) k = k < 0.0 ? k : 0.0;
      k = k * sc;
      double* a = acc + 4 * t;
      a[0] += y * bi; a[1] += r * r; a[2] += y * y; a[3] += k * k;
    }
  }
  double res[8];
  if (grid_reduce<8>(acc, rs, res) && threadIdx.x == 0)
    for (int a = 0; a < 8; a++) out[a] = res[a];
}

// row-side pass A: out per iterate: 0 y.b, 1 |primal residual|^2, 2 |y|^2
// (cupdlp_solver.c:36-63 for the residual, :79 for y.b)
__global__ void __launch_bounds__(kThreads)
row_check_a_kernel(int m, int nit, RowIter it0, RowIter it1, const double* __restrict__ b,
                   const double* __restrict__ rsca, int neq, int row_offset, ReduceScratch rs,
                   double* __restrict__ out) {
  double acc[6];
#pragma unroll
  for (int a = 0; a < 6; a++) acc[a] = 0.0;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < m; i += stride) {
    const double bi = b[i], sc = rsca[i];
    const bool ineq = (i + row_offset) >= neq;
#pragma unroll
    for (int t = 0; t < 2; t++) {
      if (t >= nit) break;
      const RowIter& it = t ? it1 : it0;
      double* a = acc + 3 * t;
      row_check_a_terms(it.y[i], it.ax[i], bi, sc, ineq, [&](int k, double v) { add_term(a[k], v, rs, 3 * t + k, i); });
    }
  }
  double res[6];
  if (grid_reduce<6>(acc, rs, res) && threadIdx.x == 0)
    for (int a = 0; a < 6; a++) out[a] = res[a];
}

// column-side pass B (needs the ray scales of pass A): per iterate
// 0 |dual-ray constraint residual|^2 (cupdlp_solver.c:289-303),
// 1 |lower-bound violation of the primal ray|^2, 2 |upper ...|^2 (:395-423)
__global__ void __launch_bounds__(kThreads)
col_check_b_kernel(int n, int nit, ColIter it0, ColIter it1, double inv_dscale0, double inv_dscale1,
                   double inv_pscale0, double inv_pscale1, const double* __restrict__ c,
                   const double* __restrict__ lo, const double* __restrict__ up,
                   const double* __restrict__ cs, ReduceScratch rs, double* __restrict__ out) {
  double acc[6];
#pragma unroll
  for (int a = 0; a < 6; a++) acc[a] = 0.0;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    const double ci = c[i], l = lo[i], u = up[i], sc = cs[i];
    const double hl = l > -INFINITY ? 1.0 : 0.0, hu = u < INFINITY ? 1.0 : 0.0;
#pragma unroll
    for (int t = 0; t < 2; t++) {
      if (t >= nit) break;
      const ColIter& it = t ? it1 : it0;
      const double ids = t ? inv_dscale1 : inv_dscale0, ips = t ? inv_pscale1 : inv_pscale0;
      double* a = acc + 3 * t;
      col_check_b_terms(it.x[i], it.aty[i], ci, hl, hu, sc, ids, ips, [&](int k, double v) { add_term(a[k], v, rs, 3 * t + k, i); });
    }
  }
  double res[6];
  if (grid_reduce<6>(acc, rs, res) && threadIdx.x == 0)
    for (int a = 0; a < 6; a++) out[a] = res[a];
}

// row-side pass B: per iterate |[A ray]_eq, min([A ray]_ineq, 0)|^2 (cupdlp_solver.c:381-392)
__global__ void __launch_bounds__(kThreads)
row_check_b_kernel(int m, int nit, RowIter it0, RowIter it1, double inv_pscale0, double inv_pscale1,
                   const double* __restrict__ rsca, int neq, int row_offset, ReduceScratch rs,
                   double* __restrict__ out) {
  double acc[2] = {0.0, 0.0};
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < m; i += stride) {
    const double sc = rsca[i];
    const bool ineq = (i + row_offset) >= neq;
#pragma unroll
    for (int t = 0; t < 2; t++) {
      if (t >= nit) break;
      const RowIter& it = t ? it1 : it0;
      add_term(acc[t], row_check_b_term(it.ax[i], t ? inv_pscale1 : inv_pscale0, sc, ineq), rs, t, i);
    }
  }
  double res[2];
  if (grid_reduce<2>(acc, rs, res) && threadIdx.x == 0) { out[0] = res[0]; out[1] = res[1]; }
}

// |a - b|^2 (PDHG_Compute_Step_Size_Ratio, cupdlp_step.c:161-164) and |a|^2
__global__ void __launch_bounds__(kThreads)
diff_norm2_kernel(int len, const double* __restrict__ a, const double* __restrict__ b, ReduceScratch rs,
                  double* __restrict__ out) {
  double acc[1] = {0.0};
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) {
    const double d = b ? (a[i] + -1.0 * b[i]) : a[i];
    add_term(acc[0], d * d, rs, 0, i);
  }
  double res[1];
  if (grid_reduce<1>(acc, rs, res) && threadIdx.x == 0) out[0] = res[0];
}

__global__ void __launch_bounds__(kThreads) scale_kernel(int len, double* __restrict__ v, double w) {
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) v[i] = v[i] * w;
}

__global__ void __launch_bounds__(kThreads) fill_kernel(int len, double* __restrict__ v, double w) {
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) v[i] = w;
}

// ================================================== device-side check iteration (tree mode, one GPU)
// The whole check -- averages, A xbar and A'ybar, residuals of both iterates, termination, infeasibility, restart --
// without a host round trip (cupdlp_solver.c:953-1106 on the host in the reference; host_check path of engine.cu for
// ordered mode / several GPUs).  Eight launches (the split check):
//   C1 check_avg_xy_kernel         xbar = (xSum + w x) / sum(w), ybar likewise   (cupdlp_step.c:377-420)
//   C2 spmv<PlainEpilogue> x 2     A xbar and A'ybar, side by side
//   C3 check_*_sweep_kernel x 2    column-side (20) and row-side (8) sums of BOTH iterates, side by side
//   C4 check_decide_kernel         adds the block partials, forms the residuals, decides (1 CTA)
//   C5 restart_sweep_kernel        only if C4 chose a restart: copies, clears the sums, |x - x_lr|^2, |y - y_lr|^2
//   C6 check_finish_kernel         restart scalars (beta, tau, sigma), trace row, next check iteration, power tables
// Every kernel is a no-op unless the check iteration has been reached and the solve is still running, so the host can
// enqueue checks speculatively between graphs of passes.
__device__ __forceinline__ bool check_live(const PdhgState* st, const SolveCtl* ctl) {
  return ctl->term < 0 && !st->done && st->iter >= st->stop_iter;
}

__global__ void __launch_bounds__(kThreads)
check_avg_x_kernel(int n, const double* __restrict__ x0, const double* __restrict__ x1, double* __restrict__ xsum,
                   double* __restrict__ xavg, const PdhgState* __restrict__ st, const SolveCtl* __restrict__ ctl) {
  if (!check_live(st, ctl)) return;
  const double* __restrict__ x = st->cur ? x1 : x0;
  const bool pending = st->pending != 0;
  const double w = st->w_pending;
  const double scale = st->sum_step > 0.0 ? 1.0 / st->sum_step : 1.0;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    double s = xsum[i];
    if (pending) { s = s + w * x[i]; xsum[i] = s; }
    xavg[i] = s * scale;
  }
}

// row-side sums of one iterate (row_check_fused_kernel's terms): 0 y.b, 1 |primal residual|^2, 2 |y|^2,
// 3 |[ax]_eq, min([ax]_ineq, 0) rowScale|^2
template <class T>
__device__ __forceinline__ void row_terms(double y, double ax, double bi, double sc, bool ineq, T t) {
  double r = ax - bi;
  if (ineq) r = r < 0.0 ? r : 0.0;
  r = r * sc;
  double k = ax;
  if (ineq) k = k < 0.0 ? k : 0.0;
  k = k * sc;
  t[0] = y * bi; t[1] = r * r; t[2] = y * y; t[3] = k * k;
}
// column-side sums of one iterate (col_check_fused_kernel's terms, 10 of them)
template <class T>
__device__ __forceinline__ void col_terms(double x, double aty, double ci, double l, double u, double sc, T t) {
  const bool hl = l > -INFINITY, hu = u < INFINITY;
  const double lf = hl ? l : 0.0, uf = hu ? u : 0.0;
  const double isc = 1.0 / sc;
  const double rc = ci - aty;
  const double sp = hl ? (rc > 0.0 ? rc : 0.0) : 0.0;
  const double sn = hu ? (rc < 0.0 ? -rc : 0.0) : 0.0;
  const double rr = (rc - sp + sn) * sc;
  const double k = (aty + sp - sn) * sc;
  const double bl = hl ? (x < 0.0 ? x : 0.0) * isc : 0.0;
  const double bu = hu ? (x > 0.0 ? x : 0.0) * isc : 0.0;
  t[0] = x * ci; t[1] = sp * lf; t[2] = sn * uf; t[3] = rr * rr; t[4] = sp * sp; t[5] = sn * sn;
  t[6] = x * x; t[7] = k * k; t[8] = bl * bl; t[9] = bu * bu;
}

// Row side of the multi-GPU check (launch_spmv_check_rows_mg): A_g xbar, with the row-side sums of BOTH iterates in the
// epilogue.  ybar is read: the partial A_g'ybar had to be launched before this kernel could run, so average_dev_kernel
// formed ybar already.
struct CheckRowEpilogue {
  static constexpr int NACC = 8;
  const PdhgState* st;
  const SolveCtl* ctl;
  const double* xavg;
  const double *y0, *y1, *ax0, *ax1;
  const double* yavg;
  double* axavg;
  const double *b, *rsc;
  int neq;
  const double *y, *ax;
  __device__ bool begin() {
    if (!check_live(st, ctl)) return false;
    const int cur = st->cur;
    y = cur ? y1 : y0; ax = cur ? ax1 : ax0;
    return true;
  }
  __device__ const double* input() const { return xavg; }
  double p_y, p_ax, p_ya, p_b, p_sc;
  __device__ void prefetch(int r) { p_y = y[r]; p_ax = ax[r]; p_ya = yavg[r]; p_b = b[r]; p_sc = rsc[r]; }
  template <class T>
  __device__ void row(int r, double s, T t) const {
    axavg[r] = s;
    const bool ineq = r >= neq;
    row_terms(p_y, p_ax, p_b, p_sc, ineq, t);
    row_terms(p_ya, s, p_b, p_sc, ineq, t + 4);
  }
};

// ---- the residual sweeps of a check as plain vector kernels (one GPU).  Two uses:
//  * SPLIT check (GIVEN = true; the default from iteration kDenseChecks on): C1 forms xbar AND ybar, two PLAIN SpMV give
//    A xbar and A'ybar at the speed of the pass kernels, and these sweeps add the 20 + 8 terms.
//  * LIGHT check (GIVEN = false; dense-check phase, PdhgState::light_on && iter < kDenseChecks): A xbar = (A xSum) / sum(w)
//    and A'ybar = (A'ySum) / sum(w) come from the sums the passes carried: no SpMV at all.
// Same per-element terms (col_terms / row_terms) and the same downstream kernels (C4-C6) in both.
template <bool GIVEN>
__global__ void __launch_bounds__(kThreads)
check_cols_sweep_kernel(int n, const double* __restrict__ x0, const double* __restrict__ x1, const double* __restrict__ aty0,
                        const double* __restrict__ aty1, double* __restrict__ xsum, double* __restrict__ atysum,
                        double* __restrict__ xavg, double* __restrict__ atyavg, const double* __restrict__ c,
                        const double* __restrict__ lo, const double* __restrict__ up, const double* __restrict__ cs,
                        const PdhgState* __restrict__ st, const SolveCtl* __restrict__ ctl, ReduceScratch rs) {
  if (!check_live(st, ctl)) return;
  const bool dense = st->light_on && st->iter < kDenseChecks;
  if (!GIVEN && !dense) return;
  const int cur = st->cur;
  const double* __restrict__ x = cur ? x1 : x0;
  const double* __restrict__ aty = cur ? aty1 : aty0;
  const bool pending = st->pending != 0;
  const double w = st->w_pending;
  const double scale = st->sum_step > 0.0 ? 1.0 / st->sum_step : 1.0;
  const bool flush2 = GIVEN && dense && pending && atysum != nullptr;   // keep A'ySum in step with xSum's flush (done by C1)
  double acc[20];
#pragma unroll
  for (int a = 0; a < 20; a++) acc[a] = 0.0;
  const int stride = gridDim.x * kThreads;
#pragma unroll 2
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    const double xc = x[i], ac = aty[i];
    double xa, aa;
    if (GIVEN) {
      xa = xavg[i];
      aa = atyavg[i];
      if (flush2) atysum[i] = atysum[i] + w * ac;
    } else {
      double xs = xsum[i], as = atysum[i];
      if (pending) { xs = xs + w * xc; xsum[i] = xs; as = as + w * ac; atysum[i] = as; }
      xa = xs * scale;
      aa = as * scale;
      xavg[i] = xa;
      atyavg[i] = aa;
    }
    const double ci = c[i], l = lo[i], u = up[i], sc = cs[i];
    double t[20];
    col_terms(xc, ac, ci, l, u, sc, t);
    col_terms(xa, aa, ci, l, u, sc, t + 10);
#pragma unroll
    for (int a = 0; a < 20; a++) acc[a] += t[a];
  }
  block_partials<20>(acc, rs);
}

template <bool GIVEN>
__global__ void __launch_bounds__(kThreads)
check_rows_sweep_kernel(int m, int neq, const double* __restrict__ y0, const double* __restrict__ y1,
                        const double* __restrict__ ax0, const double* __restrict__ ax1, double* __restrict__ ysum,
                        double* __restrict__ axsum, double* __restrict__ yavg, double* __restrict__ axavg,
                        const double* __restrict__ b, const double* __restrict__ rsc, const PdhgState* __restrict__ st,
                        const SolveCtl* __restrict__ ctl, ReduceScratch rs) {
  if (!check_live(st, ctl)) return;
  const bool dense = st->light_on && st->iter < kDenseChecks;
  if (!GIVEN && !dense) return;
  const int cur = st->cur;
  const double* __restrict__ y = cur ? y1 : y0;
  const double* __restrict__ ax = cur ? ax1 : ax0;
  const bool pending = st->pending != 0;
  const double w = st->w_pending;
  const double scale = st->sum_step > 0.0 ? 1.0 / st->sum_step : 1.0;
  const bool flush2 = GIVEN && dense && pending && axsum != nullptr;
  double acc[8];
#pragma unroll
  for (int a = 0; a < 8; a++) acc[a] = 0.0;
  const int stride = gridDim.x * kThreads;
#pragma unroll 2
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < m; i += stride) {
    const double yc = y[i], ac = ax[i];
    double ya, aa;
    if (GIVEN) {
      ya = yavg[i];
      aa = axavg[i];
      if (flush2) axsum[i] = axsum[i] + w * ac;
    } else {
      double ys = ysum[i], as = axsum[i];
      if (pending) { ys = ys + w * yc; ysum[i] = ys; as = as + w * ac; axsum[i] = as; }
      ya = ys * scale;
      aa = as * scale;
      yavg[i] = ya;
      axavg[i] = aa;
    }
    const double bi = b[i], sc = rsc[i];
    const bool ineq = i >= neq;
    double t[8];
    row_terms(yc, ac, bi, sc, ineq, t);
    row_terms(ya, aa, bi, sc, ineq, t + 4);
#pragma unroll
    for (int a = 0; a < 8; a++) acc[a] += t[a];
  }
  block_partials<8>(acc, rs);
}

// several GPUs: a FULL check inside the dense-check phase (the host predicted past it while rejected steps held the device
// back) flushes xSum / ySum but not the carried products -- the light variant is switched off for the rest of the solve
// (the host reads the flag with the state block and stops choosing it)
__global__ void check_light_off_kernel(PdhgState* st, const SolveCtl* ctl) {
  if (check_live(st, ctl) && st->light_on && st->iter < kDenseChecks) st->light_on = 0;
}
void launch_check_light_off(cudaStream_t s, PdhgState* st, const SolveCtl* ctl) { check_light_off_kernel<<<1, 1, 0, s>>>(st, ctl); }

// C1 of the split check: xbar and ybar in one launch (flushes the pending weight into xSum and ySum)
__global__ void __launch_bounds__(kThreads)
check_avg_xy_kernel(int n, int m, const double* __restrict__ x0, const double* __restrict__ x1, double* __restrict__ xsum,
                    double* __restrict__ xavg, const double* __restrict__ y0, const double* __restrict__ y1,
                    double* __restrict__ ysum, double* __restrict__ yavg, const PdhgState* __restrict__ st,
                    const SolveCtl* __restrict__ ctl) {
  if (!check_live(st, ctl)) return;
  const double* __restrict__ x = st->cur ? x1 : x0;
  const double* __restrict__ y = st->cur ? y1 : y0;
  const bool pending = st->pending != 0;
  const double w = st->w_pending;
  const double scale = st->sum_step > 0.0 ? 1.0 / st->sum_step : 1.0;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    double s = xsum[i];
    if (pending) { s = s + w * x[i]; xsum[i] = s; }
    xavg[i] = s * scale;
  }
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < m; i += stride) {
    double s = ysum[i];
    if (pending) { s = s + w * y[i]; ysum[i] = s; }
    yavg[i] = s * scale;
  }
}

// PDHG_Check_Restart_GPU (cupdlp_restart.c:3-99): 0 none, 1 to the average, 2 to the current iterate
__device__ double restart_score_dev(double beta, double pf, double df, double gap) {   // cupdlp_restart.c:113-124
  return sqrt(beta * pf * pf + df * df / beta + gap * gap);
}
__device__ int decide_restart_dev(const PdhgState* st, SolveCtl* c) {
  const DevResiduals &L = c->res[0], &A = c->res[1];
  if (st->iter == c->last_restart_iter) {
    c->pf_lr = L.pfeas; c->df_lr = L.dfeas; c->gap_lr = L.gap;
    c->pf_lc = L.pfeas; c->df_lc = L.dfeas; c->gap_lc = L.gap;
    return 0;
  }
  const double mu_cur = restart_score_dev(st->beta, L.pfeas, L.dfeas, L.gap);
  const double mu_avg = restart_score_dev(st->beta, A.pfeas, A.dfeas, A.gap);
  int choice = mu_cur < mu_avg ? 2 : 1;
  const double mu_cand = mu_cur < mu_avg ? mu_cur : mu_avg;
  if ((st->iter - c->last_restart_iter) >= 0.36 * st->iter) {
    // artificial restart
  } else {
    const double mu_lr = restart_score_dev(st->beta, c->pf_lr, c->df_lr, c->gap_lr);
    if (!(mu_cand < 0.2 * mu_lr)) {
      const double mu_lc = restart_score_dev(st->beta, c->pf_lc, c->df_lc, c->gap_lc);
      if (!(mu_cand < 0.8 * mu_lr && mu_cand > mu_lc)) choice = 0;
    }
  }
  const DevResiduals& C = mu_cur < mu_avg ? L : A;
  c->pf_lc = C.pfeas; c->df_lc = C.dfeas; c->gap_lc = C.gap;
  return choice;
}

__device__ void trace_row_dev(SolveCtl* c, const PdhgState* st, int restart) {
  if (!c->trace || c->trace_len >= c->trace_cap) return;
  double* t = c->trace + (size_t)c->trace_len * 16;
  const DevResiduals &L = restart == 1 ? c->res[1] : c->res[0], &A = c->res[1];
  t[0] = st->iter; t[1] = L.pobj; t[2] = L.dobj; t[3] = L.pfeas; t[4] = L.dfeas;
  t[5] = A.pobj; t[6] = A.dobj; t[7] = A.pfeas; t[8] = A.dfeas;
  t[9] = st->tau; t[10] = st->sigma; t[11] = st->beta; t[12] = restart; t[13] = st->step_iter;
  t[14] = st->sum_step; t[15] = 0;
  c->trace_len++;
}

constexpr int kFinishThreads = 128;
static_assert(kFinishThreads == kPowTab, "one thread per power-table entry");
// the scalar part of C6 (one thread): restart scalars when a restart was chosen, trace row, next check iteration
__device__ void finish_scalars(PdhgState* st, SolveCtl* ctl, int choice, const double* d2, int step_iter) {
  if (choice) {
    const DevResiduals& R = choice == 1 ? ctl->res[1] : ctl->res[0];
    ctl->pf_lr = R.pfeas; ctl->df_lr = R.dfeas; ctl->gap_lr = R.gap;
    const double mean = sqrt(st->tau * st->sigma);
    const double dxn = sqrt(d2[0]), dyn = sqrt(d2[1]);
    double beta = st->beta;
    if (fmin(dxn, dyn) > 1e-10) {
      const double upd = dyn / dxn;
      const double lg = 0.5 * log(upd) + 0.5 * log(sqrt(beta));
      beta = exp(lg) * exp(lg);
    }
    st->beta = beta;
    st->tau = mean / sqrt(beta);
    st->sigma = st->tau * beta;
    st->sum_step = 0.0;
    ctl->last_restart_iter = st->iter;
    ctl->restarts++;
    // arm the next pass (start of PDHG_Update_Iterate_Adaptive_Step_Size, cupdlp_step.c:230-242)
    st->eta = sqrt(st->tau * st->sigma);
    if (st->adaptive) { st->tau_try = st->eta / sqrt(beta); st->sigma_try = st->eta * sqrt(beta); }
    else { st->tau_try = st->tau; st->sigma_try = st->sigma; }
  }
  trace_row_dev(ctl, st, choice);
  ctl->restart_choice = 0;
  st->pending = 0;        // the average flush consumed the pending weight (or the sums were just cleared)
  st->accepted_last = 0;
  const int it = st->iter, lim = ctl->iter_limit, iv = ctl->interval;
  int next = it + 1;
  while (!(next < 10 || next % iv == 0 || next == lim - 1)) next++;
  st->stop_iter = next;
  st->pow_base = step_iter;
}
// (k+1)^-0.3, (k+1)^-0.6 for k = step_iter + 1 + t  (cupdlp_step.c:279-284); threads 0 .. kPowTab-1 of one CTA
__device__ __forceinline__ void finish_pow_tables(PdhgState* st, int step_iter) {
  if (threadIdx.x < kPowTab) {
    const double k = (double)(step_iter + 1 + (int)threadIdx.x);
    st->pow_red[threadIdx.x] = pow(k + 1.0, -0.3);
    st->pow_grow[threadIdx.x] = pow(k + 1.0, -0.6);
  }
}

// C4: sums (fixed order) -> residuals (PDHG_Compute_Residuals / _Infeas_Residuals, cupdlp_solver.c:473-529, :433-471)
// -> PDHG_Check_Termination[_Average] (:797-841), PDHG_Check_Infeasibility (:740-795), limits (:1057-1067), restart choice
constexpr int kCheckSums = 28;
__device__ void decide_from_sums(PdhgState* st, SolveCtl* ctl, const double* tot, bool timed_out);
// One CTA per sum (28 CTAs x 256 threads, fixed order inside each), the last CTA to finish (ticket) decides.
constexpr int kDecideThreads = 256;
__global__ void __launch_bounds__(kDecideThreads)
check_decide_kernel(PdhgState* __restrict__ st, SolveCtl* __restrict__ ctl, const double* __restrict__ prow, int nbr,
                    const double* __restrict__ pcol, int nbc, unsigned* __restrict__ ticket) {
  if (!check_live(st, ctl)) return;
  __shared__ double sm[kDecideThreads / 32];
  __shared__ bool last;
  const int a = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const double* p = a < 8 ? prow + (size_t)a * nbr : pcol + (size_t)(a - 8) * nbc;
  const int nb = a < 8 ? nbr : nbc;
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
  int i = threadIdx.x;
  for (; i + 3 * kDecideThreads < nb; i += 4 * kDecideThreads) {
    s0 += p[i]; s1 += p[i + kDecideThreads]; s2 += p[i + 2 * kDecideThreads]; s3 += p[i + 3 * kDecideThreads];
  }
  for (; i < nb; i += kDecideThreads) s0 += p[i];
  double s = warp_sum((s0 + s1) + (s2 + s3));
  if (lane == 0) sm[wid] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kDecideThreads / 32; w++) t += sm[w];
    ctl->sums[a] = t;
    __threadfence();
    const unsigned k = atomicAdd(ticket, 1u);
    last = k == (unsigned)gridDim.x - 1u;
  }
  __syncthreads();
  if (!last) return;
  __shared__ int inline_finish;
  const int step_iter = st->step_iter;
  if (threadIdx.x == 0) {
    __threadfence();
    *ticket = 0u;
    double tot[kCheckSums];
    const volatile double* vs = ctl->sums;
    for (int q = 0; q < kCheckSums; q++) tot[q] = vs[q];
    decide_from_sums(st, ctl, tot, ctl->time_flag && *ctl->time_flag);
    // no restart, not finished: C6's bookkeeping right here (C5 and C6 then see a check that is no longer due and return)
    inline_finish = (ctl->term < 0 && ctl->restart_choice == 0) ? 1 : 0;
    if (inline_finish) { const double d2[2] = {0.0, 0.0}; finish_scalars(st, ctl, 0, d2, step_iter); }
  }
  __syncthreads();
  if (inline_finish) finish_pow_tables(st, step_iter);
}

// several GPUs: the 28 sums were all-reduced over the ranks (identical on every rank, added in rank order) into
// outs[0..19] (column side, 10 per iterate), outs[20..27] (row side, 4 per iterate), outs[28] (# ranks past the time limit)
__global__ void __launch_bounds__(kFinishThreads)
check_decide_sums_kernel(PdhgState* __restrict__ st, SolveCtl* __restrict__ ctl, const double* __restrict__ outs) {
  if (!check_live(st, ctl)) return;
  __shared__ int inline_finish;
  const int step_iter = st->step_iter;
  if (threadIdx.x == 0) {
    double tot[kCheckSums];
    for (int a = 0; a < 8; a++) tot[a] = outs[20 + a];
    for (int a = 0; a < 20; a++) tot[8 + a] = outs[a];
    decide_from_sums(st, ctl, tot, outs[28] > 0.0);
    // no restart, not finished: C6's bookkeeping right here (the restart exchange and C6 then have nothing to do)
    inline_finish = (ctl->term < 0 && ctl->restart_choice == 0) ? 1 : 0;
    if (inline_finish) { const double d2[2] = {0.0, 0.0}; finish_scalars(st, ctl, 0, d2, step_iter); }
  }
  __syncthreads();
  if (inline_finish) finish_pow_tables(st, step_iter);
}

__device__ void decide_from_sums(PdhgState* st, SolveCtl* ctl, const double* tot, bool timed_out) {
  const double sense = ctl->sense, offset = ctl->offset;
  for (int t = 0; t < 2; t++) {
    const double* a = tot + 8 + 10 * t;
    const double* r = tot + 4 * t;
    DevResiduals& R = ctl->res[t];
    R.pobj = a[0] * sense + offset;
    R.pfeas = sqrt(r[1]);
    R.dobj = ((r[0] + a[1]) - a[2]) * sense + offset;
    R.dfeas = sqrt(a[3]);
    R.gap = R.pobj - R.dobj;
    R.relgap = fabs(R.pobj - R.dobj) / (1.0 + fabs(R.pobj) + fabs(R.dobj));
    double dscale = sqrt(r[2] + a[4] + a[5]);
    if (dscale < 1e-8) dscale = 1.0;
    double pscale = sqrt(a[6]);
    if (pscale < 1e-8) pscale = 1.0;
    R.pinf_obj = (R.dobj - offset) / sense / dscale;
    R.pinf_res = sqrt(a[7]) / dscale;
    R.dinf_obj = (R.pobj - offset) / sense / pscale;
    R.dinf_res = sqrt(r[3] + a[8] + a[9]) / pscale;
  }
  for (int a = 0; a < kCheckSums; a++) ctl->sums[a] = tot[a];
  ctl->checks++;
  ctl->restart_choice = 0;
  const DevResiduals &L = ctl->res[0], &A = ctl->res[1];
  int term = -1, term_iterate = 0;
  if (L.pfeas < ctl->tol_p && L.dfeas < ctl->tol_d && L.relgap < ctl->tol_gap) { term = 0; term_iterate = 0; }
  else if (A.pfeas < ctl->tol_p && A.dfeas < ctl->tol_d && A.relgap < ctl->tol_gap) { term = 0; term_iterate = 1; }
  else {
    const double ft = 1e-8;   // dFeasTol, cupdlp_utils.c:889
    bool inf = false;
    for (int t = 0; t < 2; t++) {
      const DevResiduals& R = ctl->res[t];
      if (R.pinf_obj > 0.0 && R.pinf_res < ft * R.pinf_obj) inf = true;
      if (R.dinf_obj < 0.0 && R.dinf_res < -ft * R.dinf_obj) inf = true;
    }
    if (inf) term = 3;                                              // INFEASIBLE_OR_UNBOUNDED
    else if (timed_out) term = 4;                                   // TIMELIMIT_OR_ITERLIMIT
    else if (st->iter >= ctl->iter_limit - 1) term = 4;
  }
  if (term >= 0) {
    trace_row_dev(ctl, st, 0);
    ctl->term_iterate = term_iterate;
    st->pending = 0;
    st->accepted_last = 0;
    st->done = 1;       // from here on every kernel of the solve is a no-op
    __threadfence();
    ctl->term = term;
    return;
  }
  if (ctl->restart_on) ctl->restart_choice = decide_restart_dev(st, ctl);
}

// C5: PDHG_Restart_Iterate_GPU (cupdlp_proj.c:88-148) -- the vector part.  acc 0: |x - x_lastRestart|^2, 1: |y - y_lr|^2
__global__ void __launch_bounds__(kThreads)
restart_sweep_kernel(int n, int m, double* __restrict__ x0, double* __restrict__ x1, double* __restrict__ aty0,
                     double* __restrict__ aty1, const double* __restrict__ xavg, const double* __restrict__ atyavg,
                     double* __restrict__ xsum, double* __restrict__ xlr, double* __restrict__ y0, double* __restrict__ y1,
                     double* __restrict__ ax0, double* __restrict__ ax1, const double* __restrict__ yavg,
                     const double* __restrict__ axavg, double* __restrict__ ysum, double* __restrict__ ylr,
                     const PdhgState* __restrict__ st, const SolveCtl* __restrict__ ctl, ReduceScratch rs,
                     double* __restrict__ atysum, double* __restrict__ axsum) {
  if (!check_live(st, ctl) || ctl->restart_choice == 0) return;
  const bool dense = st->light_on && st->iter < kDenseChecks;   // A xSum / A'ySum restart with the sums they mirror
  const bool to_avg = ctl->restart_choice == 1;
  const int cur = st->cur;
  double* __restrict__ x = cur ? x1 : x0;
  double* __restrict__ aty = cur ? aty1 : aty0;
  double* __restrict__ y = cur ? y1 : y0;
  double* __restrict__ ax = cur ? ax1 : ax0;
  double acc[2] = {0.0, 0.0};
  const int stride = gridDim.x * kThreads;
  // pairs with 128-bit accesses (all vectors are allocation-aligned), then the odd tail
  // every load of an element pair is issued before its first store (the compiler cannot hoist them itself: it does not
  // know that the vectors are distinct), two pairs per trip, so that a warp has four 128-bit loads in flight
  auto sweep = [&](int len, double* cur_v, double* cur_a, const double* avg_v, const double* avg_a, double* sum, double* lr,
                   double& acc_out, double* sum2) {
    const int npair = len >> 1;
    const bool z2 = dense && sum2 != nullptr;
    const double2 zero = make_double2(0.0, 0.0);
    auto one = [&](int i, double2 v, double2 a, double2 l) {
      if (to_avg) {
        reinterpret_cast<double2*>(cur_v)[i] = v;
        reinterpret_cast<double2*>(cur_a)[i] = a;
      }
      reinterpret_cast<double2*>(sum)[i] = zero;
      if (z2) reinterpret_cast<double2*>(sum2)[i] = zero;
      const double d0 = v.x + -1.0 * l.x, d1 = v.y + -1.0 * l.y;
      acc_out += d0 * d0;
      acc_out += d1 * d1;
      reinterpret_cast<double2*>(lr)[i] = v;
    };
    const double2* src_v = reinterpret_cast<const double2*>(to_avg ? avg_v : cur_v);
    const double2* src_a = reinterpret_cast<const double2*>(avg_a);
    const double2* src_l = reinterpret_cast<const double2*>(lr);
    int i = blockIdx.x * kThreads + threadIdx.x;
    for (; i + stride < npair; i += 2 * stride) {
      const double2 v0 = src_v[i], v1 = src_v[i + stride];
      const double2 l0 = src_l[i], l1 = src_l[i + stride];
      double2 a0 = zero, a1 = zero;
      if (to_avg) { a0 = src_a[i]; a1 = src_a[i + stride]; }
      one(i, v0, a0, l0);
      one(i + stride, v1, a1, l1);
    }
    if (i < npair) {
      const double2 v0 = src_v[i], l0 = src_l[i];
      const double2 a0 = to_avg ? src_a[i] : zero;
      one(i, v0, a0, l0);
    }
    if ((len & 1) && blockIdx.x == 0 && threadIdx.x == 0) {
      const int q = len - 1;
      double v = cur_v[q];
      if (to_avg) { v = avg_v[q]; cur_v[q] = v; cur_a[q] = avg_a[q]; }
      sum[q] = 0.0;
      if (z2) sum2[q] = 0.0;
      const double d = v + -1.0 * lr[q];
      acc_out += d * d;
      lr[q] = v;
    }
  };
  sweep(n, x, aty, xavg, atyavg, xsum, xlr, acc[0], atysum);
  sweep(m, y, ax, yavg, axavg, ysum, ylr, acc[1], axsum);
  block_partials<2>(acc, rs);
}

// C6: the scalar part of the restart (PDHG_Compute_Step_Size_Ratio, cupdlp_step.c:147-176), then the bookkeeping the
// host loop does after a check: trace row, next check iteration (cupdlp_solver.c:953-962), step-rule power tables
// several GPUs: block partials of the epilogue sums (acc-major, nb per accumulator) -> nacc scalars at out[], added in block
// order; `flag_slot` >= 0: out[flag_slot] = 1 if this rank's host has raised the time-limit word (summed by the exchange)
__global__ void __launch_bounds__(kStepThreads)
reduce_partials_kernel(const PdhgState* __restrict__ st, const SolveCtl* __restrict__ ctl, int nacc,
                       const double* __restrict__ partials, int nb, double* __restrict__ out, int flag_slot, int need_restart,
                       int nacc2, const double* __restrict__ partials2, int nb2, double* __restrict__ out2) {
  // one WARP per accumulator (nacc + nacc2 <= 32): lane-strided loads in a fixed order, shuffle tree, no block barrier
  if (!check_live(st, ctl)) return;
  if (need_restart && ctl->restart_choice == 0) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (wid < nacc) {
    const double* __restrict__ p = partials + (size_t)wid * nb;
    double s = 0.0;
    for (int i = lane; i < nb; i += 32) s += p[i];
    s = warp_sum(s);
    if (lane == 0) out[wid] = s;
  } else if (wid < nacc + nacc2) {
    const int a = wid - nacc;
    const double* __restrict__ p = partials2 + (size_t)a * nb2;
    double s = 0.0;
    for (int i = lane; i < nb2; i += 32) s += p[i];
    s = warp_sum(s);
    if (lane == 0) out2[a] = s;
  }
  if (threadIdx.x == 0 && flag_slot >= 0) (nacc2 > 0 ? out2 : out)[flag_slot] = (ctl->time_flag && *ctl->time_flag) ? 1.0 : 0.0;
}

// sums2 != nullptr (several GPUs): the two restart sums were reduced and all-reduced already
__global__ void __launch_bounds__(kFinishThreads)
check_finish_kernel(PdhgState* __restrict__ st, SolveCtl* __restrict__ ctl, const double* __restrict__ prst, int nbs,
                    const double* __restrict__ sums2) {
  if (!check_live(st, ctl)) return;
  __shared__ double sm[2][kFinishThreads / 32];
  const int choice = ctl->restart_choice;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (choice && !sums2) {
    for (int a = 0; a < 2; a++) {
      double s = 0.0;
      for (int i = threadIdx.x; i < nbs; i += kFinishThreads) s += prst[(size_t)a * nbs + i];
      s = warp_sum(s);
      if (lane == 0) sm[a][wid] = s;
    }
  }
  const int step_iter = st->step_iter;
  __syncthreads();
  if (threadIdx.x == 0) {
    double d2[2] = {0.0, 0.0};
    if (choice) {
      if (sums2) { d2[0] = sums2[0]; d2[1] = sums2[1]; }
      else for (int a = 0; a < 2; a++) { double s = 0.0; for (int w = 0; w < kFinishThreads / 32; w++) s += sm[a][w]; d2[a] = s; }
    }
    finish_scalars(st, ctl, choice, d2, step_iter);
  }
  finish_pow_tables(st, step_iter);
}

// ==================================================================== launchers
static inline int ew_grid(int len) {
  int g = (len + kThreads - 1) / kThreads;
  if (g < 1) g = 1;
  return g > kMaxEwBlocks ? kMaxEwBlocks : g;
}

void launch_primal_step(cudaStream_t s, int n, PdhgState* st, double* x0, double* x1, const double* aty0,
                        const double* aty1, const double* c, const double* lo, const double* up, double* xsum,
                        ReduceScratch rs, unsigned* xnz) {
  primal_step_kernel<<<ew_grid((n + 1) / 2), kThreads, 0, s>>>(n, st, x0, x1, aty0, aty1, c, lo, up, xsum, rs, xnz);
}

// the nonzero bitmap (DevSell::nzmap) of a vector that no pass kernel produced (kernel-level entry points)
__global__ void __launch_bounds__(kThreads) nz_bitmap_kernel(int len, const double* __restrict__ v, unsigned* __restrict__ out) {
  for (int i0 = blockIdx.x * kThreads + (threadIdx.x & ~31); i0 < len; i0 += gridDim.x * kThreads) {
    const int i = i0 + (threadIdx.x & 31);
    const unsigned bits = __ballot_sync(0xffffffffu, i >= len || v[i] != 0.0);
    if ((threadIdx.x & 31) == 0) out[i0 >> 5] = bits;
  }
}
void launch_nz_bitmap(cudaStream_t s, int len, const double* v, unsigned* out) {
  if (len > 0) nz_bitmap_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, v, out);
}

// CTAs of spmv_sell_zskip_kernel that fit on one SM with nz_bytes of bitmap staged (both pass epilogues); 0: none
int zskip_ctas_per_sm(int nz_bytes) {
  int best = 1 << 30;
  auto one = [&](auto kern) {
    int dev = 0, cap = 0, k = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&cap, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, kern) != cudaSuccess || (size_t)nz_bytes + fa.sharedSizeBytes > (size_t)cap) { best = 0; return; }
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, cap - (int)fa.sharedSizeBytes);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&k, kern, kZThreads, (size_t)nz_bytes) != cudaSuccess) k = 0;
    best = k < best ? k : best;
  };
  one(spmv_sell_zskip_kernel<DualEpilogue>);
  one(spmv_sell_zskip_kernel<PrimalEpilogue>);
  cudaGetLastError();
  return best;
}

void launch_spmv_plain(cudaStream_t s, const DevSell& A, const double* in, double* out, const PdhgState* due) {
  if (A.nblocks_body + A.nsegs == 0) return;
  PlainEpilogue e{in, out, due};
  if (A.tiled) { launch_tile(s, A, e, ReduceScratch{nullptr, nullptr, nullptr, 0}); return; }
  if (A.pipelined) spmv_sell_kernel<PlainEpilogue, true><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, ReduceScratch{nullptr, nullptr, nullptr, 0});
  else spmv_sell_kernel<PlainEpilogue, false><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, ReduceScratch{nullptr, nullptr, nullptr, 0});
}

void launch_spmv_dual(cudaStream_t s, const DevSell& A, PdhgState* st, const double* x0, const double* x1,
                      double* y0, double* y1, double* ax0, double* ax1, const double* b, double* ysum,
                      int neq, int row_offset, ReduceScratch rs, double* axsum, unsigned* ynz) {
  if (A.nblocks_body + A.nsegs == 0) return;   // no rows on this rank: nothing to launch, the partial count is 0
  DualEpilogue e{};
  e.st = st; e.x0 = x0; e.x1 = x1; e.y0 = y0; e.y1 = y1; e.ax0 = ax0; e.ax1 = ax1; e.b = b; e.ysum = ysum;
  e.neq = neq; e.row_offset = row_offset; e.axsum = axsum; e.ynz = ynz;
  if (A.zskip_grid) { launch_zskip(s, A, e, rs); return; }
  if (A.tiled) { launch_tile(s, A, e, rs); return; }   // (the engine tiles only in tree mode)
  if (A.pipelined) spmv_sell_kernel<DualEpilogue, true><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, rs);
  else spmv_sell_kernel<DualEpilogue, false><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, rs);
}

void launch_spmv_primal(cudaStream_t s, const DevSell& A, PdhgState* st, const double* y0, const double* y1,
                        const double* x0, const double* x1, double* aty0, double* aty1, ReduceScratch rs, double* atysum) {
  if (A.nblocks_body + A.nsegs == 0) return;   // no rows on this rank: nothing to launch, the partial count is 0
  PrimalEpilogue e{};
  e.st = st; e.y0 = y0; e.y1 = y1; e.x0 = x0; e.x1 = x1; e.aty0 = aty0; e.aty1 = aty1; e.atysum = atysum;
  if (A.zskip_grid) { launch_zskip(s, A, e, rs); return; }
  if (A.tiled) { launch_tile(s, A, e, rs); return; }   // (tree mode only: engine.cu)
  if (A.pipelined) spmv_sell_kernel<PrimalEpilogue, true><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, rs);
  else spmv_sell_kernel<PrimalEpilogue, false><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, rs);
}

// multi-GPU K3a: partial A_g' y' into buf (input chosen by the device state)
struct PartialAtyEpilogue {
  static constexpr int NACC = 0;
  PdhgState* st;       // nullptr: check iterations, input = y0 (then `due` may predicate the launch)
  const double *y0, *y1;
  double* out;
  const int* __restrict__ outpos;
  const PdhgState* due;
  __device__ bool begin() {
    if (!st) return !check_not_due(due);
    if (st->iter >= st->stop_iter) return false;
    y0 = st->cur ? y0 : y1;
    return true;
  }
  __device__ const double* input() const { return y0; }
  __device__ void prefetch(int) {}
  // the partial vector is laid out in G segments of (shard_len + 2): the two tail slots of every
  // segment carry this rank's scalars so that a reduce-scatter delivers their sums to every rank.
  // The rows of A_g^T are sorted by their LOCAL length (little ELL padding on every rank), so the
  // result goes through an index array: outpos[r] = position of that column in the segmented vector.
  __device__ void row(int r, double s, double*) const { out[outpos[r]] = s; }
};

void launch_spmv_partial_aty(cudaStream_t s, const DevSell& A, PdhgState* st, const double* y0, const double* y1,
                             double* part, const int* outpos, const PdhgState* due) {
  if (A.nblocks_body + A.nsegs == 0) return;
  PartialAtyEpilogue e{st, y0, y1, part, outpos, due};
  spmv_sell_kernel<PartialAtyEpilogue><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, ReduceScratch{nullptr, nullptr, nullptr, 0});
}

void launch_spmv_dual_mg(cudaStream_t s, const DevSell& A, PdhgState* st, const double* xfull, double* y0, double* y1,
                         double* ax0, double* ax1, const double* b, double* ysum, int neq, ReduceScratch rs, double* axsum) {
  if (A.nblocks_body + A.nsegs == 0) return;   // no rows on this rank: nothing to launch, the partial count is 0
  DualEpilogueMg e{};
  e.st = st; e.x0 = xfull; e.x1 = xfull; e.y0 = y0; e.y1 = y1; e.ax0 = ax0; e.ax1 = ax1; e.b = b; e.ysum = ysum;
  e.neq = neq; e.row_offset = 0; e.axsum = axsum;
  spmv_sell_kernel<DualEpilogueMg><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, rs);
}

void launch_primal_shard(cudaStream_t s, int len, PdhgState* st, double* xs0, double* xs1, double* aty_s,
                         const double* red, const double* c, const double* lo, const double* up, double* xsum,
                         double* send, ReduceScratch rs) {
  primal_shard_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, st, xs0, xs1, aty_s, red, c, lo, up, xsum, send, rs);
}
int primal_shard_grid(int len) { return ew_grid(len); }
int primal_shard_p2p_grid(int len) { return ew_grid((len + 1) / 2); }

void launch_stash_scalars(cudaStream_t s, int nv, PdhgState* st, const double* partials, int nb, double* dst, int copies,
                          int stride) {
  if (nv == 1) stash_scalars_kernel<1><<<1, kStepThreads, 0, s>>>(st, partials, nb, dst, copies, stride);
  else stash_scalars_kernel<2><<<1, kStepThreads, 0, s>>>(st, partials, nb, dst, copies, stride);
}

void launch_primal_shard_p2p(cudaStream_t s, int len, PdhgState* st, double* xs0, double* xs1, double* aty_s,
                             const PeerPtrs& pp, int world, int rank, int seg_len, const double* c,
                             const double* lo, const double* up, double* xsum, ReduceScratch rs, double* atysum) {
  primal_shard_p2p_kernel<<<ew_grid((len + 1) / 2), kThreads, 0, s>>>(len, st, xs0, xs1, aty_s, pp, world, rank, seg_len,
                                                                      c, lo, up, xsum, rs, atysum);
}
void launch_push_shard(cudaStream_t s, const double* src, int len, const PeerPtrs& pp, int world, int rank, int seg_len,
                       const PdhgState* due) {
  push_shard_kernel<<<ew_grid((len + 1) / 2), kThreads, 0, s>>>(src, len, pp, world, rank, seg_len, due);
}
void launch_push_rows(cudaStream_t s, const double* src, int len, const PeerPtrs& pp, int world, int rank, int seg_len) {
  if (len <= 0) return;
  push_rows_kernel<<<ew_grid(len), kThreads, 0, s>>>(src, len, pp, world, rank, seg_len);
}
void launch_p2p_exchange(cudaStream_t s, double* vals, int k, const PeerPtrs& pp, int world, int rank,
                         unsigned long long* epochs, int* fault, const PdhgState* due, const SolveCtl* only_if_restart) {
  p2p_exchange_kernel<<<1, 32, 0, s>>>(vals, k, pp, world, rank, epochs, fault, due, only_if_restart);
}
void launch_reduce_part_p2p(cudaStream_t s, int len, double* dst, const PeerPtrs& pp, int world, int rank, int seg_len,
                            int pull, const PdhgState* due, int only_if_accepted) {
  reduce_part_p2p_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, dst, pp, world, rank, seg_len, pull, due, only_if_accepted);
}
void launch_p2p_barrier(cudaStream_t s, int mode, PdhgState* st, const double* partials, int nb, const PeerPtrs& pp,
                        int world, int rank, int seg_len, int shard_len, unsigned long long* epochs, int* fault) {
  p2p_barrier_kernel<<<1, kStepThreads, 0, s>>>(mode, st, partials, nb, pp, world, rank, seg_len, shard_len, epochs, fault);
}

void launch_step_rule_mg(cudaStream_t s, PdhgState* st, const double* xfull, int world, int seg_len, int shard_len,
                         const double* red) {
  step_rule_mg_kernel<<<1, 32, 0, s>>>(st, xfull, world, seg_len, shard_len, red);
}

void launch_step_rule(cudaStream_t s, PdhgState* st, ReduceScratch r1, int nb1, ReduceScratch r2, int nb2,
                      ReduceScratch r3, int nb3, const double* dy2_override) {
  step_rule_kernel<<<1, kStepThreads, 0, s>>>(st, r1, nb1, r2, nb2, r3, nb3, dy2_override);
}

int primal_step_grid(int n) { return ew_grid((n + 1) / 2); }

// CUDA loads kernels lazily (CUDA_MODULE_LOADING=LAZY, the default since 12.2), and loading may need a context-wide
// synchronisation.  With several ranks on ONE device (logical shards) a rank's barrier kernel spins until its peers'
// kernels signal -- if a peer's next kernel still has to be loaded, that load waits for the spinning kernel: deadlock
// (observed on hardware: every direct launch of a not-yet-used kernel behind a peer's barrier timed out, while runs whose
// kernels had all been instantiated into graphs beforehand went through).  So the kernels of the multi-GPU path are
// loaded up front.
void preload_multi_gpu_kernels() {
  const void* fns[] = {
      (const void*)primal_step_kernel, (const void*)primal_shard_kernel, (const void*)primal_shard_p2p_kernel,
      (const void*)push_shard_kernel, (const void*)push_rows_kernel,
      (const void*)p2p_exchange_kernel, (const void*)reduce_part_p2p_kernel, (const void*)p2p_barrier_kernel,
      (const void*)stash_scalars_kernel<1>, (const void*)stash_scalars_kernel<2>, (const void*)step_rule_mg_kernel,
      (const void*)step_rule_kernel, (const void*)average_kernel, (const void*)average_dev_kernel,
      (const void*)check_clear_kernel, (const void*)col_check_a_kernel, (const void*)col_check_b_kernel,
      (const void*)row_check_a_kernel, (const void*)row_check_b_kernel, (const void*)col_check_fused_kernel,
      (const void*)row_check_fused_kernel, (const void*)diff_norm2_kernel, (const void*)scale_kernel,
      (const void*)fill_kernel, (const void*)check_avg_x_kernel, (const void*)check_decide_kernel,
      (const void*)check_decide_sums_kernel, (const void*)restart_sweep_kernel, (const void*)reduce_partials_kernel,
      (const void*)check_finish_kernel, (const void*)check_light_off_kernel, (const void*)check_avg_xy_kernel,
      (const void*)check_cols_sweep_kernel<false>, (const void*)check_cols_sweep_kernel<true>,
      (const void*)check_rows_sweep_kernel<false>, (const void*)check_rows_sweep_kernel<true>,
      (const void*)spmv_sell_kernel<PlainEpilogue, false>, (const void*)spmv_sell_kernel<PlainEpilogue, true>,
      (const void*)spmv_sell_kernel<DualEpilogue, false>, (const void*)spmv_sell_kernel<DualEpilogue, true>,
      (const void*)spmv_sell_kernel<PrimalEpilogue, false>, (const void*)spmv_sell_kernel<PrimalEpilogue, true>,
      (const void*)spmv_sell_kernel<DualEpilogueMg, false>, (const void*)spmv_sell_kernel<PartialAtyEpilogue, false>,
      (const void*)spmv_sell_kernel<CheckRowEpilogue, false>,
  };
  cudaFuncAttributes at;
  for (const void* f : fns) cudaFuncGetAttributes(&at, f);
  cudaGetLastError();
}

// ---- device-side check iteration
void launch_check_avg_x(cudaStream_t s, int n, const double* x0, const double* x1, double* xsum, double* xavg,
                        const PdhgState* st, const SolveCtl* ctl) {
  if (n > 0) check_avg_x_kernel<<<ew_grid(n), kThreads, 0, s>>>(n, x0, x1, xsum, xavg, st, ctl);
}
void launch_check_decide(cudaStream_t s, PdhgState* st, SolveCtl* ctl, const double* prow, int nbr, const double* pcol,
                         int nbc, unsigned* ticket) {
  check_decide_kernel<<<kCheckSums, kDecideThreads, 0, s>>>(st, ctl, prow, nbr, pcol, nbc, ticket);
}
int restart_sweep_grid(int n, int m) { return ew_grid(n > m ? n : m); }
void launch_restart_sweep(cudaStream_t s, int n, int m, double* x0, double* x1, double* aty0, double* aty1,
                          const double* xavg, const double* atyavg, double* xsum, double* xlr, double* y0, double* y1,
                          double* ax0, double* ax1, const double* yavg, const double* axavg, double* ysum, double* ylr,
                          const PdhgState* st, const SolveCtl* ctl, ReduceScratch rs, double* atysum, double* axsum) {
  rs.terms = nullptr;
  restart_sweep_kernel<<<restart_sweep_grid(n, m), kThreads, 0, s>>>(n, m, x0, x1, aty0, aty1, xavg, atyavg, xsum, xlr, y0,
                                                                    y1, ax0, ax1, yavg, axavg, ysum, ylr, st, ctl, rs, atysum,
                                                                    axsum);
}
// few, long-lived CTAs: a block's tree over 20 (8) accumulators costs as much as its share of the sweep when the grid is the
// element-wise default of ~2400 CTAs, so the grid is capped at a few CTAs per SM
int check_light_grid(int len, bool cols) {
  const int g = ew_grid(len), cap = kGridUnit * (cols ? 2 : 4);
  return g < cap ? g : cap;
}
void launch_check_cols_sweep(cudaStream_t s, bool given, int n, const double* x0, const double* x1, const double* aty0,
                             const double* aty1, double* xsum, double* atysum, double* xavg, double* atyavg, const double* c,
                             const double* lo, const double* up, const double* cs, const PdhgState* st, const SolveCtl* ctl,
                             ReduceScratch rs) {
  rs.terms = nullptr;
  if (given) check_cols_sweep_kernel<true><<<check_light_grid(n, true), kThreads, 0, s>>>(n, x0, x1, aty0, aty1, xsum, atysum, xavg, atyavg, c, lo, up, cs, st, ctl, rs);
  else check_cols_sweep_kernel<false><<<check_light_grid(n, true), kThreads, 0, s>>>(n, x0, x1, aty0, aty1, xsum, atysum, xavg, atyavg, c, lo, up, cs, st, ctl, rs);
}
void launch_check_rows_sweep(cudaStream_t s, bool given, int m, int neq, const double* y0, const double* y1, const double* ax0,
                             const double* ax1, double* ysum, double* axsum, double* yavg, double* axavg, const double* b,
                             const double* rsc, const PdhgState* st, const SolveCtl* ctl, ReduceScratch rs) {
  rs.terms = nullptr;
  if (given) check_rows_sweep_kernel<true><<<check_light_grid(m, false), kThreads, 0, s>>>(m, neq, y0, y1, ax0, ax1, ysum, axsum, yavg, axavg, b, rsc, st, ctl, rs);
  else check_rows_sweep_kernel<false><<<check_light_grid(m, false), kThreads, 0, s>>>(m, neq, y0, y1, ax0, ax1, ysum, axsum, yavg, axavg, b, rsc, st, ctl, rs);
}
void launch_check_avg_xy(cudaStream_t s, int n, int m, const double* x0, const double* x1, double* xsum, double* xavg,
                         const double* y0, const double* y1, double* ysum, double* yavg, const PdhgState* st, const SolveCtl* ctl) {
  const int len = n > m ? n : m;
  if (len > 0) check_avg_xy_kernel<<<ew_grid(len), kThreads, 0, s>>>(n, m, x0, x1, xsum, xavg, y0, y1, ysum, yavg, st, ctl);
}
void launch_check_finish(cudaStream_t s, PdhgState* st, SolveCtl* ctl, const double* prst, int nbs, const double* sums2) {
  check_finish_kernel<<<1, kFinishThreads, 0, s>>>(st, ctl, prst, nbs, sums2);
}
// ---- several GPUs
void launch_spmv_check_rows_mg(cudaStream_t s, const DevSell& A, const PdhgState* st, const SolveCtl* ctl, const double* xfull,
                               const double* y0, const double* y1, const double* ax0, const double* ax1, const double* yavg,
                               double* axavg, const double* b, const double* rsc, int neq, ReduceScratch rs) {
  if (A.nblocks_body + A.nsegs == 0) return;
  CheckRowEpilogue e{};
  e.st = st; e.ctl = ctl; e.xavg = xfull; e.y0 = y0; e.y1 = y1; e.ax0 = ax0; e.ax1 = ax1;
  e.yavg = yavg; e.axavg = axavg; e.b = b; e.rsc = rsc; e.neq = neq;
  rs.terms = nullptr;
  spmv_sell_kernel<CheckRowEpilogue><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, rs);
}
void launch_reduce_partials(cudaStream_t s, const PdhgState* st, const SolveCtl* ctl, int nacc, const double* partials, int nb,
                            double* out, int flag_slot, int need_restart, int nacc2, const double* partials2, int nb2,
                            double* out2) {
  reduce_partials_kernel<<<1, kStepThreads, 0, s>>>(st, ctl, nacc, partials, nb, out, flag_slot, need_restart, nacc2, partials2, nb2, out2);
}
void launch_check_decide_sums(cudaStream_t s, PdhgState* st, SolveCtl* ctl, const double* outs) {
  check_decide_sums_kernel<<<1, kFinishThreads, 0, s>>>(st, ctl, outs);
}


void launch_average(cudaStream_t s, int len, const double* v, double* sum, double* avg, int pending, double w,
                    double scale) {
  if (len == 0) return;
  average_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, v, sum, avg, pending, w, scale);
}

void launch_col_check_a(cudaStream_t s, int n, int nit, ColIter a, ColIter b, const double* c, const double* lo,
                        const double* up, const double* cs, ReduceScratch rs, double* out) {
  col_check_a_kernel<<<ew_grid(n), kThreads, 0, s>>>(n, nit, a, b, c, lo, up, cs, rs, out);
}
void launch_col_check_fused(cudaStream_t s, int n, ColIter a, ColIter b, const double* c, const double* lo,
                            const double* up, const double* cs, ReduceScratch rs, double* out, const PdhgState* st,
                            ColIter alt) {
  col_check_fused_kernel<<<ew_grid(n), kThreads, 0, s>>>(n, a, b, c, lo, up, cs, rs, out, st, alt);
}
void launch_row_check_fused(cudaStream_t s, int m, RowIter a, RowIter b, const double* rhs, const double* rsca, int neq,
                            ReduceScratch rs, double* out, const PdhgState* st, RowIter alt) {
  row_check_fused_kernel<<<ew_grid(m), kThreads, 0, s>>>(m, a, b, rhs, rsca, neq, rs, out, st, alt);
}
void launch_average_dev(cudaStream_t s, int len, const double* v0, const double* v1, double* sum, double* avg,
                        const PdhgState* st) {
  if (len == 0) return;
  average_dev_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, v0, v1, sum, avg, st);
}
void launch_check_clear(cudaStream_t s, PdhgState* st) { check_clear_kernel<<<1, 1, 0, s>>>(st); }
void launch_row_check_a(cudaStream_t s, int m, int nit, RowIter a, RowIter b, const double* rhs,
                        const double* rsca, int neq, int row_offset, ReduceScratch rs, double* out) {
  row_check_a_kernel<<<ew_grid(m), kThreads, 0, s>>>(m, nit, a, b, rhs, rsca, neq, row_offset, rs, out);
}
void launch_col_check_b(cudaStream_t s, int n, int nit, ColIter a, ColIter b, const double inv_d[2],
                        const double inv_p[2], const double* c, const double* lo, const double* up,
                        const double* cs, ReduceScratch rs, double* out) {
  col_check_b_kernel<<<ew_grid(n), kThreads, 0, s>>>(n, nit, a, b, inv_d[0], inv_d[1], inv_p[0], inv_p[1], c, lo,
                                                     up, cs, rs, out);
}
void launch_row_check_b(cudaStream_t s, int m, int nit, RowIter a, RowIter b, const double inv_p[2],
                        const double* rsca, int neq, int row_offset, ReduceScratch rs, double* out) {
  row_check_b_kernel<<<ew_grid(m), kThreads, 0, s>>>(m, nit, a, b, inv_p[0], inv_p[1], rsca, neq, row_offset, rs,
                                                     out);
}
void launch_diff_norm2(cudaStream_t s, int len, const double* a, const double* b, ReduceScratch rs, double* out) {
  diff_norm2_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, a, b, rs, out);
}
void launch_scale(cudaStream_t s, int len, double* v, double w) {
  if (len == 0) return;
  scale_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, v, w);
}
void launch_fill(cudaStream_t s, int len, double* v, double w) {
  if (len == 0) return;
  fill_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, v, w);
}

}  // namespace b200

// =====================================================================================================================
// HiPDLP mode (solver=hipdlp): reflected Halpern PDHG, /root/reference/highs/pdlp/hipdlp/pdhg.cc:961-1018.
// One step = primal kernel (projection, reflection, Halpern blend of x) -> A * reflected x fused with the dual
// projection / reflection / blend of y -> A' y.  There is NO reduction and no step rule inside a step, so a block of
// steps is a plain chain of kernels (graph) and the trajectory does not depend on any summation order; the reductions
// live in the checks (fixed-point error, convergence test) every 40 steps.
// STATUS (round 2): bit-exact against the oracle on hardware (tests/test_gpu_hipdlp.py, ~160 solves).
namespace b200 {

__global__ void __launch_bounds__(kThreads)
hip_primal_kernel(int n, const HipState* __restrict__ st, int k_offset, int is_major, double* __restrict__ x,
                  const double* __restrict__ xa, const double* __restrict__ c, const double* __restrict__ aty,
                  const double* __restrict__ lo, const double* __restrict__ up, double* __restrict__ rx,
                  double* __restrict__ xn, double* __restrict__ hslack) {
  const double ps = st->primal_step;
  const int k = st->halpern_iteration + k_offset;
  const double w = (double)k / (k + 1.0);
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += stride)
    hip_primal_col(i, ps, w, is_major, x, xa, c, aty, lo, up, rx, xn, hslack);
}

// y-side (:992-1003, :1010-1013) as the epilogue of ax = A * reflected x
struct HipDualEpilogue {
  static constexpr int NACC = 0;
  const HipState* st;
  int k_offset, is_major;
  const double* in;            // reflected x
  double* y;                   // current dual iterate, blended in place
  const double *ya, *rlo, *rup;
  double *yn, *ry;             // written on major steps only (the checks read them)
  double ds, w;
  __device__ bool begin() {
    ds = st->dual_step;
    const int k = st->halpern_iteration + k_offset;
    w = (double)k / (k + 1.0);
    return true;
  }
  __device__ const double* input() const { return in; }
  double p_y, p_ya, p_lo, p_up;
  __device__ void prefetch(int r) { p_y = y[r]; p_ya = ya[r]; p_lo = rlo[r]; p_up = rup[r]; }
  // the blended y of row r, given s = (A * reflected x)[r]
  __device__ double blend(int r, double s) const { return hip_dual_blend(r, p_y, p_ya, p_lo, p_up, s, ds, w, is_major, yn, ry); }
  __device__ void row(int r, double s, double*) const { y[r] = blend(r, s); }
};

void launch_hip_primal(cudaStream_t s, int n, const HipState* st, int k_offset, int is_major, double* x, const double* xa,
                       const double* c, const double* aty, const double* lo, const double* up, double* rx, double* xn,
                       double* hslack) {
  hip_primal_kernel<<<ew_grid(n), kThreads, 0, s>>>(n, st, k_offset, is_major, x, xa, c, aty, lo, up, rx, xn, hslack);
}
void launch_hip_dual(cudaStream_t s, const DevSell& A, const HipState* st, int k_offset, int is_major, const double* rx,
                     double* y, const double* ya, const double* rlo, const double* rup, double* yn, double* ry) {
  if (A.nblocks_body + A.nsegs == 0) return;
  HipDualEpilogue e{};
  e.st = st; e.k_offset = k_offset; e.is_major = is_major; e.in = rx; e.y = y; e.ya = ya; e.rlo = rlo; e.rup = rup;
  e.yn = yn; e.ry = ry;
  // the launch shape the engine chose for A (apply_spmv_grid): a persistent grid must take the pipelined walk, which visits
  // every slice; the one-slice-per-warp kernel on that capped grid would skip slices
  const ReduceScratch none{nullptr, nullptr, nullptr, 0};
  if (A.tiled) { launch_tile(s, A, e, none); return; }
  if (A.pipelined) spmv_sell_kernel<HipDualEpilogue, true><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, none);
  else spmv_sell_kernel<HipDualEpilogue, false><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, none);
}

// ------------------------------------------------------------------------------------------------ checks
// out = a - b (the dual movement y_next - reflected_y that computeFixedPointError multiplies by A', :722-726)
__global__ void __launch_bounds__(kThreads) hip_diff_kernel(int len, const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ out) {
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) out[i] = a[i] - b[i];
}
void launch_hip_diff(cudaStream_t s, int len, const double* a, const double* b, double* out) {
  if (len > 0) hip_diff_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, a, b, out);
}

// dual slacks of the checked iterate (computeDualSlacks, :1322-1378): the cached major-step slack when there is one,
// otherwise the residual projected by the signs of the bounds
__global__ void __launch_bounds__(kThreads)
hip_slack_kernel(int n, int use_cached, const double* __restrict__ hslack, const double* __restrict__ c, const double* __restrict__ aty,
                 const double* __restrict__ lo, const double* __restrict__ up, double* __restrict__ sp, double* __restrict__ sn) {
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += stride) {
    double a, b;
    hip_dual_slacks(i, use_cached, hslack, c, aty, lo, up, a, b);
    sp[i] = a;
    sn[i] = b;
  }
}
void launch_hip_slack(cudaStream_t s, int n, int use_cached, const double* hslack, const double* c, const double* aty,
                      const double* lo, const double* up, double* sp, double* sn) {
  if (n > 0) hip_slack_kernel<<<ew_grid(n), kThreads, 0, s>>>(n, use_cached, hslack, c, aty, lo, up, sp, sn);
}

// The scalars of one check, each added in the REFERENCE'S ORDER by one warp (lanes load 32 terms at once, then every
// lane adds them in index order): bit-identical to the reference's sequential loops at any size, ~1 ns per term.
//   out[0] |x_next - refl_x|^2   out[1] |y_next - refl_y|^2   out[2] (x_next - refl_x).(A' dy)          (fixed-point error, :709-740)
//   out[3] |primal residual|^2 (:1297-1320)   out[4] |dual residual|^2 (:1380-1408)
//   out[5] offset + c.x (:1496-1500)          out[6] offset + b.y + l.sp - u.sn (:1447-1472)
//   out[7] |x_next - x_anchor|^2              out[8] |y_next - y_anchor|^2                                (PID weight, :1984-1999)
template <class Term>
__device__ __forceinline__ double warp_ordered_sum(int len, double init, Term term) {
  const int lane = threadIdx.x & 31;
  double sum = init;
  for (int base = 0; base < len; base += 32) {
    const int i = base + lane;
    const double t = i < len ? term(i) : 0.0;
    const int cnt = (len - base) < 32 ? (len - base) : 32;
    for (int k = 0; k < cnt; k++) sum = sum + __shfl_sync(0xffffffffu, t, k);
  }
  return sum;
}
__global__ void __launch_bounds__(9 * 32) hip_check_ordered_kernel(HipCheckArgs a, int with_fpe, double* __restrict__ out) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double v = 0.0;
  switch (w) {
    case 0: if (with_fpe) v = warp_ordered_sum(a.n, 0.0, [&](int i) { return hip_fpe_x_term(a, i); }); break;
    case 1: if (with_fpe) v = warp_ordered_sum(a.m, 0.0, [&](int i) { return hip_fpe_y_term(a, i); }); break;
    case 2: if (with_fpe) v = warp_ordered_sum(a.n, 0.0, [&](int i) { return hip_fpe_inter_term(a, i); }); break;
    case 3: v = warp_ordered_sum(a.m, 0.0, [&](int i) { return hip_primal_res_term(a, i); }); break;
    case 4: v = warp_ordered_sum(a.n, 0.0, [&](int i) { return hip_dual_res_term(a, i); }); break;
    case 5: v = warp_ordered_sum(a.n, a.offset, [&](int i) { return hip_pobj_term(a, i); }); break;
    case 6: {
      v = warp_ordered_sum(a.m, a.offset, [&](int i) { return hip_dobj_row_term(a, i); });
      v = warp_ordered_sum(a.n, v, [&](int i) { return hip_dobj_lo_term(a, i); });
      v = warp_ordered_sum(a.n, v, [&](int i) { return hip_dobj_up_term(a, i); });
      break;
    }
    case 7: v = warp_ordered_sum(a.n, 0.0, [&](int i) { return hip_anchor_x_term(a, i); }); break;
    case 8: v = warp_ordered_sum(a.m, 0.0, [&](int i) { return hip_anchor_y_term(a, i); }); break;
  }
  if (lane == 0) out[w] = v;
}
// the same scalars with grid-wide tree sums (large problems; deterministic, not the reference's order)
__global__ void __launch_bounds__(kThreads) hip_check_tree_kernel(HipCheckArgs a, int with_fpe, ReduceScratch rs, double* __restrict__ out) {
  double acc[9];
#pragma unroll
  for (int q = 0; q < 9; q++) acc[q] = 0.0;
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < a.n; i += stride) {
    if (with_fpe) { const double d = a.x[i] - a.rx[i]; acc[0] += d * d; acc[2] += d * a.atdy[i]; }
    double r = (a.c[i] - a.aty[i]) - a.sp[i] + a.sn[i];
    if (a.scaled) r = r * a.colscale[i];
    acc[4] += r * r;
    acc[5] += a.c[i] * a.x[i];
    if (a.lo[i] > -INFINITY) acc[6] += a.lo[i] * a.sp[i];
    if (a.up[i] < INFINITY) acc[6] -= a.up[i] * a.sn[i];
    const double d2 = a.x[i] - a.xa[i];
    acc[7] += d2 * d2;
  }
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < a.m; i += stride) {
    if (with_fpe) { const double d = a.y[i] - a.ry[i]; acc[1] += d * d; }
    double r = a.ax[i] - a.rlo[i];
    if (i >= a.neq) r = std_min(0.0, r);
    if (a.scaled) r = r * a.rowscale[i];
    acc[3] += r * r;
    acc[6] += a.rlo[i] * a.y[i];
    const double d2 = a.y[i] - a.ya[i];
    acc[8] += d2 * d2;
  }
  double res[9];
  if (grid_reduce<9>(acc, rs, res) && threadIdx.x == 0) {
    for (int q = 0; q < 9; q++) out[q] = res[q];
    out[5] += a.offset;
    out[6] += a.offset;
  }
}
void launch_hip_check(cudaStream_t s, const HipCheckArgs& a, int with_fpe, int ordered, ReduceScratch rs, double* out) {
  if (ordered) hip_check_ordered_kernel<<<1, 9 * 32, 0, s>>>(a, with_fpe, out);
  else {
    rs.terms = nullptr;
    const int len = a.n > a.m ? a.n : a.m;
    hip_check_tree_kernel<<<ew_grid(len), kThreads, 0, s>>>(a, with_fpe, rs, out);
  }
}

}  // namespace b200

// ---- HiPDLP power method on the device (pdhg.cc:1529-1671): dot products in index order (one warp) or as tree sums
namespace b200 {
__global__ void __launch_bounds__(32) hip_dot_ordered_kernel(int len, const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ out) {
  const double v = warp_ordered_sum(len, 0.0, [&](int i) { return a[i] * b[i]; });
  if (threadIdx.x == 0) out[0] = v;
}
__global__ void __launch_bounds__(kThreads) hip_dot_tree_kernel(int len, const double* __restrict__ a, const double* __restrict__ b, ReduceScratch rs, double* __restrict__ out) {
  double acc[1] = {0.0};
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) acc[0] += a[i] * b[i];
  double res[1];
  if (grid_reduce<1>(acc, rs, res) && threadIdx.x == 0) out[0] = res[0];
}
// v[i] /= sqrt(*norm_sq)   (z /= ||z||, :1646-1648)
__global__ void __launch_bounds__(kThreads) hip_div_norm_kernel(int len, double* __restrict__ v, const double* __restrict__ norm_sq) {
  const double nrm = sqrt(*norm_sq);
  const int stride = gridDim.x * kThreads;
  for (int i = blockIdx.x * kThreads + threadIdx.x; i < len; i += stride) v[i] = v[i] / nrm;
}
void launch_hip_dot(cudaStream_t s, int len, const double* a, const double* b, int ordered, ReduceScratch rs, double* out) {
  if (ordered) hip_dot_ordered_kernel<<<1, 32, 0, s>>>(len, a, b, out);
  else { rs.terms = nullptr; hip_dot_tree_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, a, b, rs, out); }
}
void launch_hip_div_norm(cudaStream_t s, int len, double* v, const double* norm_sq) {
  if (len > 0) hip_div_norm_kernel<<<ew_grid(len), kThreads, 0, s>>>(len, v, norm_sq);
}
}  // namespace b200

// ---- HiPDLP shards: the Halpern step on several GPUs (engine_hipdlp.cu, "HiPDLP on several GPUs").  Rank g owns device columns
// [c0, c1) and device rows [r0, r1); every vector is held full length in the one-GPU device order.  The step's two
// exchanged vectors are stored straight into the peers' copies: the reflected x by the primal kernel, the blended y by the
// dual epilogue.  The flag barrier carries no data: a Halpern step has no reduction, so nothing but arrival is exchanged.
namespace b200 {

__global__ void __launch_bounds__(kThreads)
hip_primal_shard_kernel(int c0, int c1, const HipState* __restrict__ st, int k_offset, int is_major, double* __restrict__ x,
                        const double* __restrict__ xa, const double* __restrict__ c, const double* __restrict__ aty,
                        const double* __restrict__ lo, const double* __restrict__ up, double* __restrict__ rx,
                        double* __restrict__ xn, double* __restrict__ hslack, PeerVec rx_peers, int world, int rank) {
  const double ps = st->primal_step;
  const int k = st->halpern_iteration + k_offset;
  const double w = (double)k / (k + 1.0);
  const int stride = gridDim.x * kThreads;
  for (int i = c0 + blockIdx.x * kThreads + threadIdx.x; i < c1; i += stride) {
    const double r = hip_primal_col(i, ps, w, is_major, x, xa, c, aty, lo, up, rx, xn, hslack);
#pragma unroll
    for (int h = 0; h < kMaxPeers; h++)   // (constant indices: the peer table stays in parameter space)
      if (h < world && h != rank) rx_peers.v[h][i] = r;
  }
}

// HipDualEpilogue over rank g's rows (the pointers are offset to the rank's first row) + the blended y into every peer
struct HipDualShardEpilogue : HipDualEpilogue {
  PeerVec y_peers;
  int world, rank;
  __device__ void row(int r, double s, double*) const {
    const double v = blend(r, s);
    y[r] = v;
#pragma unroll
    for (int h = 0; h < kMaxPeers; h++)
      if (h < world && h != rank) y_peers.v[h][r] = v;
  }
};

__global__ void __launch_bounds__(kThreads) hip_gather_kernel(HipGather g, int world, int rank) {
  const int stride = gridDim.x * kThreads;
  for (int q = 0; q < g.nv; q++)
    for (int i = g.lo + blockIdx.x * kThreads + threadIdx.x; i < g.hi; i += stride) {
      const double v = g.src[q][i];
#pragma unroll
      for (int h = 0; h < kMaxPeers; h++)
        if (h < world && h != rank) g.dst[q].v[h][i] = v;
    }
}

// Flag barrier: lane h stores the new epoch into peer h's arrival word for this rank (release, system scope: it publishes
// every store this rank made into peer h's memory before it, by this or an earlier kernel of the stream) and waits for
// peer h's word here (acquire).  Epochs only grow and no rank can pass barrier e + 1 before every rank has arrived at
// it, so a word is never more than one epoch ahead: "seen >= e" needs no double buffering.  The wait is bounded like
// p2p_barrier_kernel's: a peer that never arrives raises the fault word, and later barriers return at once.
__global__ void hip_barrier_kernel(PeerFlags pf, int world, int rank, unsigned long long* epoch, int* fault) {
  if (*reinterpret_cast<volatile int*>(fault)) return;
  const int lane = threadIdx.x;
  unsigned long long e = 0;
  if (lane == 0) { e = *epoch + 1; *epoch = e; }
  e = __shfl_sync(0xffffffffu, e, 0);
  __threadfence_system();
  if (lane < world) {
    unsigned long long* theirs = pf.f[lane] + rank;
    const unsigned long long* mine = pf.f[rank] + lane;
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(theirs), "l"(e) : "memory");
    long long spins = 0;
    const unsigned long long t0 = global_ns();
    unsigned long long seen = 0;
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(mine) : "memory");
      if (seen < e && barrier_expired(spins, t0)) { *fault = 1; break; }
    } while (seen < e);
  }
}

void launch_hip_primal_shard(cudaStream_t s, int c0, int c1, const HipState* st, int k_offset, int is_major, double* x,
                             const double* xa, const double* c, const double* aty, const double* lo, const double* up,
                             double* rx, double* xn, double* hslack, const PeerVec& rx_peers, int world, int rank) {
  if (c1 <= c0) return;
  hip_primal_shard_kernel<<<ew_grid(c1 - c0), kThreads, 0, s>>>(c0, c1, st, k_offset, is_major, x, xa, c, aty, lo, up, rx,
                                                                 xn, hslack, rx_peers, world, rank);
}
// one slice per warp only: the shape the sharded solve uses (the tiled and persistent shapes stay one-GPU)
void launch_hip_dual_shard(cudaStream_t s, const DevSell& A, const HipState* st, int k_offset, int is_major, const double* rx,
                           double* y, const double* ya, const double* rlo, const double* rup, double* yn, double* ry,
                           const PeerVec& y_peers, int world, int rank) {
  if (A.nblocks_body + A.nsegs == 0) return;
  HipDualShardEpilogue e{};
  e.st = st; e.k_offset = k_offset; e.is_major = is_major; e.in = rx; e.y = y; e.ya = ya; e.rlo = rlo; e.rup = rup;
  e.yn = yn; e.ry = ry; e.y_peers = y_peers; e.world = world; e.rank = rank;
  const ReduceScratch none{nullptr, nullptr, nullptr, 0};
  spmv_sell_kernel<HipDualShardEpilogue, false><<<A.nblocks_body + A.nsegs, kThreads, 0, s>>>(A, e, none);
}
void launch_hip_gather(cudaStream_t s, const HipGather& g, int world, int rank) {
  if (g.hi <= g.lo || g.nv == 0) return;
  hip_gather_kernel<<<ew_grid(g.hi - g.lo), kThreads, 0, s>>>(g, world, rank);
}
void launch_hip_barrier(cudaStream_t s, const PeerFlags& flags, int world, int rank, unsigned long long* epoch, int* fault) {
  hip_barrier_kernel<<<1, 32, 0, s>>>(flags, world, rank, epoch, fault);
}

// every kernel a sharded HiPDLP solve launches, loaded before the first barrier can spin (see preload_multi_gpu_kernels)
void preload_hipdlp_shard_kernels() {
  const void* fns[] = {
      (const void*)hip_primal_shard_kernel, (const void*)spmv_sell_kernel<HipDualShardEpilogue, false>,
      (const void*)hip_gather_kernel, (const void*)hip_barrier_kernel, (const void*)spmv_sell_kernel<PlainEpilogue, false>,
      (const void*)hip_diff_kernel, (const void*)hip_slack_kernel, (const void*)hip_check_ordered_kernel,
      (const void*)hip_check_tree_kernel, (const void*)hip_dot_ordered_kernel, (const void*)hip_dot_tree_kernel,
      (const void*)hip_div_norm_kernel, (const void*)fill_kernel,
  };
  cudaFuncAttributes at;
  for (const void* f : fns) cudaFuncGetAttributes(&at, f);
}
}  // namespace b200
