// highs_b200/csrc/kernels.cuh -- sm_90a (H100) kernels of the PDHG hot path.
//
// What the reference does with cuSPARSE SpMV + a chain of element-wise kernels +
// cuBLAS reductions that synchronise with the host every iteration
// (/root/reference/highs/pdlp/cupdlp/cuda/cupdlp_cudalinalg.cu:65-94,253-342,
//  cupdlp_cuda_kernels.cu:166-189,225-311) is four launches per PDHG pass here:
//
//   K1 primal_step_kernel   x' = proj(x - tau (c - A'y)), |x-x'|^2, xSum += w x
//   K2 spmv<DualEpilogue>   ax' = A x' fused with y' = proj(y + sigma(b - 2ax' + ax)),
//                           |y-y'|^2, ySum += w y
//   K3 spmv<PrimalEpilogue> aty' = A'y' fused with (x-x').(aty-aty')
//   K4 step_rule_kernel     one CTA adds the block partials of K1..K3 in a fixed order and
//                           evaluates the adaptive step rule ON THE DEVICE
//                           (cupdlp_step.c:266-285), flipping the double buffer on acceptance
//
// No host synchronisation inside a pass: every kernel reads the PdhgState block
// in device memory and is a no-op once state.iter reaches state.stop_iter, so the
// host can enqueue a whole check interval (CUDA graph) and read the state once.
//
// All arithmetic is fp64 and un-contracted (compile with -fmad=false): products
// and sums round separately, in the reference CPU path's operation order, so the
// element-wise results are bit-identical to HiGHS's CPU pdlp; only the ORDER of
// the long reductions (norms, dot products) differs (fixed tree instead of a
// sequential loop), and it is deterministic run to run.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// NVTX ranges (SURVEY.md section 5): phases of a solve show up by name in Nsight Systems / ncu --nvtx; header-only NVTX3,
// a no-op when no tool is attached.
#include <nvtx3/nvToolsExt.h>
namespace b200 {
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange&) = delete;
  NvtxRange& operator=(const NvtxRange&) = delete;
};
}  // namespace b200

namespace b200 {

constexpr int kThreads = 256;          // threads per block, every kernel
constexpr int kNnzBlk = 2048;          // == host_prep kNnzPerBlock
constexpr int kPowTab = 128;           // entries of the step-rule power tables
// Unit of the fixed grid caps (element-wise kernels, reductions of the prologue and of the checks).  The caps are constants,
// not multiples of the device's SM count, because the partial sums of a tree reduction are grouped by CTA: fixed caps keep
// every result bit-identical from one GPU model to the next.  On an H100 (132 SMs, 8 CTAs of 256 threads resident per SM)
// kMaxEwBlocks is 2.2 resident waves.
constexpr int kGridUnit = 148;
constexpr int kMaxEwBlocks = kGridUnit * 16; // grid cap of the element-wise kernels

// Device-resident control block of the PDHG loop (one per problem).
// cuPDLP checks EVERY one of the first 10 iterations (cupdlp_solver.c:953-962).  During that phase the passes keep
// axsum = A xSum and atysum = A'ySum up to date (the products of the accepted iterates are at hand in K2 / K3, weighted
// like xSum / ySum), so that those checks need no SpMV of the average iterate: two vector sweeps instead.
constexpr int kDenseChecks = 10;
struct PdhgState {
  // step sizes (cupdlp_defs.h CUPDLPstepsize): eta = dStepSizeUpdate carried into the next pass
  double eta, beta, tau, sigma;      // tau/sigma = dPrimalStep/dDualStep of the last accepted step
  double tau_try, sigma_try;         // eta/sqrt(beta), eta*sqrt(beta) for the pass about to run
  double sum_step;                   // dSumPrimalStep (== dSumDualStep)
  double w_pending;                  // weight of the iterate not yet added to xSum/ySum
  double dx2, dy2, inter;            // reductions of the running pass
  double mov, lim;                   // last movement / step limit (diagnostics)
  int iter;                          // accepted iterations = timers->nIter
  int step_iter;                     // nStepSizeIter (counts rejected passes too)
  int cur;                           // which half of the double buffers is current
  int pending;                       // 1: x[cur], y[cur] still to be added to the sums
  int stop_iter;                     // passes are no-ops once iter >= stop_iter
  int adaptive;                      // 1 adaptive line search, 0 fixed step
  int passes, rejects;
  int pow_base;                      // step_iter value that pow tables entry 0 belongs to
  int accepted_last;                 // multi-GPU: the previous pass was accepted (its A^T y' becomes current)
  int done;                          // device-driven loop: the solve has terminated -- every later kernel is a no-op
  int light_on;                      // 1: while iter < kDenseChecks the passes also carry A xSum and A'ySum (see "light check")
  double pow_red[kPowTab];           // (k+1)^-0.3 for k = pow_base+1+i   (host-computed, glibc pow)
  double pow_grow[kPowTab];          // (k+1)^-0.6
};

// Device-resident control of a whole solve (tree mode): the check iterations decide ON THE DEVICE -- termination,
// infeasibility, restarts, the next check iteration -- so that the host only enqueues work and reads this block
// (cupdlp_solver.c:939-1106 is the host loop this replaces; cupdlp_restart.c:3-99, cupdlp_proj.c:88-148).
struct DevResiduals {   // CUPDLPresobj of one iterate
  double pobj, dobj, pfeas, dfeas, gap, relgap, pinf_obj, pinf_res, dinf_obj, dinf_res;
};
struct SolveCtl {
  // constants of the solve
  double tol_p, tol_d, tol_gap;      // tol_p / tol_d already multiplied by (1 + |b|) / (1 + |c|)
  double sense, offset;
  int iter_limit, interval, restart_on, world;
  const volatile int* time_flag;     // mapped pinned host word: nonzero once the time limit has passed
  // restart memo (cupdlp_restart.c: dPrimalFeasLastRestart ..., dPrimalFeasLastCandidate ...)
  double pf_lr, df_lr, gap_lr, pf_lc, df_lc, gap_lc;
  int last_restart_iter;
  // per-check scratch
  int restart_choice;                // 0 none, 1 to the average, 2 to the current iterate (this check)
  // results
  int term;                          // -1 while running, else a b200pdlp_term
  int term_iterate, restarts, checks;
  DevResiduals res[2];               // residuals of the last check: current, average
  double* trace;                     // device [trace_cap][16] or nullptr
  int trace_cap, trace_len;
  double sums[32];                   // the reduced sums of the last check (diagnostics)
};

// HiPDLP mode: the few scalars a Halpern step reads on the device (so that a block of steps is graph-capturable)
struct HipState {
  double primal_step, dual_step;
  int halpern_iteration;   // steps since the last restart BEFORE the block that is running
  int pad;
};

// device view of a SellMatrix (host_prep.hpp)
struct DevSell {
  int nrows, nslices;
  int nblocks_body;                       // CTAs that process slices (8 slices = 256 rows each; fewer when `pipelined`)
  int nblocks_full;                       // one CTA per 8 slices, whatever nblocks_body says (sizes the partial-sum scratch)
  int nsegs;                              // + one CTA per long-row segment
  const int4* __restrict__ slices;        // {ptr, len, skipmask, -}
  const int* __restrict__ col;
  const double* __restrict__ val;
  const int4* __restrict__ segs;          // {row, nnz_begin, nnz_end, long_id}
  const int4* __restrict__ long_rows;     // {row, first_seg, nseg, partial_offset}
  const int* __restrict__ lcol;
  const double* __restrict__ lval;
  double* long_partial;
  unsigned* long_counter;
  int pipelined;                          // 1: nblocks_body is a persistent grid (a few CTAs per SM), slices walked in a software pipeline
  // TILED shape (structured matrices; spmv_sell_tile_kernel): one 1024-thread CTA per kTileSlices consecutive slices (= one
  // 8192-row sort window); the window of the input vector those rows touch, [tile_lo[t], tile_lo[t] + tile_w[t]), is staged in
  // shared memory by one bulk copy and the gathers read it there.  tile_w[t] == 0: window wider than the staging buffer, that
  // tile gathers from global memory.  tiled != 0: nblocks_body counts tiles.
  int tiled;                              // 0 off, 1 staged by cp.async.bulk (TMA unit) + mbarrier, 2 staged by cooperative loads
  const int* __restrict__ tile_lo;
  const int* __restrict__ tile_w;
  // ZERO-SKIP shape (the PDHG pass SpMVs only, one GPU, tree mode; spmv_sell_zskip_kernel): a nonzero bitmap of the input
  // vector, written by the kernel that produces that vector in the same pass (K1 for x', K2's epilogue for y').  Bit i is
  // word i >> 5, bit i & 31; 0 means "entry i is exactly +-0.0", 1 means "may be nonzero" (whoever cannot tell writes 1).
  // Every CTA stages the bitmap in shared memory and gathers only the entries whose bit is 1.  zskip_grid > 0: K2 / K3 of
  // this matrix run that kernel on zskip_grid CTAs; nblocks_body / pipelined keep describing the shape whose partial sums it
  // reproduces (and the one every other launch of this matrix uses).
  int zskip_grid;
  int nz_bytes;                           // staged bytes: the bitmap rounded up to 16 bytes
  unsigned* nzmap;
  int l2_hints;                           // 1: K1 and the zero-skip K2 / K3 load and store with L2 cache policies (L2Hints)
};
constexpr int kTileSlices = 256;          // slices per tile (8192 rows)
constexpr int kTileThreads = 1024;
constexpr int kTileMaxWindow = 24576;     // doubles staged per tile (192 KB of the 227 KB a CTA may use)
constexpr int kZThreads = 768;            // threads of a zero-skip CTA: kZGroups groups of kThreads, each one CTA of the walk
constexpr int kZGroups = kZThreads / kThreads;

// peer-memory view for the fused multi-GPU path (one process per GPU, buffers mapped with CUDA IPC)
constexpr int kMaxPeers = 16;
struct PeerPtrs {
  double* part[kMaxPeers];                 // every rank's partial A_g^T y buffer (G segments of seg_len)
  double* recv[kMaxPeers];                 // every rank's receive buffer: G slots (one per sender) of seg_len
  double* xfull[kMaxPeers];                // every rank's gathered trial x (G segments of seg_len)
  unsigned long long* flags[kMaxPeers];    // every rank's barrier flags [2][kMaxPeers]
};

// scratch of the two-stage deterministic reductions
struct ReduceScratch {
  double* partials;   // [nacc][gridDim.x]
  unsigned* counter;  // ticket of the last-block pattern (self-resetting)
  // ORDERED mode (small problems only): every element's term is also parked in
  // terms[acc][index]; the last block then adds them in index order, one thread per
  // accumulator -- the summation order of the reference's sequential CPU loops
  // (cupdlp_linalg.c:111-126,320-336), which makes whole trajectories bit-identical.
  double* terms;      // nullptr = tree mode
  int len;            // elements per accumulator in terms[]
};

// ----------------------------------------------------------------- reductions
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// sum over the block (fixed tree: lanes, then warps); result valid in thread 0
__device__ __forceinline__ double block_sum(double v, double* smem /*[kThreads/32]*/) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) smem[wid] = v;
  __syncthreads();
  double r = 0.0;
  if (wid == 0) {
    r = (lane < kThreads / 32) ? smem[lane] : 0.0;
    r = warp_sum(r);
  }
  return r;
}

// term bookkeeping used by every reducing kernel
__device__ __forceinline__ void add_term(double& acc, double term, const ReduceScratch& rs, int a, int i) {
  acc += term;
  if (rs.terms) rs.terms[(size_t)a * rs.len + i] = term;
}

// Stage 1 of the per-pass reductions: the block's partial sums go to partials[acc][block]; no fence,
// no ticket -- the (tiny) step_rule_kernel that follows in the stream adds them up in a fixed order.
// (A ticketed in-kernel final reduction would add a fence and an atomic to every one of the thousands of CTAs of a launch.)
template <int NACC>
__device__ __forceinline__ void block_partials(const double (&acc)[NACC], const ReduceScratch& rs) {
  constexpr int kWarps = kThreads / 32;
  __shared__ double smp[NACC][kWarps];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int a = 0; a < NACC; a++) {
    const double s = warp_sum(acc[a]);
    if (lane == 0) smp[a][wid] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int a = 0; a < NACC; a++) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < kWarps; w++) s += smp[a][w];
      rs.partials[(size_t)a * gridDim.x + blockIdx.x] = s;
    }
  }
}

// block_partials for one group of kThreads threads inside a wider CTA (threads [g kThreads, (g + 1) kThreads)): the same tree,
// synchronised by named barrier 1 + g, into slot `slot` of partials arrays `nslots` long.  smp: [groups][NACC][kThreads / 32].
template <int NACC>
__device__ __forceinline__ void group_partials(const double (&acc)[NACC], const ReduceScratch& rs, int slot, int nslots,
                                               double (*smp)[NACC][kThreads / 32]) {
  constexpr int kWarps = kThreads / 32;
  const int lane = threadIdx.x & 31, g = threadIdx.x / kThreads, wid = (threadIdx.x % kThreads) >> 5;
#pragma unroll
  for (int a = 0; a < NACC; a++) {
    const double s = warp_sum(acc[a]);
    if (lane == 0) smp[g][a][wid] = s;
  }
  asm volatile("bar.sync %0, %1;" ::"r"(1 + g), "r"(kThreads) : "memory");
  if (threadIdx.x % kThreads == 0) {
#pragma unroll
    for (int a = 0; a < NACC; a++) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < kWarps; w++) s += smp[g][a][w];
      rs.partials[(size_t)a * nslots + slot] = s;
    }
  }
  asm volatile("bar.sync %0, %1;" ::"r"(1 + g), "r"(kThreads) : "memory");   // smp is the group's again
}

// Two-stage deterministic sum over the grid.  Every warp parks its shuffle-reduced partials in
// shared memory; after ONE block barrier warps 1.. retire and warp 0 alone writes the block's
// partials, takes a ticket, and -- if it is the last block of the grid -- re-reduces all block
// partials in a fixed order.  Returns true in the last block only, with the sums in out[] (valid in
// thread 0).  Only threads of warp 0 return true/false meaningfully; other warps return false.
template <int NACC>
__device__ __forceinline__ bool grid_reduce(const double (&acc)[NACC], ReduceScratch rs, double (&out)[NACC]) {
  constexpr int kWarps = kThreads / 32;
  __shared__ double sm[NACC][kWarps];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nb = gridDim.x;
#pragma unroll
  for (int a = 0; a < NACC; a++) {
    const double s = warp_sum(acc[a]);
    if (lane == 0) sm[a][wid] = s;
  }
  if (rs.terms) __threadfence();   // ordered mode: every thread's terms[] must be visible to the last block
  __syncthreads();
  if (wid != 0) return false;
  if (lane == 0) {
#pragma unroll
    for (int a = 0; a < NACC; a++) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < kWarps; w++) s += sm[a][w];
      rs.partials[(size_t)a * nb + blockIdx.x] = s;
    }
    __threadfence();
  }
  unsigned ticket = 0;
  if (lane == 0) ticket = atomicAdd(rs.counter, 1u);
  ticket = __shfl_sync(0xffffffffu, ticket, 0);
  if (ticket != (unsigned)nb - 1u) return false;
  __threadfence();
  if (rs.terms) {
    // ordered mode: lane a adds accumulator a's terms in index order
    double s = 0.0;
    if (lane < NACC) {
      const volatile double* t = rs.terms + (size_t)lane * rs.len;
      for (int i = 0; i < rs.len; i++) s += t[i];
    }
#pragma unroll
    for (int a = 0; a < NACC; a++) out[a] = __shfl_sync(0xffffffffu, s, a);
  } else {
#pragma unroll
    for (int a = 0; a < NACC; a++) {
      // fixed order: lane l adds partials l, l+32, ... (four independent L2 loads in flight), then a warp tree
      const double* p = rs.partials + (size_t)a * nb;
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
      int i = lane;
      for (; i + 96 < nb; i += 128) {
        const double v0 = __ldcg(p + i), v1 = __ldcg(p + i + 32), v2 = __ldcg(p + i + 64), v3 = __ldcg(p + i + 96);
        s0 += v0; s1 += v1; s2 += v2; s3 += v3;
      }
      for (; i < nb; i += 32) s0 += __ldcg(p + i);
      out[a] = warp_sum((s0 + s1) + (s2 + s3));
    }
  }
  if (lane == 0) *rs.counter = 0u;
  return true;
}

}  // namespace b200
