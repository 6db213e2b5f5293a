// highs_b200/csrc/engine.cu -- host side of the B200 PDLP engine + the C ABI (include/b200pdlp.h).
//
// The host owns what cuPDLP-C's PDHG_Solve owns (/root/reference/highs/pdlp/cupdlp/
// cupdlp_solver.c:899-1106): the outer loop, the check schedule (first 10
// iterations, then every 40), termination, infeasibility detection and the
// restart decisions (cupdlp_restart.c:3-99, cupdlp_proj.c:88-148).  Everything that
// touches an n- or m-vector runs in pdhg_kernels.cu.  Between two checks the host
// does not synchronise: it points state.stop_iter at the next check iteration and
// replays a CUDA graph of PDHG passes; the adaptive step rule runs on the device.
#include <dlfcn.h>
#include <nccl.h>   // types only: the library is bound at run time (see NcclApi below)

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstddef>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <limits>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "batch_kernels.hpp"
#include "batch_prep.hpp"
#include "device_prep.hpp"
#include "host_prep.hpp"
#include "kkt_batch.hpp"
#include "pdhg_kernels.hpp"

namespace b200 {

static thread_local std::string g_last_error;

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define CUDA_OK(call)                                                                              \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess)                                                                         \
      throw Error(B200PDLP_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_) + " at " + \
                                         __FILE__ + ":" + std::to_string(__LINE__));               \
  } while (0)
#define NCCL_OK(call)                                                                                 \
  do {                                                                                                \
    ncclResult_t r_ = (call);                                                                         \
    if (r_ != ncclSuccess)                                                                            \
      throw Error(B200PDLP_ERR_NCCL, std::string(#call) + ": " + nccl().GetErrorString(r_) + " at " + \
                                         __FILE__ + ":" + std::to_string(__LINE__));                  \
  } while (0)

// NCCL is bound lazily with dlopen/dlsym: a single-GPU solve needs no NCCL at all, and in a
// process that already carries a libnccl.so.2 (PyTorch bundles its own, newer than the system one)
// we must use THAT copy instead of dragging a second one in at link time.
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*ReduceScatter)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
  static NcclApi& get() {
    static NcclApi api = load();
    return api;
  }
  static NcclApi load() {
    NcclApi a;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);          // already in the process?
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return a;
    a.GetUniqueId = (decltype(a.GetUniqueId))dlsym(h, "ncclGetUniqueId");
    a.CommInitRank = (decltype(a.CommInitRank))dlsym(h, "ncclCommInitRank");
    a.AllReduce = (decltype(a.AllReduce))dlsym(h, "ncclAllReduce");
    a.AllGather = (decltype(a.AllGather))dlsym(h, "ncclAllGather");
    a.ReduceScatter = (decltype(a.ReduceScatter))dlsym(h, "ncclReduceScatter");
    a.CommDestroy = (decltype(a.CommDestroy))dlsym(h, "ncclCommDestroy");
    a.GetErrorString = (decltype(a.GetErrorString))dlsym(h, "ncclGetErrorString");
    a.ok = a.GetUniqueId && a.CommInitRank && a.AllReduce && a.AllGather && a.ReduceScatter && a.CommDestroy && a.GetErrorString;
    return a;
  }
};
static NcclApi& nccl() {
  NcclApi& a = NcclApi::get();
  if (!a.ok) throw Error(B200PDLP_ERR_NCCL, "libnccl.so.2 not found: multi-GPU solves need NCCL");
  return a;
}

// Device buffer; the memory comes from (and returns to) the process-wide block cache of device_prep.cu, so the ~60
// allocations of a solve cost nothing after the first solve of a process (cudaMalloc / cudaFree are milliseconds each
// at these sizes, and cudaFree synchronises the device).
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) dev_cache_free(p); }
  void alloc(size_t count, bool zero = true) {
    if (p) { dev_cache_free(p); p = nullptr; }
    n = count;
    try { p = static_cast<T*>(dev_cache_alloc(std::max<size_t>(count, 1) * sizeof(T))); }
    catch (const std::exception& e) { throw Error(B200PDLP_ERR_ALLOC, e.what()); }
    if (zero) CUDA_OK(cudaMemset(p, 0, std::max<size_t>(count, 1) * sizeof(T)));
  }
  // take over a block that came from dev_cache_alloc
  void adopt(T* ptr, size_t count) {
    if (p) dev_cache_free(p);
    p = ptr; n = count;
  }
  void upload(const T* src, size_t count) {
    if (count) CUDA_OK(cudaMemcpy(p, src, count * sizeof(T), cudaMemcpyHostToDevice));
  }
  template <class A> void from(const std::vector<T, A>& v) { alloc(v.size(), false); upload(v.data(), v.size()); }
};

struct DeviceMatrix {
  SellMatrix host;
  DevBuf<int> col, lcol;
  DevBuf<double> val, lval, long_partial;
  DevBuf<int4> slices, segs, long_rows;
  DevBuf<unsigned> long_counter;
  DevBuf<int> tile_lo, tile_w;   // tiled shape (DevSell::tiled): windows of the input vector per tile of kTileSlices slices
  int ntiles = 0, tiles_staged = 0;
  DevSell dev{};
  void upload() {
    col.from(host.col);
    val.from(host.val);
    lcol.from(host.lcol);
    lval.from(host.lval);
    static_assert(sizeof(SellMatrix::Slice) == sizeof(int4) && sizeof(SellMatrix::Seg) == sizeof(int4) &&
                  sizeof(SellMatrix::LongRow) == sizeof(int4), "descriptor layouts");
    slices.alloc(host.slices.size(), false);
    slices.upload(reinterpret_cast<const int4*>(host.slices.data()), host.slices.size());
    segs.alloc(host.segs.size(), false);
    segs.upload(reinterpret_cast<const int4*>(host.segs.data()), host.segs.size());
    long_rows.alloc(host.long_rows.size(), false);
    long_rows.upload(reinterpret_cast<const int4*>(host.long_rows.data()), host.long_rows.size());
    long_partial.alloc(host.n_partials);
    long_counter.alloc(host.long_rows.size());
    dev.nrows = host.nrows;
    dev.nslices = (int)host.slices.size();
    dev.nblocks_body = (dev.nslices + kThreads / 32 - 1) / (kThreads / 32);
    dev.nblocks_full = dev.nblocks_body;
    dev.nsegs = (int)host.segs.size();
    dev.slices = slices.p; dev.col = col.p; dev.val = val.p; dev.segs = segs.p; dev.long_rows = long_rows.p;
    dev.lcol = lcol.p; dev.lval = lval.p; dev.long_partial = long_partial.p; dev.long_counter = long_counter.p;
    // the big host copies are not needed any more
    RawVec<int>().swap(host.col); RawVec<double>().swap(host.val);
    std::vector<int>().swap(host.lcol); std::vector<double>().swap(host.lval);
  }
  int grid() const { return dev.nblocks_body + dev.nsegs; }
  int grid_full() const { return dev.nblocks_full + dev.nsegs; }   // launch shape of the check kernels (and the larger of the two)
};

struct CudaEvent {   // RAII: released on every exit path
  cudaEvent_t e = nullptr;
  CudaEvent() { CUDA_OK(cudaEventCreate(&e)); }
  ~CudaEvent() { if (e) cudaEventDestroy(e); }
  CudaEvent(const CudaEvent&) = delete;
  CudaEvent& operator=(const CudaEvent&) = delete;
  operator cudaEvent_t() const { return e; }
};

// Logical shards (several ranks of ONE process, normally on one device): host-side rendezvous of the ranks' solve threads.
// A rank's barrier kernel spins until its peers' kernels signal; on one device that needs the peers' kernels to be
// schedulable -- anything on a peer's host thread that makes the driver serialise against running kernels (graph
// instantiation / upload, allocations) must therefore happen BEFORE the first spinning kernel of any rank is launched.
struct LocalGroup {
  std::mutex m;
  std::condition_variable cv;
  int world = 0, count = 0;
  unsigned long long gen = 0;
  bool shared[2] = {false, false};
  // returns rank 0's `v` to every rank (rank < 0: a plain rendezvous).  The value sits in the slot of the generation's
  // parity: rank 0 writes that slot again two generations later, which it cannot reach before every rank has passed the
  // generation in between, i.e. has read this one.
  bool arrive_and_wait(int rank = -1, bool v = false) {
    std::unique_lock<std::mutex> lk(m);
    const unsigned long long g = gen;
    if (rank == 0) shared[g & 1] = v;
    if (++count == world) { count = 0; gen++; cv.notify_all(); return shared[g & 1]; }
    if (!cv.wait_for(lk, std::chrono::seconds(120), [&] { return gen != g; })) {
      count--;
      throw std::runtime_error("logical shards: a peer rank's solve thread did not arrive");
    }
    return shared[g & 1];
  }
};

struct Residuals {      // CUPDLPresobj for one iterate
  double pobj = 0, dobj = 0, pfeas = 0, dfeas = 0, gap = 0, relgap = 0;
  double pinf_obj = 0, pinf_res = 1, dinf_obj = 0, dinf_res = 1;
};

}  // namespace b200

using namespace b200;

struct b200pdlp_form { StdForm f; };

struct b200pdlp_problem {
  StdForm form;
  int rank = 0, world = 1, device = 0;
  int r0 = 0, r1 = 0;              // local rows [r0,r1) of the permuted matrix
  int n = 0, m = 0, ml = 0;        // form cols, global rows, local rows
  DeviceMatrix A, AT;              // A_local (ml x n), A_local^T (n x ml)
  Csr csr_local;                   // A_local in standard-form order (tests)
  std::vector<int> rperm, rinv;    // device row order: rperm[new] = old local row
  std::vector<int> cperm, cinv;    // device column order: cperm[new] = old column (same on every rank)
  int neq_local = 0;               // local equality rows (they stay first under rperm)
  // multi-GPU column sharding (world > 1): rank g owns device columns [c0, c0 + nl_real); n-vectors are
  // allocated with nl = shard_len entries (zero padded); full vectors use G segments of seg_len
  int nl = 0, nl_real = 0, c0 = 0, shard_len = 0, seg_len = 0;
  DevBuf<double> xfull, part, red, send, recv;
  DevBuf<int> at_outpos;           // A_g^T body row -> position in the segmented partial vector
  // fused P2P path
  std::vector<int> row_bounds;     // row offsets of every rank's block
  // HiPDLP mode (reflected Halpern PDHG): its own iterate set; cost/lower/upper/colscale/rowscale/rhs (= row lower) are shared
  struct HipBuffers {
    DevBuf<double> x, y, xn, yn, rx, ry, xa, ya, aty, axp, atyp, dy, atdy, hslack, sp, sn, rup;
    DevBuf<HipState> state;
    HipState* hstate = nullptr;    // pinned
    cudaGraphExec_t graph = nullptr;
    long long graph_launches = 0;  // kernels in `graph`
    ~HipBuffers() { if (graph) cudaGraphExecDestroy(graph); if (hstate) pinned_cache_free(hstate); }
  } hip;
  // HiPDLP on several GPUs (b200pdlp_solve_hipdlp_multi): every rank's problem, by rank (empty on one GPU).  This rank owns
  // device rows [hip_r0, hip_r1) and device columns [hip_c0, hip_c1) of the one-GPU orders; its vectors are full length.
  std::vector<b200pdlp_problem*> hip_peers;
  int hip_r0 = 0, hip_r1 = 0, hip_c0 = 0, hip_c1 = 0;
  bool local_link = false;         // peers are problems of this process (logical shards, b200pdlp_p2p_link_local)
  std::shared_ptr<b200::LocalGroup> group;   // their host-side rendezvous
  bool no_graph = false;           // B200PDLP_NO_GRAPH: every pass and check as direct launches (debugging aid)
  bool p2p = false;
  PeerPtrs peers{};
  std::vector<void*> ipc_opened;
  DevBuf<unsigned long long> flags, epochs;
  DevBuf<int> fault;
  cudaStream_t stream = nullptr;
  // side stream + fork/join events: the two residual sweeps of a check are independent and neither fills the device
  // (296 / 592 CTAs), so they run next to each other (inside the check's graph: two branches)
  cudaStream_t side_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // n-vectors (replicated across ranks)
  DevBuf<double> x[2], aty[2], xsum, xavg, atyavg, xlr, cost, lower, upper, colscale;
  // m_local-vectors
  DevBuf<double> y[2], ax[2], ysum, yavg, axavg, ylr, rhs, rowscale;
  DevBuf<double> redbuf;           // all-reduce staging: n + 16
  DevBuf<double> partials;         // reduction scratch
  DevBuf<unsigned> counters;
  DevBuf<double> outs;             // device scalars written by check kernels
  DevBuf<PdhgState> state;
  PdhgState* hstate = nullptr;     // pinned mirror
  double* houts = nullptr;         // pinned
  double* hflag = nullptr;         // pinned: time-limit flag of the speculative check
  ncclComm_t comm = nullptr;
  cudaGraphExec_t graph_main = nullptr, graph_small = nullptr;
  int graph_main_passes = 0, graph_small_passes = 0;
  // device-side check iterations (tree mode, one GPU): control block, its pinned mirror, the time-limit word the
  // device reads from mapped host memory, graphs of 4/8/16/32 passes (captured on demand) and of the check sequence
  // device-resident prologue (device_prep.cu): the standard form never exists on the host; the index maps of the
  // formulation and the device orderings stay in HBM, the host keeps scalars only
  bool dev_form = false;
  DevicePrologue prep;
  double beta_cost_sq = 0.0, beta_rhs_sq = 0.0;   // |c|^2, |b|^2 of the scaled data (tree sums)
  DevBuf<double> io_col, io_row;   // staging of the hot start / the returned solution (original order)
  DevBuf<SolveCtl> ctl;
  SolveCtl* hctl = nullptr;        // pinned
  int* htime = nullptr;            // pinned + mapped
  DevBuf<double> trace_dev;
  cudaGraphExec_t graph_pow2[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // 1 << k passes
  cudaGraphExec_t graph_check = nullptr;
  int check_launches[2] = {0, 0};                 // kernels in graph_check / graph_check_light
  cudaGraphExec_t graph_check_light = nullptr;   // the dense-check phase's check: two sweeps instead of two SpMV (see kDenseChecks)
  DevBuf<double> axsum, atysum;                   // A xSum (ml), A'ySum (n): carried by the passes while iter < kDenseChecks
  long long launches = 0;
  int kernels_per_pass = 4;

  ~b200pdlp_problem() {
    if (stream) cudaStreamSynchronize(stream);   // the buffers go back to the block cache: nothing may still use them
    if (dev_form) { prep.A.release(); prep.AT.release(); prep.release_arrays(); prep.release_form(); }   // (A / AT: only if never adopted)
    if (graph_main) cudaGraphExecDestroy(graph_main);
    if (graph_small) cudaGraphExecDestroy(graph_small);
    for (cudaGraphExec_t g : graph_pow2) if (g) cudaGraphExecDestroy(g);
    if (graph_check) cudaGraphExecDestroy(graph_check);
    if (graph_check_light) cudaGraphExecDestroy(graph_check_light);
    if (hctl) pinned_cache_free(hctl);
    if (htime) pinned_cache_free(htime);
    for (void* q : ipc_opened) cudaIpcCloseMemHandle(q);
    if (comm) NcclApi::get().CommDestroy(comm);
    if (hstate) pinned_cache_free(hstate);
    if (houts) pinned_cache_free(houts);
    if (hflag) pinned_cache_free(hflag);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
    if (side_stream) cudaStreamDestroy(side_stream);
    if (stream) cudaStreamDestroy(stream);
  }
  ReduceScratch rs(int slot, int len) const {
    // slot-private partial arrays: 16 accumulators x kMaxEwBlocks-or-nblocks each
    double* t = (ordered && len <= ordered_cap) ? terms.p + (size_t)slot * 16 * ordered_cap : nullptr;
    return ReduceScratch{partials.p + (size_t)slot * scratch_stride, counters.p + slot, t, len};
  }
  size_t scratch_stride = 0;
  DevBuf<double> terms;            // ordered-mode term scratch
  bool ordered = false;
  int ordered_cap = 0;
};

namespace b200 {

static constexpr int kSlotK1 = 0, kSlotK2 = 1, kSlotK3 = 2, kSlotChk = 3, kNumSlots = 4;
static constexpr int kOutsCount = 64;

static void set_device(const b200pdlp_problem* p) { CUDA_OK(cudaSetDevice(p->device)); }
static void ensure_side_stream(b200pdlp_problem* p);

static void allreduce_inplace(b200pdlp_problem* p, double* dptr, size_t count) {
  if (p->world <= 1) return;
  if (!p->comm) throw Error(B200PDLP_ERR_STATE, "world > 1 but b200pdlp_comm_init was not called");
  NCCL_OK(nccl().AllReduce(dptr, dptr, count, ncclDouble, ncclSum, p->comm, p->stream));
}

static void need_comm(b200pdlp_problem* p) {
  if (!p->comm) throw Error(B200PDLP_ERR_STATE, "world > 1 but b200pdlp_comm_init was not called");
}
// shards (+ scalar tails) of every rank -> xfull
static void gather_shards(b200pdlp_problem* p) {
  need_comm(p);
  NCCL_OK(nccl().AllGather(p->send.p, p->xfull.p, (size_t)p->seg_len, ncclDouble, p->comm, p->stream));
}
// sum over ranks of `part`, my segment -> red
static void reduce_scatter_part(b200pdlp_problem* p) {
  need_comm(p);
  NCCL_OK(nccl().ReduceScatter(p->part.p, p->red.p, (size_t)p->seg_len, ncclDouble, ncclSum, p->comm, p->stream));
}
// position of device column j in a segmented full vector
static inline size_t seg_pos(const b200pdlp_problem* p, int j) {
  return p->world == 1 ? (size_t)j : (size_t)(j / p->shard_len) * p->seg_len + (size_t)(j % p->shard_len);
}

// sum over ranks of k (<= 32) doubles at dptr, in place
static void allreduce_small(b200pdlp_problem* p, double* dptr, int k) {
  if (p->world <= 1) return;
  if (p->p2p) { launch_p2p_exchange(p->stream, dptr, k, p->peers, p->world, p->rank, p->epochs.p, p->fault.p); p->launches++; }
  else allreduce_inplace(p, dptr, (size_t)k);
}

// B200PDLP_TIMING=1: wall-clock laps of the non-iterating parts on stderr (where does a short solve's time go)
struct Laps {
  bool on = getenv("B200PDLP_TIMING") != nullptr;
  int rank = -1;
  std::chrono::steady_clock::time_point t = std::chrono::steady_clock::now();
  void operator()(const char* phase, const char* what) {
    if (!on) return;
    const auto t1 = std::chrono::steady_clock::now();
    if (rank >= 0) fprintf(stderr, "[b200pdlp %s r%d] %-28s %8.1f ms\n", phase, rank, what, std::chrono::duration<double, std::milli>(t1 - t).count());
    else fprintf(stderr, "[b200pdlp %s] %-28s %8.1f ms\n", phase, what, std::chrono::duration<double, std::milli>(t1 - t).count());
    t = t1;
  }
};

// experiment (B200PDLP_SPMV_CTAS_PER_SM=k, one GPU, tree mode): the SpMV bodies run on a persistent grid of k CTAs per SM and
// walk their slices in a software pipeline (spmv_sell_kernel<Epi, true>) instead of one CTA per 8 slices
static void apply_spmv_grid(b200pdlp_problem* p) {
  if (p->world != 1 || p->ordered) return;
  auto val = [](const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; };
  const int both = val("B200PDLP_SPMV_CTAS_PER_SM", -1);
  // measured on one H100 (S3, DESIGN.md section 6): the pipelined walk at 3 CTAs per SM helps A'y a little (K3 87.3 -> 85.8
  // us) and hurts A x (K2 92.8 -> 99.5 us), so it is the default for A' only
  // ... unless the matrix is structured: where a warp's gathers share sectors (the device prologue samples it: distinct
  // 32-byte sectors per live lane, 1.0 on a uniformly random pattern, 0.25 on consecutive columns) the gather pipe is not
  // the limit and the persistent shape helps A x as well (S3D with the tiled shape off: K2 67.8 -> 65.6 us)
  int ka_default = 0;
  if (p->dev_form && p->prep.sc.a_lanes > 0 && 2 * p->prep.sc.a_sectors <= p->prep.sc.a_lanes) ka_default = 4;
  const int ka = val("B200PDLP_SPMV_A_CTAS_PER_SM", both >= 0 ? both : ka_default);
  const int kat = val("B200PDLP_SPMV_AT_CTAS_PER_SM", both >= 0 ? both : 3);
  int sms = 132;   // (H100 SXM; the query below sets it)
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, p->device);
  auto apply = [&](DeviceMatrix& M, int k) {
    if (k > 0 && M.dev.nblocks_body > sms * k) { M.dev.nblocks_body = sms * k; M.dev.pipelined = 1; }
  };
  // Tiled shape (shared-memory staged gathers, spmv_sell_tile_kernel): B200PDLP_TILE=1 (bulk copy by the TMA unit) or 2
  // (cooperative loads) for both matrices, B200PDLP_TILE_A / _AT for one.  Only where every tile's window fits the staging
  // buffer and there are enough tiles to occupy the device.
  auto tile = [&](DeviceMatrix& M, int mode) {
    // (a few tiles may miss -- wrap-around patterns put both ends of the vector into one window: those gather from global memory)
    if (mode <= 0 || M.ntiles <= 0 || 10 * M.tiles_staged < 9 * M.ntiles) return false;
    if (2 * M.ntiles < sms && !getenv("B200PDLP_TILE_FORCE")) return false;   // fewer than half the SMs would have a tile (tests force it)
    M.dev.tiled = mode; M.dev.tile_lo = M.tile_lo.p; M.dev.tile_w = M.tile_w.p;
    M.dev.nblocks_body = M.ntiles; M.dev.pipelined = 0;
    return true;
  };
  // default: tiled (bulk copy) wherever the prologue found windows that fit for >= 90 % of the tiles (B200PDLP_TILE=0: off).
  // Measured on one H100 (DESIGN.md section 6): S3B K2 74.3 -> 63.8 us, 5.99 k -> 6.64 k it/s; S3D K2 65.6 -> 62.8 us against
  // the persistent shape; S3 (random columns): no window fits, never chosen.
  const int tdef = p->dev_form ? 1 : 0;
  const int tboth = val("B200PDLP_TILE", -1);
  const int ta = val("B200PDLP_TILE_A", tboth >= 0 ? tboth : tdef);
  const int tat = val("B200PDLP_TILE_AT", tboth >= 0 ? tboth : tdef);
  if (!tile(p->A, ta)) apply(p->A, ka);
  if (!tile(p->AT, tat)) apply(p->AT, kat);
  if (getenv("B200PDLP_TIMING"))
    fprintf(stderr, "[b200pdlp setup] SpMV shapes: A %s (%d CTAs, tiles staged %d/%d)  A' %s (%d CTAs, tiles staged %d/%d)\n",
            p->A.dev.tiled ? "tiled" : (p->A.dev.pipelined ? "persistent" : "one slice per warp"), p->A.dev.nblocks_body,
            p->A.tiles_staged, p->A.ntiles,
            p->AT.dev.tiled ? "tiled" : (p->AT.dev.pipelined ? "persistent" : "one slice per warp"), p->AT.dev.nblocks_body,
            p->AT.tiles_staged, p->AT.ntiles);
}

// ---- problem construction.  Every creator below is a sequence of these steps plus what is its own.

// the number of CUDA devices; none is an error: the engine has no CPU fallback
static int device_count_checked() {
  int ndev = 0;
  const cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    throw Error(B200PDLP_ERR_CUDA, std::string("no CUDA device: the engine has no CPU fallback (") + cudaGetErrorString(e) + ")");
  return ndev;
}

// rank `rank` of `world` on `device` (< 0: the caller's current device): selects the device and creates the problem's stream
static void open_problem(b200pdlp_problem* p, int device, int rank, int world) {
  device_count_checked();
  if (device >= 0) p->device = device; else CUDA_OK(cudaGetDevice(&p->device));
  set_device(p);
  p->rank = rank; p->world = world;
  CUDA_OK(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
}

// the only caller of DevicePrologue::run: bad input -> ERR_ARG, CUDA errors -> ERR_CUDA; a host std::bad_alloc passes
// through (guarded: ERR_ALLOC)
static void run_prologue(DevicePrologue& P, cudaStream_t s, const b200pdlp_lp& lp, bool do_scale) {
  try {
    P.run(s, lp, do_scale, /*long_threshold=*/512);
  } catch (const std::invalid_argument& ex) {
    throw Error(B200PDLP_ERR_ARG, ex.what());
  } catch (const std::runtime_error& ex) {
    throw Error(B200PDLP_ERR_CUDA, ex.what());
  }
}

// A prologue run on the current device that no single problem holds: its stream, and whatever no problem adopted (A / A',
// the rank blocks, the arrays, the kept form), released when the holder goes.
struct TempPrologue {
  int device = 0;
  cudaStream_t stream = nullptr;
  DevicePrologue P;
  TempPrologue() {
    CUDA_OK(cudaGetDevice(&device));
    CUDA_OK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  }
  TempPrologue(const TempPrologue&) = delete;
  TempPrologue& operator=(const TempPrologue&) = delete;
  ~TempPrologue() {
    cudaSetDevice(device);
    cudaStreamSynchronize(stream);
    cudaStreamDestroy(stream);
    P.A.release(); P.AT.release(); P.release_blocks(); P.release_arrays(); P.release_form();
  }
};

// the scalars of the standard form a device prologue built (the form itself stays on the device)
static StdForm form_scalars(const b200pdlp_lp& lp, const DevicePrologue& P) {
  StdForm f;
  f.hipdlp = P.hipdlp; f.scaled = P.sc.scaled != 0;
  f.n = P.arr.n; f.m = P.arr.m; f.nnz = P.arr.nnz; f.neq = P.arr.neq; f.n_orig = P.arr.n0;
  f.sense = lp.sense; f.offset = lp.offset;
  f.norm_cost = std::sqrt(P.sc.norm_cost_sq); f.norm_rhs = std::sqrt(P.sc.norm_rhs_sq);
  f.amax = P.sc.amax;
  return f;
}

// the standard form the prologue kept on the device (DevicePrologue::keep_form) into f, whose sizes are set
static void download_form(const DevStdForm& d, StdForm& f, cudaStream_t s) {
  const int n = f.n, m = f.m, nnz = f.nnz;
  f.cbeg.resize(n + 1); f.cidx.resize(nnz); f.cval.resize(nnz);
  f.cost.resize(n); f.lower.resize(n); f.upper.resize(n); f.col_scale.resize(n); f.rhs.resize(m); f.row_scale.resize(m);
  f.rptr.resize(m + 1); f.rpos.resize(nnz); f.rcol.resize(nnz);
  auto dn = [&](auto& h, const auto* dv) {
    if (!h.empty()) CUDA_OK(cudaMemcpyAsync(h.data(), dv, h.size() * sizeof(h[0]), cudaMemcpyDeviceToHost, s));
  };
  dn(f.cbeg, d.cbeg); dn(f.cidx, d.cidx); dn(f.cval, d.cval);
  dn(f.cost, d.cost); dn(f.lower, d.lower); dn(f.upper, d.upper); dn(f.col_scale, d.colscale); dn(f.rhs, d.rhs); dn(f.row_scale, d.rowscale);
  dn(f.rptr, d.rptr); dn(f.rpos, d.rpos); dn(f.rcol, d.rcol);
  CUDA_OK(cudaStreamSynchronize(s));
}

// dimensions of a host layout (host_prep.cpp build_layout); p->form holds the standard form
static void take_layout(b200pdlp_problem* p, HostLayout&& L) {
  p->n = p->form.n; p->m = p->form.m;
  p->r0 = L.r0; p->r1 = L.r1; p->ml = L.ml; p->neq_local = L.neq_local; p->ordered = L.ordered;
  p->row_bounds = std::move(L.bounds);
  p->nl = L.nl; p->nl_real = L.nl_real; p->c0 = L.c0; p->shard_len = L.shard_len; p->seg_len = L.seg_len;
  p->csr_local = std::move(L.csr_local);
  p->rperm = std::move(L.rperm); p->rinv = std::move(L.rinv);
  p->cperm = std::move(L.cperm); p->cinv = std::move(L.cinv);
  p->A.host = std::move(L.A); p->AT.host = std::move(L.AT);
  if (L.world > 1) p->at_outpos.from(L.at_outpos);
}

// dimensions of a rank that holds every row and full-length vectors (one GPU, and the HiPDLP shards); p->form holds the scalars
static void set_full_length_dims(b200pdlp_problem* p) {
  const StdForm& f = p->form;
  const int n = f.n, m = f.m;
  p->n = n; p->m = m; p->ml = m; p->r0 = 0; p->r1 = m; p->neq_local = f.neq;
  p->row_bounds = {0, m};
  p->nl = p->nl_real = n; p->c0 = 0; p->shard_len = n; p->seg_len = n;
  p->csr_local.nrows = m; p->csr_local.ncols = n; p->csr_local.nnz = f.nnz;   // dimensions only (built on demand)
}

// what a problem that holds every row takes from a device prologue: the form's scalars, the dimensions and the device-order
// vectors, adopted on one GPU; in block mode every rank takes its own copy (the matrices are the caller's: A / A' or a block)
static void take_prologue(const b200pdlp_lp& lp, DevicePrologue& P, b200pdlp_problem* p) {
  p->form = form_scalars(lp, P);
  set_full_length_dims(p);
  DevProblemArrays& a = P.arr;
  auto take = [&](DevBuf<double>& d, double*& src, int len) {
    if (P.world == 1) { d.adopt(src, len); src = nullptr; return; }
    d.alloc(len, false);
    if (len > 0) CUDA_OK(cudaMemcpyAsync(d.p, src, (size_t)len * sizeof(double), cudaMemcpyDeviceToDevice, p->stream));
  };
  take(p->cost, a.cost, a.n); take(p->lower, a.lower, a.n); take(p->upper, a.upper, a.n); take(p->colscale, a.colscale, a.n);
  take(p->rhs, a.rhs, a.m); take(p->rowscale, a.rowscale, a.m);
  if (P.hipdlp) take(p->hip.rup, a.rup, a.m);
}

// a host vector into device order: d[i] = v[offset + perm[i]] for i < len, then `pad` up to `size` entries
static void upload_permuted(DevBuf<double>& d, const std::vector<double>& v, const int* perm, int offset, int len, int size,
                            double pad = 0.0) {
  std::vector<double> t((size_t)std::max(size, 1), pad);
  for (int i = 0; i < len; i++) t[i] = v[offset + perm[i]];
  d.alloc(size, false);
  d.upload(t.data(), size);
}

// reduction scratch (sized for the larger launch shape, so after apply_spmv_grid), the check's device scalars and their pinned
// mirror.  The term scratch has p->ordered_cap entries per accumulator: set by pdlp in ordered mode, 0 for HiPDLP, whose check
// reduces without it.  zero: every buffer zeroed at allocation; the counters are zero before the first launch either way.
static void alloc_scratch(b200pdlp_problem* p, bool zero) {
  const size_t maxgrid = std::max<size_t>(kMaxEwBlocks, std::max(p->A.grid_full(), p->AT.grid_full()));
  p->scratch_stride = 24 * maxgrid;
  p->partials.alloc(p->scratch_stride * kNumSlots, zero);
  p->counters.alloc(kNumSlots, zero);
  if (!zero) CUDA_OK(cudaMemsetAsync(p->counters.p, 0, kNumSlots * sizeof(unsigned), p->stream));
  p->terms.alloc(p->ordered_cap > 0 ? (size_t)kNumSlots * 16 * p->ordered_cap : 1, zero);
  p->outs.alloc(kOutsCount, zero);
  p->houts = static_cast<double*>(pinned_cache_alloc(kOutsCount * sizeof(double), false));
}

// the PDHG solve's pinned mirrors, zeroed
static void alloc_host_mirrors(b200pdlp_problem* p) {
  p->hstate = static_cast<PdhgState*>(pinned_cache_alloc(sizeof(PdhgState), false));
  p->hflag = static_cast<double*>(pinned_cache_alloc(4 * sizeof(double), false));   // [0] time-limit flag, [2] read-back of the barrier fault word
  memset(p->hflag, 0, 4 * sizeof(double));
  memset(p->hstate, 0, sizeof(PdhgState));
}

// the HiPDLP shards' arrival words, one per peer (hip_barrier_kernel), epoch and fault word
static void alloc_peer_words(b200pdlp_problem* p) {
  p->flags.alloc(kMaxPeers);
  p->epochs.alloc(1);
  p->fault.alloc(1);
}

// staging of the hot start and of the solution in original order (device postsolve)
static void alloc_postsolve_staging(b200pdlp_problem* p) {
  p->io_col.alloc((size_t)2 * std::max(p->form.n_orig, 1), false);
  p->io_row.alloc((size_t)2 * std::max(p->m, 1), false);
}

// The size rule of both device prologues.  Ordered mode keeps the host prologue; it is decided on the STANDARD FORM's size,
// n = num_col + one slack column per ranged or free row (CupdlpWrapper.cpp:328-345; `inf` is the mode's infinite row bound),
// so count them when the answer depends on it.  An empty matrix keeps it too.
static int std_form_cols(const b200pdlp_lp& lp, double inf) {
  int nslack = 0;
  for (int i = 0; i < lp.num_row; i++) {
    const bool lo = lp.row_lower[i] > -inf, up = lp.row_upper[i] < inf;
    nslack += (lo && up && lp.row_lower[i] != lp.row_upper[i]) || (!lo && !up);
  }
  return lp.num_col + nslack;
}
static bool device_prep_fits(const b200pdlp_lp& lp, int ordered_max, double inf) {
  const int omax = ordered_max == 0 ? 4096 : ordered_max;
  if (omax > 0 && lp.num_col <= omax && lp.num_row <= omax && std_form_cols(lp, inf) <= omax) return false;
  return lp.num_col > 0 && lp.num_row > 0 && lp.a_start[lp.num_col] > 0;
}

// Several GPUs (default; B200PDLP_MG_DEVICE_PREP=0 for the host path): every rank needs the whole scaled standard form to cut its shard out of
// it.  Instead of G processes running the host prologue side by side (they share the host's cores and memory bandwidth),
// each rank formulates and scales on ITS GPU (a few milliseconds, identical bits on every rank) and downloads the result;
// the per-rank layouts are then built by the host as before.
static void device_form_to_host(const b200pdlp_lp& lp, const b200pdlp_params& prm, StdForm& f) {
  TempPrologue T;
  T.P.keep_form = true;
  T.P.stop_after_scaling = true;
  run_prologue(T.P, T.stream, lp, prm.scaling != 0);
  f = form_scalars(lp, T.P);
  download_form(T.P.form, f, T.stream);
  const DevProblemArrays& a = T.P.arr;
  f.row_new_idx.resize(f.m); f.row_class.resize(f.m);
  CUDA_OK(cudaMemcpy(f.row_new_idx.data(), a.row_new_idx, (size_t)f.m * sizeof(int), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(f.row_class.data(), a.row_class, (size_t)f.m * sizeof(int), cudaMemcpyDeviceToHost));
}

// shared_form != nullptr: the standard form was formulated and scaled already (by another rank of this process)
static void create_problem(const b200pdlp_lp& lp, const b200pdlp_params& prm, int rank, int world, b200pdlp_problem* p,
                           const StdForm* shared_form = nullptr) {
  NvtxRange nvtx("b200pdlp: prologue (host threads) + upload");
  open_problem(p, prm.device, rank, world);
  Laps laps;
  auto lap = [&](const char* what) { laps("setup", what); };
  bool mg_dev_form = false;
  if (!shared_form && world > 1 && lp.num_row > 0 && lp.num_col > 0 && lp.a_start[lp.num_col] > 0) {
    // default (the ranks do not compete for the host's cores and memory bandwidth): B200PDLP_MG_DEVICE_PREP=0 keeps the host
    // formulate + scale
    mg_dev_form = true;
    if (const char* ev = getenv("B200PDLP_MG_DEVICE_PREP")) mg_dev_form = atoi(ev) != 0;
  }
  if (shared_form) {
    p->form = *shared_form;
    lap("copy of the scaled form");
  } else if (mg_dev_form) {
    device_form_to_host(lp, prm, p->form);
    lap("formulate + scale on the device, download");
  } else {
    formulate(lp, p->form);
    lap("formulate");
  }
  if (!shared_form && !mg_dev_form) scale(p->form, prm.scaling != 0);
  lap("scale");
  StdForm& f = p->form;
  {
    // host layout (row block, device orderings, sliced-ELL of A_g and A_g^T): host_prep.cpp build_layout
    HostLayout L;
    build_layout(f, rank, world, prm.ordered_max, L, lap);
    take_layout(p, std::move(L));
  }
  const int n = p->n, ml = p->ml, nl = p->nl;
  if (world == 1) ensure_side_stream(p);
  p->A.upload();
  p->AT.upload();
  lap("matrix upload");
  apply_spmv_grid(p);
  for (int k = 0; k < 2; k++) { p->x[k].alloc(nl); p->aty[k].alloc(nl); p->y[k].alloc(ml); p->ax[k].alloc(ml); }
  p->xsum.alloc(nl); p->xavg.alloc(nl); p->atyavg.alloc(nl); p->xlr.alloc(nl);
  p->ysum.alloc(ml); p->yavg.alloc(ml); p->axavg.alloc(ml); p->ylr.alloc(ml);
  if (!p->ordered) { p->axsum.alloc(ml); p->atysum.alloc(nl); }
  if (world > 1) {
    p->xfull.alloc((size_t)world * p->seg_len); p->part.alloc((size_t)world * p->seg_len);
    p->recv.alloc((size_t)world * p->seg_len);
    p->red.alloc(p->seg_len); p->send.alloc(p->seg_len);
    p->flags.alloc(5 * kMaxPeers + 2 * kMaxPeers * 32);   // [3][16] flags, [16][2] pass mailbox, [2][16][32] check mailbox
    p->epochs.alloc(16); p->fault.alloc(1);
  }
  // my shard of the column vectors in device order (padding: cost 0, bounds [0,0], scale 1) and my rows
  const int* cperm = p->cperm.data() + p->c0;
  upload_permuted(p->cost, f.cost, cperm, 0, p->nl_real, nl); upload_permuted(p->lower, f.lower, cperm, 0, p->nl_real, nl);
  upload_permuted(p->upper, f.upper, cperm, 0, p->nl_real, nl); upload_permuted(p->colscale, f.col_scale, cperm, 0, p->nl_real, nl, 1.0);
  upload_permuted(p->rhs, f.rhs, p->rperm.data(), p->r0, ml, ml); upload_permuted(p->rowscale, f.row_scale, p->rperm.data(), p->r0, ml, ml);
  p->redbuf.alloc((size_t)std::max(n, p->m) + 16);
  p->ordered_cap = p->ordered ? std::max(std::max(p->n, p->m), 1) : 0;
  alloc_scratch(p, true);
  p->state.alloc(1);
  alloc_host_mirrors(p);
  CUDA_OK(cudaDeviceSynchronize());
  lap("vectors + scratch");
}

// One GPU, tree mode: the whole prologue on the device (device_prep.cu).  params.device_scaling = -1 or
// B200PDLP_DEVICE_PREP=0 keeps the host prologue (its tested twin); ordered mode (small problems, bit-identical
// trajectories) and several GPUs always do.
static bool use_device_prep(const b200pdlp_lp& lp, const b200pdlp_params& prm, int world) {
  if (world != 1) return false;
  if (const char* e = getenv("B200PDLP_DEVICE_PREP")) { if (atoi(e) == 0) return false; }
  else if (prm.device_scaling == -1) return false;   // the host prologue on request (check_params allows 0 and -1 only)
  return device_prep_fits(lp, prm.ordered_max, 1e20);
}

// the engine takes over one sliced-ELL matrix the device prologue built
static void adopt_matrix(DeviceMatrix& M, DevSellOwned& O) {
  M.slices.adopt(O.slices, O.nslices); M.col.adopt(O.col, (size_t)O.padded + 32); M.val.adopt(O.val, (size_t)O.padded + 32);
  M.segs.adopt(O.segs, O.nsegs); M.long_rows.adopt(O.long_rows, O.nlong); M.lcol.adopt(O.lcol, (size_t)O.lcount);
  M.lval.adopt(O.lval, (size_t)O.lcount); M.long_partial.adopt(O.long_partial, O.nsegs);
  M.long_counter.adopt(O.long_counter, O.nlong);
  if (O.ntiles > 0) { M.tile_lo.adopt(O.tile_lo, O.ntiles); M.tile_w.adopt(O.tile_w, O.ntiles); }
  M.ntiles = O.ntiles; M.tiles_staged = O.tiles_staged;
  M.host.nrows = O.nrows; M.host.ncols = O.ncols; M.host.padded = O.padded; M.host.lcount = O.lcount; M.host.n_partials = O.nsegs;
  M.dev.nrows = O.nrows; M.dev.nslices = O.nslices;
  M.dev.nblocks_body = (O.nslices + kThreads / 32 - 1) / (kThreads / 32);
  M.dev.nblocks_full = M.dev.nblocks_body;
  M.dev.nsegs = O.nsegs;
  M.dev.slices = M.slices.p; M.dev.col = M.col.p; M.dev.val = M.val.p; M.dev.segs = M.segs.p; M.dev.long_rows = M.long_rows.p;
  M.dev.lcol = M.lcol.p; M.dev.lval = M.lval.p; M.dev.long_partial = M.long_partial.p; M.dev.long_counter = M.long_counter.p;
  O = DevSellOwned();   // ownership moved
}

static void create_problem_device(const b200pdlp_lp& lp, const b200pdlp_params& prm, b200pdlp_problem* p) {
  NvtxRange nvtx("b200pdlp: prologue (device)");
  open_problem(p, prm.device, 0, 1);
  Laps lap;
  ensure_side_stream(p);
  p->dev_form = true;
  if (getenv("B200PDLP_KEEP_FORM")) p->prep.keep_form = true;
  DevicePrologue& P = p->prep;
  run_prologue(P, p->stream, lp, prm.scaling != 0);
  lap("setup", "device prologue");
  if (lap.on)
    fprintf(stderr, "[b200pdlp setup] sectors per gathered lane (sampled): A %.3f  A' %.3f\n",
            P.sc.a_lanes ? (double)P.sc.a_sectors / P.sc.a_lanes : 0.0, P.sc.at_lanes ? (double)P.sc.at_sectors / P.sc.at_lanes : 0.0);
  take_prologue(lp, P, p);
  p->beta_cost_sq = P.sc.beta_cost_sq; p->beta_rhs_sq = P.sc.beta_rhs_sq;
  const int n = p->n, m = p->m;
  adopt_matrix(p->A, P.A);
  adopt_matrix(p->AT, P.AT);
  apply_spmv_grid(p);
  // iterates and scratch: uninitialised (the solve's initial-point kernels write every entry they read)
  for (int k = 0; k < 2; k++) { p->x[k].alloc(n, false); p->aty[k].alloc(n, false); p->y[k].alloc(m, false); p->ax[k].alloc(m, false); }
  p->xsum.alloc(n, false); p->xavg.alloc(n, false); p->atyavg.alloc(n, false); p->xlr.alloc(n, false);
  p->ysum.alloc(m, false); p->yavg.alloc(m, false); p->axavg.alloc(m, false); p->ylr.alloc(m, false);
  p->axsum.alloc(m, false); p->atysum.alloc(n, false);
  alloc_postsolve_staging(p);
  alloc_scratch(p, false);
  p->state.alloc(1, false);
  p->redbuf.alloc(16, false);
  alloc_host_mirrors(p);
  lap("setup", "vectors + scratch");
}

// host copies of what the device prologue keeps in HBM, fetched when a test accessor needs them
static void ensure_host_maps(b200pdlp_problem* p) {
  if (!p->dev_form || !p->rperm.empty() || p->m == 0) return;
  const DevProblemArrays& a = p->prep.arr;
  p->rperm.resize(p->m); p->rinv.resize(p->m); p->cperm.resize(p->n); p->cinv.resize(p->n);
  p->form.row_new_idx.resize(p->m); p->form.row_class.resize(p->m);
  CUDA_OK(cudaMemcpy(p->rperm.data(), a.rperm, (size_t)p->m * sizeof(int), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(p->rinv.data(), a.rinv, (size_t)p->m * sizeof(int), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(p->cperm.data(), a.cperm, (size_t)p->n * sizeof(int), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(p->cinv.data(), a.cinv, (size_t)p->n * sizeof(int), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(p->form.row_new_idx.data(), a.row_new_idx, (size_t)p->m * sizeof(int), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(p->form.row_class.data(), a.row_class, (size_t)p->m * sizeof(int), cudaMemcpyDeviceToHost));
}

// the scaled standard form itself (tests: b200pdlp_problem_get_vector / get_csr), when the prologue kept it
static void ensure_host_form(b200pdlp_problem* p) {
  if (!p->dev_form || !p->form.cbeg.empty()) return;
  const DevStdForm& d = p->prep.form;
  if (!d.cbeg) throw Error(B200PDLP_ERR_STATE, "the standard form was not kept on the device (one-shot solve)");
  download_form(d, p->form, p->stream);
  ensure_host_maps(p);
}

// ------------------------------------------------------------------ PDHG passes
static void enqueue_pass_mg(b200pdlp_problem* p);
static void enqueue_pass(b200pdlp_problem* p) {
  if (p->world > 1) { enqueue_pass_mg(p); return; }
  cudaStream_t s = p->stream;
  PdhgState* st = p->state.p;
  const ReduceScratch r1 = p->rs(kSlotK1, p->n), r2 = p->rs(kSlotK2, p->ml), r3 = p->rs(kSlotK3, p->n);
  launch_primal_step(s, p->n, st, p->x[0].p, p->x[1].p, p->aty[0].p, p->aty[1].p, p->cost.p, p->lower.p,
                     p->upper.p, p->xsum.p, r1);
  launch_spmv_dual(s, p->A.dev, st, p->x[0].p, p->x[1].p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p,
                   p->rhs.p, p->ysum.p, p->neq_local, 0, r2, p->axsum.p);
  launch_spmv_primal(s, p->AT.dev, st, p->y[0].p, p->y[1].p, p->x[0].p, p->x[1].p, p->aty[0].p, p->aty[1].p, r3, p->atysum.p);
  launch_step_rule(s, st, r1, primal_step_grid(p->n), r2, p->A.grid(), r3, p->AT.grid(), nullptr);
}

// world > 1: sharded primal step, all-gather, local rows, partial A^T y, reduce-scatter, step rule
static void enqueue_pass_mg(b200pdlp_problem* p) {
  cudaStream_t s = p->stream;
  PdhgState* st = p->state.p;
  const ReduceScratch r1 = p->rs(kSlotK1, p->nl), r2 = p->rs(kSlotK2, p->ml);
  if (p->p2p) {
    // fused compute + collective over NVLink peer memory (5 launches, no NCCL)
    launch_primal_shard_p2p(s, p->nl, st, p->x[0].p, p->x[1].p, p->aty[0].p, p->peers, p->world, p->rank, p->seg_len,
                            p->cost.p, p->lower.p, p->upper.p, p->xsum.p, r1, p->atysum.p);
    launch_p2p_barrier(s, 0, st, r1.partials, primal_shard_p2p_grid(p->nl), p->peers, p->world, p->rank, p->seg_len,
                       p->shard_len, p->epochs.p, p->fault.p);
    launch_spmv_dual_mg(s, p->A.dev, st, p->xfull.p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->rhs.p,
                        p->ysum.p, p->neq_local, r2, p->axsum.p);
    launch_spmv_partial_aty(s, p->AT.dev, st, p->y[0].p, p->y[1].p, p->part.p, p->at_outpos.p);
    launch_p2p_barrier(s, 1, st, r2.partials, p->A.grid(), p->peers, p->world, p->rank, p->seg_len, p->shard_len,
                       p->epochs.p, p->fault.p);
    return;
  }
  launch_primal_shard(s, p->nl, st, p->x[0].p, p->x[1].p, p->aty[0].p, p->red.p, p->cost.p, p->lower.p, p->upper.p,
                      p->xsum.p, p->send.p, r1);
  launch_stash_scalars(s, 1, st, r1.partials, primal_shard_grid(p->nl), p->send.p + p->shard_len, 1, 0);
  gather_shards(p);
  launch_spmv_dual_mg(s, p->A.dev, st, p->xfull.p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->rhs.p,
                      p->ysum.p, p->neq_local, r2);
  launch_stash_scalars(s, 2, st, r2.partials, p->A.grid(), p->part.p + p->shard_len, p->world, p->seg_len);
  launch_spmv_partial_aty(s, p->AT.dev, st, p->y[0].p, p->y[1].p, p->part.p, p->at_outpos.p);
  reduce_scatter_part(p);
  launch_step_rule_mg(s, st, p->xfull.p, p->world, p->seg_len, p->shard_len, p->red.p);
}

static cudaGraphExec_t capture_passes(b200pdlp_problem* p, int passes) {
  cudaGraph_t g = nullptr;
  CUDA_OK(cudaStreamBeginCapture(p->stream, cudaStreamCaptureModeThreadLocal));
  for (int i = 0; i < passes; i++) enqueue_pass(p);
  CUDA_OK(cudaStreamEndCapture(p->stream, &g));
  cudaGraphExec_t ge = nullptr;
  CUDA_OK(cudaGraphInstantiate(&ge, g, 0));
  CUDA_OK(cudaGraphDestroy(g));
  return ge;
}

static void fill_pow_tables(PdhgState* h) {
  // step_iter k takes values pow_base+1 ... ; entry t serves k = pow_base+1+t (cupdlp_step.c:279-284)
  h->pow_base = h->step_iter;
  for (int t = 0; t < kPowTab; t++) {
    const double k = (double)(h->step_iter + 1 + t);
    h->pow_red[t] = std::pow(k + 1.0, -0.3);
    h->pow_grow[t] = std::pow(k + 1.0, -0.6);
  }
}

static void push_state(b200pdlp_problem* p) {
  CUDA_OK(cudaMemcpyAsync(p->state.p, p->hstate, sizeof(PdhgState), cudaMemcpyHostToDevice, p->stream));
}
static void pull_state(b200pdlp_problem* p) {
  CUDA_OK(cudaMemcpyAsync(p->hstate, p->state.p, sizeof(PdhgState), cudaMemcpyDeviceToHost, p->stream));
  int* hfault = reinterpret_cast<int*>(p->hflag + 2);
  if (p->p2p) CUDA_OK(cudaMemcpyAsync(hfault, p->fault.p, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
  CUDA_OK(cudaStreamSynchronize(p->stream));
  // a barrier gave up waiting for a peer: stop here instead of iterating on inconsistent data
  if (p->p2p && *hfault) throw Error(B200PDLP_ERR_STATE, "P2P barrier timed out (a peer rank did not arrive)");
}
static void pull_outs(b200pdlp_problem* p, int count) {
  CUDA_OK(cudaMemcpyAsync(p->houts, p->outs.p, count * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  CUDA_OK(cudaStreamSynchronize(p->stream));
}

// aty (my column shard) = sum over ranks of A_g^T y   [world == 1: the whole vector]
static void full_aty(b200pdlp_problem* p, const double* y, double* aty) {
  if (p->world == 1) {
    launch_spmv_plain(p->stream, p->AT.dev, y, aty);
    p->launches++;
  } else {
    launch_spmv_partial_aty(p->stream, p->AT.dev, nullptr, y, y, p->part.p, p->at_outpos.p);
    p->launches++;
    if (p->p2p) {
      launch_p2p_exchange(p->stream, p->outs.p + 60, 0, p->peers, p->world, p->rank, p->epochs.p, p->fault.p);
      launch_reduce_part_p2p(p->stream, p->nl, aty, p->peers, p->world, p->rank, p->seg_len, 1);
      // (the peers' `part` buffers stay untouched until their next partial SpMV, which comes after a barrier that this
      //  rank only passes once it has finished reading)
      p->launches += 3;
    } else {
      reduce_scatter_part(p);
      CUDA_OK(cudaMemcpyAsync(aty, p->red.p, (size_t)p->nl * sizeof(double), cudaMemcpyDeviceToDevice, p->stream));
    }
  }
}
// ax (my rows) = A_g x, x given as my column shard   [world == 1: the whole vector]
static void full_ax(b200pdlp_problem* p, const double* x, double* ax) {
  if (p->world == 1) {
    launch_spmv_plain(p->stream, p->A.dev, x, ax);
  } else {
    if (p->p2p) {
      launch_push_shard(p->stream, x, p->nl, p->peers, p->world, p->rank, p->seg_len);
      launch_p2p_exchange(p->stream, p->outs.p + 60, 0, p->peers, p->world, p->rank, p->epochs.p, p->fault.p);
      p->launches += 2;
    } else {
      CUDA_OK(cudaMemcpyAsync(p->send.p, x, (size_t)p->nl * sizeof(double), cudaMemcpyDeviceToDevice, p->stream));
      gather_shards(p);
    }
    launch_spmv_plain(p->stream, p->A.dev, p->xfull.p, ax);
  }
  p->launches++;
}

struct CheckResult { Residuals it[2]; bool timed_out = false; };

// host arithmetic on the 29 scalars of the fused (tree-mode) residual sweeps, already in p->houts
static CheckResult parse_fused_check(b200pdlp_problem* p, bool timed_out_local) {
  const StdForm& f = p->form;
  CheckResult cr;
  cr.timed_out = p->world > 1 ? p->houts[28] > 0.0 : timed_out_local;
  for (int t = 0; t < 2; t++) {
    const double* a = p->houts + 10 * t;
    const double* r = p->houts + 20 + 4 * t;
    Residuals& R = cr.it[t];
    R.pobj = a[0] * f.sense + f.offset;
    R.pfeas = std::sqrt(r[1]);
    R.dobj = ((r[0] + a[1]) - a[2]) * f.sense + f.offset;
    R.dfeas = std::sqrt(a[3]);
    R.gap = R.pobj - R.dobj;
    R.relgap = std::fabs(R.pobj - R.dobj) / (1.0 + std::fabs(R.pobj) + std::fabs(R.dobj));
    double dscale = std::sqrt(r[2] + a[4] + a[5]);
    if (dscale < 1e-8) dscale = 1.0;
    double pscale = std::sqrt(a[6]);
    if (pscale < 1e-8) pscale = 1.0;
    R.pinf_obj = (R.dobj - f.offset) / f.sense / dscale;
    R.pinf_res = std::sqrt(a[7]) / dscale;
    R.dinf_obj = (R.pobj - f.offset) / f.sense / pscale;
    R.dinf_res = std::sqrt(r[3] + a[8] + a[9]) / pscale;
  }
  return cr;
}

// SPECULATIVE check: the same sequence as run_check's tree-mode branch, but enqueued right behind the PDHG passes
// BEFORE the host has read the state -- every kernel takes buffer parity, pending weight and step sum from the device
// state block and does nothing unless state.iter has reached state.stop_iter.  The host launch overhead of the ~10
// kernels hides behind the running pass graph, one synchronisation per check interval remains, and on several GPUs
// the barriers inside the check no longer wait for every rank's host thread.
static bool can_speculate_check(const b200pdlp_problem* p) { return !p->ordered && (p->world == 1 || p->p2p); }

static void enqueue_check_dev(b200pdlp_problem* p, bool timed_out_local) {
  cudaStream_t s = p->stream;
  PdhgState* st = p->state.p;
  const int n = p->nl, ml = p->ml;
  if (p->world > 1) {
    launch_reduce_part_p2p(s, n, p->aty[0].p, p->peers, p->world, p->rank, p->seg_len, 1, st, 1);   // if accepted_last
    p->launches++;
  }
  launch_average_dev(s, n, p->x[0].p, p->x[1].p, p->xsum.p, p->xavg.p, st);
  launch_average_dev(s, ml, p->y[0].p, p->y[1].p, p->ysum.p, p->yavg.p, st);
  launch_check_clear(s, st);
  p->launches += 3;
  if (p->world == 1) {
    launch_spmv_plain(s, p->A.dev, p->xavg.p, p->axavg.p, st);
    launch_spmv_plain(s, p->AT.dev, p->yavg.p, p->atyavg.p, st);
    p->launches += 2;
  } else {
    launch_push_shard(s, p->xavg.p, p->nl, p->peers, p->world, p->rank, p->seg_len, st);
    launch_spmv_partial_aty(s, p->AT.dev, nullptr, p->yavg.p, p->yavg.p, p->recv.p, p->at_outpos.p, st);
    launch_p2p_exchange(s, p->outs.p + 60, 0, p->peers, p->world, p->rank, p->epochs.p, p->fault.p, st);
    launch_spmv_plain(s, p->A.dev, p->xfull.p, p->axavg.p, st);
    launch_reduce_part_p2p(s, n, p->atyavg.p, p->peers, p->world, p->rank, p->seg_len, 2, st, 0);
    p->launches += 5;
  }
  double* o = p->outs.p;
  const bool one_aty = p->world > 1;   // multi-GPU keeps a single current A^T y shard
  ColIter c0{p->x[0].p, p->aty[0].p}, calt{p->x[1].p, one_aty ? p->aty[0].p : p->aty[1].p}, c1{p->xavg.p, p->atyavg.p};
  RowIter r0{p->y[0].p, p->ax[0].p}, ralt{p->y[1].p, p->ax[1].p}, r1{p->yavg.p, p->axavg.p};
  launch_col_check_fused(s, n, c0, c1, p->cost.p, p->lower.p, p->upper.p, p->colscale.p, p->rs(kSlotChk, n), o, st, calt);
  launch_row_check_fused(s, ml, r0, r1, p->rhs.p, p->rowscale.p, p->neq_local, p->rs(kSlotChk, ml), o + 20, st, ralt);
  p->launches += 2;
  if (p->world > 1) {
    p->hflag[0] = timed_out_local ? 1.0 : 0.0;
    CUDA_OK(cudaMemcpyAsync(o + 28, p->hflag, sizeof(double), cudaMemcpyHostToDevice, s));
    launch_p2p_exchange(s, o, 29, p->peers, p->world, p->rank, p->epochs.p, p->fault.p, st);
    p->launches++;
  }
  CUDA_OK(cudaMemcpyAsync(p->houts, o, 29 * sizeof(double), cudaMemcpyDeviceToHost, s));
}

// Ordered-mode check, host arithmetic on the sums of sweeps A (o[0..20]: 7 column sums, then 3 row sums, per iterate):
// residuals of both iterates and the ray scales sweeps B need
static void assemble_check_a(const StdForm& f, const double* o, CheckResult& cr, double dscale[2], double pscale[2]) {
  for (int t = 0; t < 2; t++) {
    const double* a = o + 7 * t;
    const double* r = o + 14 + 3 * t;
    Residuals& R = cr.it[t];
    R.pobj = a[0] * f.sense + f.offset;                        // cupdlp_solver.c:24
    R.pfeas = std::sqrt(r[1]);
    double d = r[0];                                           // :79
    d += a[1];                                                 // :92 / :164
    d -= a[2];                                                 // :98 / :180
    R.dobj = d * f.sense + f.offset;                           // :100 / :182
    R.dfeas = std::sqrt(a[3]);
    R.gap = R.pobj - R.dobj;                                   // :513-516
    R.relgap = std::fabs(R.pobj - R.dobj) / (1.0 + std::fabs(R.pobj) + std::fabs(R.dobj));
    dscale[t] = std::sqrt(r[2] + a[4] + a[5]);                 // :262-266
    if (dscale[t] < 1e-8) dscale[t] = 1.0;
    pscale[t] = std::sqrt(a[6]);                               // :367-371
    if (pscale[t] < 1e-8) pscale[t] = 1.0;
  }
}

// ... and on the sums of sweeps B (o[24..29]: 3 column sums per iterate, o[30..31]: 1 row sum per iterate): the ray residuals
static void assemble_check_b(const StdForm& f, const double* o, CheckResult& cr, const double dscale[2], const double pscale[2]) {
  for (int t = 0; t < 2; t++) {
    Residuals& R = cr.it[t];
    const double* b = o + 24 + 3 * t;
    R.pinf_obj = (R.dobj - f.offset) / f.sense / dscale[t];    // :282-283
    R.pinf_res = std::sqrt(b[0]);
    R.dinf_obj = (R.pobj - f.offset) / f.sense / pscale[t];    // :376-377
    R.dinf_res = std::sqrt(o[30 + t] + b[1] + b[2]);           // :425
  }
}

// PDHG_Compute_Average_Iterate + PDHG_Compute_Residuals + PDHG_Compute_Infeas_Residuals
// (cupdlp_step.c:377-420, cupdlp_solver.c:473-529, :433-471) for current and average iterate
static CheckResult run_check(b200pdlp_problem* p, bool timed_out_local) {
  NvtxRange nvtx("b200pdlp: check iteration (host-driven)");
  cudaStream_t s = p->stream;
  PdhgState* h = p->hstate;
  const StdForm& f = p->form;
  const int n = p->nl, ml = p->ml, cur = h->cur;   // n = column entries held by this rank
  const int acur = p->world == 1 ? cur : 0;        // multi-GPU keeps one current A^T y shard
  const double scale = h->sum_step > 0.0 ? 1.0 / h->sum_step : 1.0;
  const bool fused = p->world > 1 && p->p2p;
  if (p->world > 1 && h->accepted_last) {
    // the last accepted pass left its A^T y' un-reduced (P2P) / in the reduce-scatter buffer (NCCL): make it current
    if (p->p2p) {
      launch_reduce_part_p2p(s, n, p->aty[0].p, p->peers, p->world, p->rank, p->seg_len, 1);
      p->launches++;
    } else {
      CUDA_OK(cudaMemcpyAsync(p->aty[0].p, p->red.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s));
    }
    h->accepted_last = 0;
    push_state(p);
  }
  launch_average(s, n, p->x[cur].p, p->xsum.p, p->xavg.p, h->pending, h->w_pending, scale);
  launch_average(s, ml, p->y[cur].p, p->ysum.p, p->yavg.p, h->pending, h->w_pending, scale);
  p->launches += 2;
  if (h->pending) { h->pending = 0; push_state(p); }
  if (fused) {
    // one barrier for both exchanges: x-bar shards are stored into every peer's xfull, the partial A_g^T y-bar is
    // parked in my `recv` buffer (so `part`, which a slower peer may still be reducing from, stays intact)
    launch_push_shard(s, p->xavg.p, p->nl, p->peers, p->world, p->rank, p->seg_len);
    launch_spmv_partial_aty(s, p->AT.dev, nullptr, p->yavg.p, p->yavg.p, p->recv.p, p->at_outpos.p);
    launch_p2p_exchange(s, p->outs.p + 60, 0, p->peers, p->world, p->rank, p->epochs.p, p->fault.p);
    launch_spmv_plain(s, p->A.dev, p->xfull.p, p->axavg.p);
    launch_reduce_part_p2p(s, n, p->atyavg.p, p->peers, p->world, p->rank, p->seg_len, 2);
    p->launches += 5;
  } else {
    full_ax(p, p->xavg.p, p->axavg.p);
    full_aty(p, p->yavg.p, p->atyavg.p);
  }
  ColIter c0{p->x[cur].p, p->aty[acur].p}, c1{p->xavg.p, p->atyavg.p};
  RowIter r0{p->y[cur].p, p->ax[cur].p}, r1{p->yavg.p, p->axavg.p};
  double* o = p->outs.p;
  if (!p->ordered) {
    // tree mode: one fused sweep per side, one read-back, one all-reduce (see col_check_fused_kernel)
    launch_col_check_fused(s, n, c0, c1, p->cost.p, p->lower.p, p->upper.p, p->colscale.p, p->rs(kSlotChk, n), o);
    launch_row_check_fused(s, ml, r0, r1, p->rhs.p, p->rowscale.p, p->neq_local, p->rs(kSlotChk, ml), o + 20);
    p->launches += 2;
    if (p->world > 1) {
      double flag = timed_out_local ? 1.0 : 0.0;
      CUDA_OK(cudaMemcpyAsync(o + 28, &flag, sizeof(double), cudaMemcpyHostToDevice, s));
      allreduce_small(p, o, 29);
    }
    pull_outs(p, 29);
    CheckResult cr = parse_fused_check(p, timed_out_local);
    return cr;
  }
  launch_col_check_a(s, n, 2, c0, c1, p->cost.p, p->lower.p, p->upper.p, p->colscale.p, p->rs(kSlotChk, n), o);
  launch_row_check_a(s, ml, 2, r0, r1, p->rhs.p, p->rowscale.p, p->neq_local, 0, p->rs(kSlotChk, ml), o + 14);
  p->launches += 2;
  if (p->world > 1) {
    // column-shard and row-block partial sums + the time-limit flag travel in one small all-reduce
    double flag = timed_out_local ? 1.0 : 0.0;
    CUDA_OK(cudaMemcpyAsync(o + 20, &flag, sizeof(double), cudaMemcpyHostToDevice, s));
    allreduce_inplace(p, o, 21);
  }
  pull_outs(p, 21);
  CheckResult cr;
  cr.timed_out = p->world > 1 ? p->houts[20] > 0.0 : timed_out_local;
  double inv_d[2], inv_p[2], dscale[2], pscale[2];
  assemble_check_a(f, p->houts, cr, dscale, pscale);
  for (int t = 0; t < 2; t++) {
    inv_d[t] = 1 / dscale[t];
    inv_p[t] = 1.0 / pscale[t];
  }
  launch_col_check_b(s, n, 2, c0, c1, inv_d, inv_p, p->cost.p, p->lower.p, p->upper.p, p->colscale.p,
                     p->rs(kSlotChk, n), o + 24);
  launch_row_check_b(s, ml, 2, r0, r1, inv_p, p->rowscale.p, p->neq_local, 0, p->rs(kSlotChk, ml), o + 30);
  p->launches += 2;
  if (p->world > 1) allreduce_inplace(p, o + 24, 8);
  CUDA_OK(cudaMemcpyAsync(p->houts + 24, o + 24, 8 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  assemble_check_b(f, p->houts, cr, dscale, pscale);
  return cr;
}

static double restart_score(double beta, double pf, double df, double gap) {  // cupdlp_restart.c:113-124
  return std::sqrt(beta * pf * pf + df * df / beta + gap * gap);
}

struct RestartMemo { double pf_lr = 0, df_lr = 0, gap_lr = 0, pf_lc = 0, df_lc = 0, gap_lc = 0; int last_iter = 0; };

// PDHG_Check_Restart_GPU (cupdlp_restart.c:3-99): 0 none, 1 to average, 2 to current
static int decide_restart(const PdhgState* h, const CheckResult& c, RestartMemo& mm) {
  const Residuals &L = c.it[0], &A = c.it[1];
  if (h->iter == mm.last_iter) {
    mm.pf_lr = L.pfeas; mm.df_lr = L.dfeas; mm.gap_lr = L.gap;
    mm.pf_lc = L.pfeas; mm.df_lc = L.dfeas; mm.gap_lc = L.gap;
    return 0;
  }
  const double mu_cur = restart_score(h->beta, L.pfeas, L.dfeas, L.gap);
  const double mu_avg = restart_score(h->beta, A.pfeas, A.dfeas, A.gap);
  int choice = mu_cur < mu_avg ? 2 : 1;
  const double mu_cand = mu_cur < mu_avg ? mu_cur : mu_avg;
  if ((h->iter - mm.last_iter) >= 0.36 * h->iter) {
    // artificial restart
  } else {
    const double mu_lr = restart_score(h->beta, mm.pf_lr, mm.df_lr, mm.gap_lr);
    if (!(mu_cand < 0.2 * mu_lr)) {
      const double mu_lc = restart_score(h->beta, mm.pf_lc, mm.df_lc, mm.gap_lc);
      if (!(mu_cand < 0.8 * mu_lr && mu_cand > mu_lc)) choice = 0;
    }
  }
  const Residuals& C = mu_cur < mu_avg ? L : A;
  mm.pf_lc = C.pfeas; mm.df_lc = C.dfeas; mm.gap_lc = C.gap;
  return choice;
}

// the host part of a restart, given |x - x_lr|^2 and |y - y_lr|^2 of the iterate restarted to: the memo, the step sum, and
// beta / tau / sigma (glibc log / exp, which the device's do not reproduce)
static void restart_steps(PdhgState* h, int choice, const CheckResult& c, RestartMemo& mm, double dx2, double dy2) {
  h->sum_step = 0.0;
  const Residuals& R = choice == 1 ? c.it[1] : c.it[0];
  mm.pf_lr = R.pfeas; mm.df_lr = R.dfeas; mm.gap_lr = R.gap;
  const double mean = std::sqrt(h->tau * h->sigma);
  const double dxn = std::sqrt(dx2), dyn = std::sqrt(dy2);
  if (std::fmin(dxn, dyn) > 1e-10) {
    const double upd = dyn / dxn;
    const double lg = 0.5 * std::log(upd) + 0.5 * std::log(std::sqrt(h->beta));
    h->beta = std::exp(lg) * std::exp(lg);
  }
  h->tau = mean / std::sqrt(h->beta);
  h->sigma = h->tau * h->beta;
  mm.last_iter = h->iter;
}

// PDHG_Restart_Iterate_GPU (cupdlp_proj.c:88-148) + PDHG_Compute_Step_Size_Ratio (cupdlp_step.c:147-176)
static void do_restart(b200pdlp_problem* p, int choice, const CheckResult& c, RestartMemo& mm) {
  NvtxRange nvtx("b200pdlp: restart");
  cudaStream_t s = p->stream;
  PdhgState* h = p->hstate;
  const int n = p->nl, ml = p->ml, cur = h->cur;
  const int acur = p->world == 1 ? cur : 0;
  CUDA_OK(cudaMemsetAsync(p->xsum.p, 0, (size_t)n * sizeof(double), s));
  CUDA_OK(cudaMemsetAsync(p->ysum.p, 0, (size_t)std::max(ml, 1) * sizeof(double), s));
  if (choice == 1) {
    CUDA_OK(cudaMemcpyAsync(p->x[cur].p, p->xavg.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s));
    CUDA_OK(cudaMemcpyAsync(p->y[cur].p, p->yavg.p, (size_t)ml * sizeof(double), cudaMemcpyDeviceToDevice, s));
    CUDA_OK(cudaMemcpyAsync(p->ax[cur].p, p->axavg.p, (size_t)ml * sizeof(double), cudaMemcpyDeviceToDevice, s));
    CUDA_OK(cudaMemcpyAsync(p->aty[acur].p, p->atyavg.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s));
  }
  double* o = p->outs.p + 40;
  launch_diff_norm2(s, n, p->x[cur].p, p->xlr.p, p->rs(kSlotChk, n), o);
  launch_diff_norm2(s, ml, p->y[cur].p, p->ylr.p, p->rs(kSlotChk, ml), o + 1);
  p->launches += 2;
  if (p->world > 1) allreduce_small(p, o, 2);
  CUDA_OK(cudaMemcpyAsync(p->houts + 40, o, 2 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaMemcpyAsync(p->xlr.p, p->x[cur].p, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s));
  CUDA_OK(cudaMemcpyAsync(p->ylr.p, p->y[cur].p, (size_t)ml * sizeof(double), cudaMemcpyDeviceToDevice, s));
  CUDA_OK(cudaStreamSynchronize(s));
  restart_steps(h, choice, c, mm, p->houts[40], p->houts[41]);
}

// state for the next pass after the host touched tau/sigma/beta (start of
// PDHG_Update_Iterate_Adaptive_Step_Size, cupdlp_step.c:230-242)
static void arm_step(PdhgState* h) {
  h->eta = std::sqrt(h->tau * h->sigma);
  if (h->adaptive) {
    h->tau_try = h->eta / std::sqrt(h->beta);
    h->sigma_try = h->eta * std::sqrt(h->beta);
  } else {
    h->tau_try = h->tau;
    h->sigma_try = h->sigma;
  }
}

static double vec_norm2_sq(b200pdlp_problem* p, const double* v, int len, bool reduce_over_ranks) {
  double* o = p->outs.p + 44;
  launch_diff_norm2(p->stream, len, v, nullptr, p->rs(kSlotChk, len), o);
  p->launches++;
  if (reduce_over_ranks && p->world > 1) allreduce_inplace(p, o, 1);
  CUDA_OK(cudaMemcpyAsync(p->houts + 44, o, sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  CUDA_OK(cudaStreamSynchronize(p->stream));
  return p->houts[44];
}

// PDHG_Power_Method (cupdlp_step.c:71-145): 20 iterations on A A'
static double power_method(b200pdlp_problem* p) {
  if (p->world > 1) throw Error(B200PDLP_ERR_ARG, "fixed-step mode (adaptive_step = 0) is single-GPU only");
  cudaStream_t s = p->stream;
  double* q = p->ylr.p;  // scratch (re-zeroed by the caller)
  launch_fill(s, p->ml, q, 1.0);
  p->launches++;
  double lambda = 0.0;
  for (int it = 0; it < 20; it++) {
    full_aty(p, q, p->aty[0].p);
    launch_spmv_plain(s, p->A.dev, p->aty[0].p, p->ax[0].p);
    p->launches++;
    CUDA_OK(cudaMemcpyAsync(q, p->ax[0].p, (size_t)p->ml * sizeof(double), cudaMemcpyDeviceToDevice, s));
    const double qn = std::sqrt(vec_norm2_sq(p, q, p->ml, true));
    launch_scale(s, p->ml, q, 1.0 / qn);
    p->launches++;
    full_aty(p, q, p->aty[0].p);
    lambda = vec_norm2_sq(p, p->aty[0].p, p->n, false);
  }
  return lambda;
}

// What a check decides (cupdlp_solver.c:939-1106): a termination code, or -1 to go on (then *choice = the restart decided,
// 0 none, 1 to the average, 2 to the current iterate).  chk.timed_out: the time limit had passed when the check began.
static int check_decision(const b200pdlp_params& prm, double tol_p, double tol_d, const PdhgState* h, const CheckResult& chk,
                          RestartMemo& memo, int* term_iterate, int* choice) {
  const Residuals &L = chk.it[0], &A = chk.it[1];
  *choice = 0;
  if (L.pfeas < tol_p && L.dfeas < tol_d && L.relgap < prm.tol_gap) { *term_iterate = 0; return B200PDLP_OPTIMAL; }
  if (A.pfeas < tol_p && A.dfeas < tol_d && A.relgap < prm.tol_gap) { *term_iterate = 1; return B200PDLP_OPTIMAL; }
  {  // PDHG_Check_Infeasibility, cupdlp_solver.c:740-795 (dFeasTol = 1e-8, cupdlp_utils.c:889)
    const double ft = 1e-8;
    bool inf = false;
    for (int t = 0; t < 2; t++) {
      const Residuals& R = chk.it[t];
      if (R.pinf_obj > 0.0 && R.pinf_res < ft * R.pinf_obj) inf = true;
      if (R.dinf_obj < 0.0 && R.dinf_res < -ft * R.dinf_obj) inf = true;
    }
    if (inf) return B200PDLP_INFEASIBLE_OR_UNBOUNDED;
  }
  if (chk.timed_out) return B200PDLP_TIMELIMIT_OR_ITERLIMIT;
  if (h->iter >= prm.iter_limit - 1) return B200PDLP_TIMELIMIT_OR_ITERLIMIT;
  if (prm.restart) *choice = decide_restart(h, chk, memo);
  return -1;
}

// the next check iteration: < 10, multiple of the interval, or iter_limit - 1 (cupdlp_solver.c:953-962)
static int next_check_iter(int iter, int interval, int iter_limit) {
  int next = iter + 1;
  while (!(next < 10 || next % interval == 0 || next == iter_limit - 1)) next++;
  return next;
}

// PDHG_PreSolve's hot start (cupdlp_solver.c:1217-1279) + PDHG_Project_Bounds in standard-form order: x0[n], y0[m] (zero
// without a complete hot start)
static void host_start_point(const StdForm& f, const b200pdlp_warm* warm, std::vector<double>& x0, std::vector<double>& y0) {
  const int n = f.n, m = f.m;
  x0.assign(n, 0.0);
  y0.assign(m, 0.0);
  if (warm && warm->col_value && warm->row_value && warm->row_dual) {
    int jc = 0;
    for (; jc < f.n_orig; jc++) x0[jc] = warm->col_value[jc];
    for (int i = 0; i < m; i++) {
      const double mu = f.row_class[i] == kLeq ? -1 : 1;
      y0[f.row_new_idx[i]] = f.sense * mu * warm->row_dual[i];
      if (f.row_class[i] == kBound) x0[jc++] = warm->row_value[i];
    }
    for (int j = 0; j < n; j++) x0[j] *= f.col_scale[j];
    for (int i = 0; i < m; i++) y0[i] *= f.row_scale[i];
  }
  for (int j = 0; j < n; j++) {  // PDHG_Project_Bounds: upper first, then lower
    double v = x0[j];
    v = v < f.upper[j] ? v : f.upper[j];
    v = v > f.lower[j] ? v : f.lower[j];
    x0[j] = v;
  }
}

// proj(0) of column j: where xSum starts (PDHG_Init_Variables, cupdlp_solver.c:577-583)
static double proj_zero(const StdForm& f, int j) {
  double v = 0.0;
  v = v < f.upper[j] ? v : f.upper[j];
  v = v > f.lower[j] ? v : f.lower[j];
  return v;
}

// PDHG_PostSolve (cupdlp_solver.c:1281-1435) on the host: x, y, A x, A'y of the returned iterate in standard-form order ->
// the four HighsSolution vectors in `out` (scaled in place)
static void host_postsolve(const StdForm& f, bool have_check, std::vector<double>& hx, std::vector<double>& hy,
                           std::vector<double>& hax, const std::vector<double>& haty, b200pdlp_result* out) {
  const int n = f.n, m = f.m;
  const double inf = std::numeric_limits<double>::infinity();
  if (!(out->col_value && out->col_dual && out->row_value && out->row_dual)) return;
  std::vector<double> sp(n, 0.0), sn(n, 0.0);
  if (have_check) {
    for (int j = 0; j < n; j++) {   // dSlackPos / dSlackNeg of the returned iterate (cupdlp_solver.c:150-176)
      double rc = haty[j] * -1.0;
      rc = rc + 1.0 * f.cost[j];
      double a = rc > 0.0 ? rc : 0.0;
      a = a * (f.lower[j] > -inf ? 1.0 : 0.0);
      double b = rc < 0.0 ? rc : 0.0;
      b = b * -1.0;
      b = b * (f.upper[j] < inf ? 1.0 : 0.0);
      sp[j] = a; sn[j] = b;
    }
  }
  for (int j = 0; j < n; j++) { hx[j] /= f.col_scale[j]; sp[j] *= f.col_scale[j]; sn[j] *= f.col_scale[j]; }
  for (int i = 0; i < m; i++) { hy[i] /= f.row_scale[i]; hax[i] *= f.row_scale[i]; }
  for (int j = 0; j < f.n_orig; j++) out->col_value[j] = hx[j];
  for (int i = 0, j = 0; i < m; i++) {
    double v = hax[f.row_new_idx[i]];
    if (f.row_class[i] == kLeq) v = -v;
    else if (f.row_class[i] == kBound) { v = v + hx[f.n_orig + j]; j++; }
    out->row_value[i] = v;
  }
  for (int j = 0; j < f.n_orig; j++) { double v = sp[j] - sn[j]; out->col_dual[j] = v * f.sense; }
  for (int i = 0; i < m; i++) {
    double v = hy[f.row_new_idx[i]] * f.sense;
    if (f.row_class[i] == kLeq) v = -v;
    out->row_dual[i] = v;
  }
}

// the per-solve fields of a result (the timings and kernel_launches are the caller's)
static void fill_result(b200pdlp_result* out, const StdForm& f, const PdhgState* h, int term, int term_iterate, int restarts,
                        const CheckResult& chk) {
  out->value_valid = 1; out->dual_valid = 1;
  out->term_code = term; out->term_iterate = term_iterate;
  out->iters = h->iter; out->passes = h->passes; out->restarts = restarts;
  const Residuals& R = chk.it[(term == B200PDLP_OPTIMAL && term_iterate == 1) ? 1 : 0];
  out->primal_obj = R.pobj; out->dual_obj = R.dobj; out->primal_feas = R.pfeas; out->dual_feas = R.dfeas;
  out->gap = R.gap; out->rel_gap = R.relgap;
  out->form_cols = f.n; out->form_rows = f.m; out->form_nnz = f.nnz; out->form_neq = f.neq;
}

static void trace_row(b200pdlp_result* out, const PdhgState* h, const CheckResult& c, int restart) {
  if (!out->trace || out->trace_len >= out->trace_cap) return;
  double* t = out->trace + (size_t)out->trace_len * B200PDLP_TRACE_COLS;
  // after a restart to the average the reference re-evaluates the residuals of the (new) current
  // iterate (cupdlp_proj.c:145), which are those of the average it was copied from
  const Residuals &L = restart == 1 ? c.it[1] : c.it[0], &A = c.it[1];
  t[0] = h->iter; t[1] = L.pobj; t[2] = L.dobj; t[3] = L.pfeas; t[4] = L.dfeas;
  t[5] = A.pobj; t[6] = A.dobj; t[7] = A.pfeas; t[8] = A.dfeas;
  t[9] = h->tau; t[10] = h->sigma; t[11] = h->beta; t[12] = restart; t[13] = h->step_iter;
  t[14] = h->sum_step; t[15] = 0;
  out->trace_len++;
}

// ---------------------------------------------------------------- device-side check iterations (tree mode, one GPU)
// graphs bake pointers and launch shapes in: (re)wiring the peers invalidates all of them
static void drop_graphs(b200pdlp_problem* p) {
  if (p->graph_main) { cudaGraphExecDestroy(p->graph_main); p->graph_main = nullptr; }
  if (p->graph_small) { cudaGraphExecDestroy(p->graph_small); p->graph_small = nullptr; }
  for (cudaGraphExec_t& g : p->graph_pow2) if (g) { cudaGraphExecDestroy(g); g = nullptr; }
  if (p->graph_check) { cudaGraphExecDestroy(p->graph_check); p->graph_check = nullptr; }
  if (p->graph_check_light) { cudaGraphExecDestroy(p->graph_check_light); p->graph_check_light = nullptr; }
}

static bool use_device_checks(const b200pdlp_problem* p, const b200pdlp_params& prm) {
  if (p->ordered || prm.log_level >= 2 || prm.iter_limit <= 0) return false;
  if (p->world != 1) {
    // several GPUs: only on the fused peer-memory path (the checks' collectives are our own barrier / exchange kernels)
    if (!p->p2p) return false;
    // default since it passed on hardware against the oracle (2 GPUs: tests/test_gpu_multi.py; 2 / 3 / 4 logical shards:
    // tests/test_gpu_logical_shards.py; both run both settings).  B200PDLP_MG_DEVICE_CHECK=0: round 1's host-driven checks.
    const char* e = getenv("B200PDLP_MG_DEVICE_CHECK");
    if (e && atoi(e) == 0) return false;
  }
  if (const char* e = getenv("B200PDLP_HOST_CHECK")) if (atoi(e) != 0) return false;   // the round-1 host-driven checks
  return true;
}

// several GPUs (fused peer-memory path): the same check with the vectors sharded -- xbar shards go to every peer's xfull,
// the partial A_g'ybar are parked in `recv` and reduced by their owners after a barrier, the 28 sums (+ the time-limit
// word) are all-reduced by the exchange kernel (identical on every rank, added in rank order), so every rank takes the
// same decisions; a restart costs one more exchange of two scalars.  15 launches, 3 cross-GPU synchronisations.
static int enqueue_check_device_mg(b200pdlp_problem* p, bool light) {
  cudaStream_t s = p->stream;
  PdhgState* st = p->state.p;
  SolveCtl* ctl = p->ctl.p;
  const int nl = p->nl, ml = p->ml;
  double* o = p->outs.p;
  const ReduceScratch rrow = p->rs(kSlotK2, ml), rcol = p->rs(kSlotChk, nl), rrst = p->rs(kSlotK1, nl);
  int launches = 0;
  launch_reduce_part_p2p(s, nl, p->aty[0].p, p->peers, p->world, p->rank, p->seg_len, 1, st, 1);   // if the last pass was accepted
  if (light) {
    // dense-check phase: the passes carried A_g xSum (my rows) and my shard of A'ySum -- no all-gather of xbar, no partial
    // A_g'ybar, no reduce: two sweeps over my shard / my rows, then the same exchange of the 28 sums (+ time-limit word)
    launch_check_cols_sweep(s, false, nl, p->x[0].p, p->x[1].p, p->aty[0].p, p->aty[0].p, p->xsum.p, p->atysum.p, p->xavg.p,
                            p->atyavg.p, p->cost.p, p->lower.p, p->upper.p, p->colscale.p, st, ctl, rcol);
    launch_check_rows_sweep(s, false, ml, p->neq_local, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->ysum.p, p->axsum.p,
                            p->yavg.p, p->axavg.p, p->rhs.p, p->rowscale.p, st, ctl, rrow);
    launch_reduce_partials(s, st, ctl, 20, rcol.partials, check_light_grid(nl, true), o, /*flag_slot=*/8, 0,    // o[0..19]
                           8, rrow.partials, check_light_grid(ml, false), o + 20);                             // o[20..27], flag at o[28]
    launches = 4;
  } else {
    launch_check_light_off(s, st, ctl);
    launch_check_avg_x(s, nl, p->x[0].p, p->x[1].p, p->xsum.p, p->xavg.p, st, ctl);
    launch_average_dev(s, ml, p->y[0].p, p->y[1].p, p->ysum.p, p->yavg.p, st);
    launch_push_shard(s, p->xavg.p, nl, p->peers, p->world, p->rank, p->seg_len, st);
    launch_spmv_partial_aty(s, p->AT.dev, nullptr, p->yavg.p, p->yavg.p, p->recv.p, p->at_outpos.p, st);
    launch_p2p_exchange(s, o + 60, 0, p->peers, p->world, p->rank, p->epochs.p, p->fault.p, st);
    launch_spmv_check_rows_mg(s, p->A.dev, st, ctl, p->xfull.p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->yavg.p,
                              p->axavg.p, p->rhs.p, p->rowscale.p, p->neq_local, rrow);
    launch_reduce_part_p2p(s, nl, p->atyavg.p, p->peers, p->world, p->rank, p->seg_len, 2, st, 0);
    ColIter c0{p->x[0].p, p->aty[0].p}, calt{p->x[1].p, p->aty[0].p}, c1{p->xavg.p, p->atyavg.p};   // one current A'y shard
    launch_col_check_fused(s, nl, c0, c1, p->cost.p, p->lower.p, p->upper.p, p->colscale.p, rcol, o, st, calt);
    launch_reduce_partials(s, st, ctl, 8, rrow.partials, p->A.grid(), o + 20, /*flag_slot=*/8, 0);   // o[20..27], flag at o[28]
    launches = 11;
  }
  launch_p2p_exchange(s, o, 29, p->peers, p->world, p->rank, p->epochs.p, p->fault.p, st);
  launch_check_decide_sums(s, st, ctl, o);
  launch_restart_sweep(s, nl, ml, p->x[0].p, p->x[1].p, p->aty[0].p, p->aty[0].p, p->xavg.p, p->atyavg.p, p->xsum.p, p->xlr.p,
                       p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->yavg.p, p->axavg.p, p->ysum.p, p->ylr.p, st, ctl, rrst,
                       p->atysum.p, p->axsum.p);
  launch_reduce_partials(s, st, ctl, 2, rrst.partials, restart_sweep_grid(nl, ml), o + 40, -1, 1);
  launch_p2p_exchange(s, o + 40, 2, p->peers, p->world, p->rank, p->epochs.p, p->fault.p, st, ctl);   // only on a restart
  launch_check_finish(s, st, ctl, rrst.partials, restart_sweep_grid(nl, ml), o + 40);
  return launches + 6;
}

// run `a` on the problem's stream and `b` next to it on the side stream (graph capture turns this into two branches)
static void ensure_side_stream(b200pdlp_problem* p) {   // at problem creation: never inside a stream capture
  if (p->side_stream) return;
  CUDA_OK(cudaStreamCreateWithFlags(&p->side_stream, cudaStreamNonBlocking));
  CUDA_OK(cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming));
  CUDA_OK(cudaEventCreateWithFlags(&p->ev_join, cudaEventDisableTiming));
}
template <class FA, class FB>
static void run_side_by_side(b200pdlp_problem* p, FA&& a, FB&& b) {
  if (!p->side_stream) { a(p->stream); b(p->stream); return; }
  CUDA_OK(cudaEventRecord(p->ev_fork, p->stream));
  CUDA_OK(cudaStreamWaitEvent(p->side_stream, p->ev_fork, 0));
  b(p->side_stream);
  CUDA_OK(cudaEventRecord(p->ev_join, p->side_stream));
  a(p->stream);
  CUDA_OK(cudaStreamWaitEvent(p->stream, p->ev_join, 0));
}

// the eight launches of one check (pdhg_kernels.cu "device-side check iteration"); no-ops unless the check is due.
// light: the dense-check phase's variant (five launches: the two sweeps use the carried A xSum / A'ySum, no C1 / C2)
static int enqueue_check_device(b200pdlp_problem* p, bool light = false) {
  if (p->world > 1) return enqueue_check_device_mg(p, light);
  cudaStream_t s = p->stream;
  PdhgState* st = p->state.p;
  SolveCtl* ctl = p->ctl.p;
  const int n = p->n, ml = p->ml;
  const ReduceScratch rrow = p->rs(kSlotChk, ml), rcol = p->rs(kSlotK3, n), rrst = p->rs(kSlotK1, n);
  const bool given = !light;
  auto sweeps = [&]() {
    run_side_by_side(p,
        [&](cudaStream_t q) {
          launch_check_cols_sweep(q, given, n, p->x[0].p, p->x[1].p, p->aty[0].p, p->aty[1].p, p->xsum.p, p->atysum.p, p->xavg.p,
                                  p->atyavg.p, p->cost.p, p->lower.p, p->upper.p, p->colscale.p, st, ctl, rcol);
        },
        [&](cudaStream_t q) {
          launch_check_rows_sweep(q, given, ml, p->neq_local, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->ysum.p, p->axsum.p,
                                  p->yavg.p, p->axavg.p, p->rhs.p, p->rowscale.p, st, ctl, rrow);
        });
  };
  if (!light) {
    // split check: averages, two plain SpMV (as fast as the pass kernels), two vector sweeps for the 20 + 8 sums
    launch_check_avg_xy(s, n, ml, p->x[0].p, p->x[1].p, p->xsum.p, p->xavg.p, p->y[0].p, p->y[1].p, p->ysum.p, p->yavg.p, st, ctl);
    run_side_by_side(p, [&](cudaStream_t q) { launch_spmv_plain(q, p->A.dev, p->xavg.p, p->axavg.p, st); },
                     [&](cudaStream_t q) { launch_spmv_plain(q, p->AT.dev, p->yavg.p, p->atyavg.p, st); });
  }
  sweeps();
  launch_check_decide(s, st, ctl, rrow.partials, check_light_grid(ml, false), rcol.partials, check_light_grid(n, true), rrow.counter);
  launch_restart_sweep(s, n, ml, p->x[0].p, p->x[1].p, p->aty[0].p, p->aty[1].p, p->xavg.p, p->atyavg.p, p->xsum.p,
                       p->xlr.p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->yavg.p, p->axavg.p, p->ysum.p, p->ylr.p,
                       st, ctl, rrst, p->atysum.p, p->axsum.p);
  launch_check_finish(s, st, ctl, rrst.partials, restart_sweep_grid(n, ml));
  return light ? 5 : 8;
}

static cudaGraphExec_t capture_check(b200pdlp_problem* p, bool light, int* launches) {
  cudaGraph_t g = nullptr;
  cudaGraphExec_t ge = nullptr;
  CUDA_OK(cudaStreamBeginCapture(p->stream, cudaStreamCaptureModeThreadLocal));
  *launches = enqueue_check_device(p, light);
  CUDA_OK(cudaStreamEndCapture(p->stream, &g));
  CUDA_OK(cudaGraphInstantiate(&ge, g, 0));
  CUDA_OK(cudaGraphDestroy(g));
  return ge;
}

static void launch_check_graph(b200pdlp_problem* p, bool light = false) {
  if (p->no_graph) { p->launches += enqueue_check_device(p, light); return; }
  cudaGraphExec_t& ge = light ? p->graph_check_light : p->graph_check;
  int& nl = p->check_launches[light ? 1 : 0];
  if (!ge) ge = capture_check(p, light, &nl);
  CUDA_OK(cudaGraphLaunch(ge, p->stream));
  p->launches += nl;
}

// `d` PDHG passes: the main graph (one check interval + spare passes) when d is about an interval, otherwise graphs of
// 32/16/8/4 passes and single passes.  Kernels beyond the check iteration are no-ops.
static void enqueue_passes_device(b200pdlp_problem* p, int d) {
  if (d <= 0) return;
  const int kp = p->kernels_per_pass;
  if (p->no_graph) { for (; d > 0; d--) { enqueue_pass(p); p->launches += kp; } return; }
  if (d > p->graph_main_passes - 12 && !p->graph_main) p->graph_main = capture_passes(p, p->graph_main_passes);
  if (d > p->graph_main_passes - 12 && d <= p->graph_main_passes) {
    CUDA_OK(cudaGraphLaunch(p->graph_main, p->stream));
    p->launches += (long long)p->graph_main_passes * kp;
    return;
  }
  while (d > p->graph_main_passes) {
    CUDA_OK(cudaGraphLaunch(p->graph_main, p->stream));
    p->launches += (long long)p->graph_main_passes * kp;
    d -= p->graph_main_passes;
  }
  for (int k = 5; k >= 2; k--) {
    while (d >= (1 << k)) {
      if (!p->graph_pow2[k]) p->graph_pow2[k] = capture_passes(p, 1 << k);
      CUDA_OK(cudaGraphLaunch(p->graph_pow2[k], p->stream));
      p->launches += (long long)(1 << k) * kp;
      d -= 1 << k;
    }
  }
  for (; d > 0; d--) { enqueue_pass(p); p->launches += kp; }
}

static void solve_on_device(b200pdlp_problem* p, const b200pdlp_params& prm, const b200pdlp_warm* warm, b200pdlp_result* out) {
  NvtxRange nvtx("b200pdlp: solve");
  nvtxRangePushA("b200pdlp: initial point + graphs");
  using clk = std::chrono::steady_clock;
  set_device(p);
  const auto t_begin = clk::now();
  const StdForm& f = p->form;
  cudaStream_t s = p->stream;
  const int n = p->n, m = p->m, ml = p->ml;
  const int interval = prm.check_interval > 0 ? prm.check_interval : 40;
  const double t_lim = (prm.time_limit >= 0 && std::isfinite(prm.time_limit)) ? prm.time_limit : -1.0;   // < 0: none
  const long long launches0 = p->launches;
  PdhgState* h = p->hstate;
  memset(h, 0, sizeof(PdhgState));
  h->adaptive = prm.adaptive_step != 0;
  out->trace_len = 0;
  Laps lap;
  lap.rank = p->world > 1 ? p->rank : -1;
  if (p->local_link && p->group) {
    // logical shards: everything that allocates or instantiates happens before ANY rank launches a kernel that waits for
    // its peers (see LocalGroup)
    const int interval0 = prm.check_interval > 0 ? prm.check_interval : 40;
    const int want0 = std::min(prm.graph_passes > 0 ? prm.graph_passes : interval0 + 4, kPowTab - 16);
    p->kernels_per_pass = p->p2p ? 5 : 6;
    if (p->graph_main && p->graph_main_passes != want0) { cudaGraphExecDestroy(p->graph_main); p->graph_main = nullptr; }
    p->graph_main_passes = want0;
    if (!getenv("B200PDLP_NO_GRAPH")) {
      if (!p->graph_main) p->graph_main = capture_passes(p, want0);
      if (!p->graph_small) { p->graph_small_passes = 4; p->graph_small = capture_passes(p, 4); }
      CUDA_OK(cudaGraphUpload(p->graph_main, s));
      CUDA_OK(cudaGraphUpload(p->graph_small, s));
      if (use_device_checks(p, prm)) {
        if (!p->hctl) {
          p->hctl = static_cast<SolveCtl*>(pinned_cache_alloc(sizeof(SolveCtl), false));
          p->htime = static_cast<int*>(pinned_cache_alloc(64, true));
          p->ctl.alloc(1, false);
        }
        for (int k = 2; k <= 5; k++) if (!p->graph_pow2[k]) { p->graph_pow2[k] = capture_passes(p, 1 << k); CUDA_OK(cudaGraphUpload(p->graph_pow2[k], s)); }
        if (!p->graph_check) { p->graph_check = capture_check(p, false, &p->check_launches[0]); CUDA_OK(cudaGraphUpload(p->graph_check, s)); }
        if (!p->graph_check_light) { p->graph_check_light = capture_check(p, true, &p->check_launches[1]); CUDA_OK(cudaGraphUpload(p->graph_check_light, s)); }
      }
    }
    CUDA_OK(cudaStreamSynchronize(s));
    lap("solve", "graphs ready (logical shards)");
    p->group->arrive_and_wait();
  }

  // ---- initial point: PDHG_PreSolve (hot start, cupdlp_solver.c:1217-1279) + PDHG_Init_Variables (:531-591)
  const bool dev_form = p->dev_form;
  std::vector<double> x0, y0;
  if (!dev_form) host_start_point(f, warm, x0, y0);
  const int nl = p->nl;   // column entries held by this rank (== n on one GPU)
  for (int k = 0; k < 2; k++) {
    CUDA_OK(cudaMemsetAsync(p->x[k].p, 0, (size_t)nl * sizeof(double), s));
    CUDA_OK(cudaMemsetAsync(p->aty[k].p, 0, (size_t)nl * sizeof(double), s));
    CUDA_OK(cudaMemsetAsync(p->y[k].p, 0, (size_t)std::max(ml, 1) * sizeof(double), s));
    CUDA_OK(cudaMemsetAsync(p->ax[k].p, 0, (size_t)std::max(ml, 1) * sizeof(double), s));
  }
  if (p->world > 1) {
    CUDA_OK(cudaMemsetAsync(p->xfull.p, 0, p->xfull.n * sizeof(double), s));
    CUDA_OK(cudaMemsetAsync(p->part.p, 0, p->part.n * sizeof(double), s));
    CUDA_OK(cudaMemsetAsync(p->red.p, 0, p->red.n * sizeof(double), s));
    CUDA_OK(cudaMemsetAsync(p->send.p, 0, p->send.n * sizeof(double), s));
    // fused path: nobody may store into a peer's xfull / recv before that peer has cleared them
    if (p->p2p) CUDA_OK(cudaMemsetAsync(p->fault.p, 0, sizeof(int), s));
    if (p->p2p) { launch_p2p_exchange(s, p->outs.p + 60, 0, p->peers, p->world, p->rank, p->epochs.p, p->fault.p); p->launches++; }
  }
  if (dev_form) {
    // maps and scales live in HBM: the hot start goes up in original order and is permuted / scaled / projected there
    const double *wc = nullptr, *wv = nullptr, *wd = nullptr;
    if (warm && warm->col_value && warm->row_value && warm->row_dual) {
      CUDA_OK(cudaMemcpyAsync(p->io_col.p, warm->col_value, (size_t)f.n_orig * sizeof(double), cudaMemcpyHostToDevice, s));
      CUDA_OK(cudaMemcpyAsync(p->io_row.p, warm->row_value, (size_t)m * sizeof(double), cudaMemcpyHostToDevice, s));
      CUDA_OK(cudaMemcpyAsync(p->io_row.p + m, warm->row_dual, (size_t)m * sizeof(double), cudaMemcpyHostToDevice, s));
      wc = p->io_col.p; wv = p->io_row.p; wd = p->io_row.p + m;
    }
    launch_init_point(s, p->prep.arr, f.sense, wc, wv, wd, p->colscale.p, p->lower.p, p->upper.p, p->rowscale.p, p->x[0].p,
                      p->xsum.p, p->y[0].p);
    p->launches += 2;
  } else {
    std::vector<double> xp(std::max(nl, 1), 0.0), yp(std::max(ml, 1));
    for (int i = 0; i < p->nl_real; i++) xp[i] = x0[p->cperm[p->c0 + i]];
    for (int i = 0; i < ml; i++) yp[i] = y0[p->r0 + p->rperm[i]];
    CUDA_OK(cudaMemcpyAsync(p->x[0].p, xp.data(), (size_t)nl * sizeof(double), cudaMemcpyHostToDevice, s));
    if (ml) CUDA_OK(cudaMemcpyAsync(p->y[0].p, yp.data(), (size_t)ml * sizeof(double), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));
  }

  // ---- PDHG_Init_Step_Sizes (cupdlp_step.c:312-375)
  {
    double a = 0.0, b = 0.0;   // cupdlp_twoNormSquared = dot(x,x), sequential on the reference's CPU path
    if (dev_form) { a = p->beta_cost_sq; b = p->beta_rhs_sq; }   // tree sums from the device prologue
    else {
      for (int j = 0; j < n; j++) a += f.cost[j] * f.cost[j];
      for (int i = 0; i < m; i++) b += f.rhs[i] * f.rhs[i];
    }
    h->beta = std::fmin(a, b) > 1e-6 ? a / b : 1.0;
    if (h->adaptive) {
      h->tau = (1.0 / f.amax) / std::sqrt(h->beta);
      h->sigma = h->tau * h->beta;
    } else {
      const double lambda = power_method(p);
      h->tau = 0.8 / std::sqrt(lambda);
      h->sigma = h->tau;
      h->tau /= std::sqrt(h->beta);
      h->sigma *= std::sqrt(h->beta);
    }
  }
  full_ax(p, p->x[0].p, p->ax[0].p);
  full_aty(p, p->y[0].p, p->aty[0].p);
  // sums start at proj(0) like PDHG_Init_Variables :577-583; the average is recomputed at every check
  if (!dev_form) {
    std::vector<double> z(std::max(nl, 1), 0.0);
    bool nz = false;
    for (int i = 0; i < p->nl_real; i++) {
      const double v = proj_zero(f, p->cperm[p->c0 + i]);
      z[i] = v;
      nz |= (v != 0.0);
    }
    if (nz) CUDA_OK(cudaMemcpyAsync(p->xsum.p, z.data(), (size_t)nl * sizeof(double), cudaMemcpyHostToDevice, s));
    else CUDA_OK(cudaMemsetAsync(p->xsum.p, 0, (size_t)nl * sizeof(double), s));
    CUDA_OK(cudaStreamSynchronize(s));
  }
  CUDA_OK(cudaMemsetAsync(p->ysum.p, 0, (size_t)std::max(ml, 1) * sizeof(double), s));
  CUDA_OK(cudaMemsetAsync(p->xlr.p, 0, (size_t)nl * sizeof(double), s));
  CUDA_OK(cudaMemsetAsync(p->ylr.p, 0, (size_t)std::max(ml, 1) * sizeof(double), s));
  arm_step(h);
  fill_pow_tables(h);
  push_state(p);
  CUDA_OK(cudaStreamSynchronize(s));
  lap("solve", "initial point + state");

  // ---- graphs: one check interval of passes, and a short one for top-ups after rejected steps
  // a few spare passes per replay: a rejected line-search step then still reaches the next check iteration inside
  // the same replay (spare passes are no-ops once state.iter == state.stop_iter) instead of costing a host round trip
  const int want_main = std::min(prm.graph_passes > 0 ? prm.graph_passes : interval + 4, kPowTab - 16);   // the step-rule tables cover one replay
  const bool dev_checks = use_device_checks(p, prm);
  if (p->graph_main && p->graph_main_passes != want_main) { cudaGraphExecDestroy(p->graph_main); p->graph_main = nullptr; }
  p->graph_main_passes = want_main;
  p->no_graph = getenv("B200PDLP_NO_GRAPH") != nullptr;
  if (!dev_checks && !p->no_graph) {   // (the device-driven loop captures the graphs it needs when it first needs them)
    if (!p->graph_main) p->graph_main = capture_passes(p, want_main);
    if (!p->graph_small) { p->graph_small_passes = 4; p->graph_small = capture_passes(p, 4); }
  }
  p->kernels_per_pass = p->world == 1 ? 4 : (p->p2p ? 5 : 6);   // ours; NCCL kernels not counted
  lap("solve", "graph capture");
  nvtxRangePop();
  nvtxRangePushA("b200pdlp: PDHG loop");

  const double tol_p = prm.tol_primal * (1.0 + f.norm_rhs), tol_d = prm.tol_dual * (1.0 + f.norm_cost);
  RestartMemo memo;
  CheckResult chk;
  int term = B200PDLP_TIMELIMIT_OR_ITERLIMIT, term_iterate = 0, restarts = 0;
  bool have_check = false;
  bool have_spec = false, spec_flag = false;   // a speculative check already produced the next check's scalars
  const bool speculate = can_speculate_check(p);
  bool h_light = false;
  CudaEvent ev0, ev1, evl0, evl1;
  double iter_ms = 0.0;
  CUDA_OK(cudaEventRecord(evl0, s));
  const auto t_loop = clk::now();

  if (dev_checks) {
    // ---- device-driven loop: the checks decide on the device (termination, restarts, next check iteration); the host
    // enqueues [check, passes to the next check] rounds ahead from the deterministic check schedule and reads the
    // control block once per batch.  A rejected line-search step makes a round fall short; the following rounds make
    // up for it (kernels are no-ops outside their turn) and the next read-back re-synchronises the prediction.
    if (!p->hctl) {
      p->hctl = static_cast<SolveCtl*>(pinned_cache_alloc(sizeof(SolveCtl), false));
      p->htime = static_cast<int*>(pinned_cache_alloc(64, true));
      p->ctl.alloc(1, false);   // (filled by the copy below; a cudaMemset on the legacy stream would not be ordered against p->stream)
    }
    SolveCtl* c = p->hctl;
    memset(c, 0, sizeof(SolveCtl));
    c->tol_p = tol_p; c->tol_d = tol_d; c->tol_gap = prm.tol_gap;
    c->sense = f.sense; c->offset = f.offset;
    c->iter_limit = prm.iter_limit; c->interval = interval; c->restart_on = prm.restart != 0; c->world = p->world;
    *p->htime = (t_lim >= 0 && std::chrono::duration<double>(clk::now() - t_loop).count() > t_lim) ? 1 : 0;
    {
      int* dflag = nullptr;
      CUDA_OK(cudaHostGetDevicePointer(&dflag, p->htime, 0));
      c->time_flag = t_lim >= 0 ? dflag : nullptr;   // (no limit: spare the device the read over PCIe)
    }
    c->term = -1;
    // dense-check phase (iterations 0 .. kDenseChecks-1 are all check iterations): the passes carry A xSum and A'ySum, the
    // checks are two vector sweeps.  B200PDLP_LIGHT_CHECK=0: every check multiplies the average iterate by A and A'.
    const bool hot = warm && warm->col_value && warm->row_value && warm->row_dual;
    h_light = p->axsum.p && p->atysum.p && (p->world == 1 || !hot);   // (several GPUs: A_g xSum of a hot start would need the gathered xSum)
    if (const char* e = getenv("B200PDLP_LIGHT_CHECK")) if (atoi(e) == 0) h_light = false;
    h->light_on = h_light ? 1 : 0;
    if (h_light) {
      // xSum starts at proj(0) (PDHG_Init_Variables): without a hot start that IS x, whose product is at hand
      if (hot) { launch_spmv_plain(s, p->A.dev, p->xsum.p, p->axsum.p); p->launches++; }
      else CUDA_OK(cudaMemcpyAsync(p->axsum.p, p->ax[0].p, (size_t)std::max(ml, 1) * sizeof(double), cudaMemcpyDeviceToDevice, s));
      CUDA_OK(cudaMemsetAsync(p->atysum.p, 0, (size_t)std::max(nl, 1) * sizeof(double), s));
    }
    if (out->trace && out->trace_cap > 0) {
      if (p->trace_dev.n < (size_t)out->trace_cap * B200PDLP_TRACE_COLS) p->trace_dev.alloc((size_t)out->trace_cap * B200PDLP_TRACE_COLS, false);
      c->trace = p->trace_dev.p; c->trace_cap = out->trace_cap;
    }
    CUDA_OK(cudaMemcpyAsync(p->ctl.p, c, sizeof(SolveCtl), cudaMemcpyHostToDevice, s));
    h->stop_iter = 0;   // the first check is due at once (iteration 0)
    push_state(p);
    auto next_stop = [&](int it) { return next_check_iter(it, interval, prm.iter_limit); };
    std::vector<std::unique_ptr<CudaEvent>> evs;
    int pred_iter = 0, carry = 0;   // carry: passes still owed before the next check (after a re-synchronisation)
    while (true) {
      size_t nev = 0;
      NvtxRange nvtx_batch("b200pdlp: batch of [check, passes] rounds");
      auto ev = [&]() -> cudaEvent_t {
        if (nev == evs.size()) evs.emplace_back(new CudaEvent());
        return *evs[nev++];
      };
      int rounds = 0, passes = 0;
      bool pred_term = false;
      if (carry > 0) {
        CUDA_OK(cudaEventRecord(ev(), s));
        enqueue_passes_device(p, carry);
        CUDA_OK(cudaEventRecord(ev(), s));
        passes += carry; pred_iter += carry; carry = 0;
      }
      while (rounds < 12 && passes < 48) {
        // pred_iter never runs behind the device's iteration count, so pred_iter < kDenseChecks implies the device is
        // inside the dense phase as well (the light kernels check it once more themselves)
        launch_check_graph(p, h_light && pred_iter < kDenseChecks);
        rounds++;
        if (pred_iter >= prm.iter_limit - 1) { pred_term = true; break; }
        const int next = next_stop(pred_iter);
        CUDA_OK(cudaEventRecord(ev(), s));
        enqueue_passes_device(p, next - pred_iter);
        CUDA_OK(cudaEventRecord(ev(), s));
        passes += next - pred_iter;
        pred_iter = next;
      }
      (void)pred_term;
      CUDA_OK(cudaMemcpyAsync(c, p->ctl.p, sizeof(SolveCtl), cudaMemcpyDeviceToHost, s));
      CUDA_OK(cudaMemcpyAsync(h, p->state.p, sizeof(PdhgState), cudaMemcpyDeviceToHost, s));
      int* hfault = reinterpret_cast<int*>(p->hflag + 2);
      if (p->p2p) CUDA_OK(cudaMemcpyAsync(hfault, p->fault.p, sizeof(int), cudaMemcpyDeviceToHost, s));
      const size_t npairs = nev / 2;   // events so far come in (before, after) pairs around the passes
      cudaEvent_t fin = ev();
      CUDA_OK(cudaEventRecord(fin, s));
      if (t_lim >= 0) {
        // poll, so that the time-limit word can be raised while the batch runs
        while (cudaEventQuery(fin) == cudaErrorNotReady) {
          if (std::chrono::duration<double>(clk::now() - t_loop).count() > t_lim) *p->htime = 1;
          std::this_thread::yield();
        }
      }
      CUDA_OK(cudaEventSynchronize(fin));
      if (p->p2p && *hfault) throw Error(B200PDLP_ERR_STATE, "P2P barrier timed out (a peer rank did not arrive)");
      for (size_t k = 0; k < npairs; k++) {
        float ms = 0.f;
        CUDA_OK(cudaEventElapsedTime(&ms, *evs[2 * k], *evs[2 * k + 1]));
        iter_ms += ms;
      }
      if (c->term >= 0) break;
      // not finished: continue from where the device really is
      h_light = h_light && h->light_on != 0;
      pred_iter = h->iter;
      carry = std::max(0, h->stop_iter - h->iter);
    }
    term = c->term; term_iterate = c->term_iterate; restarts = c->restarts;
    have_check = c->checks > 0;
    for (int t = 0; t < 2; t++) {
      const DevResiduals& d = c->res[t];
      Residuals& R = chk.it[t];
      R.pobj = d.pobj; R.dobj = d.dobj; R.pfeas = d.pfeas; R.dfeas = d.dfeas; R.gap = d.gap; R.relgap = d.relgap;
      R.pinf_obj = d.pinf_obj; R.pinf_res = d.pinf_res; R.dinf_obj = d.dinf_obj; R.dinf_res = d.dinf_res;
    }
    if (c->trace) {
      out->trace_len = std::min(c->trace_len, out->trace_cap);
      if (out->trace_len > 0)
        CUDA_OK(cudaMemcpyAsync(out->trace, p->trace_dev.p, (size_t)out->trace_len * B200PDLP_TRACE_COLS * sizeof(double),
                                cudaMemcpyDeviceToHost, s));
    }
  } else
  // ---- main loop (cupdlp_solver.c:939-1106)
  while (h->iter < prm.iter_limit) {
    const double elapsed = std::chrono::duration<double>(clk::now() - t_loop).count();
    const bool timed_out_local = t_lim >= 0 && elapsed > t_lim;
    if (have_spec) { chk = parse_fused_check(p, spec_flag); have_spec = false; }
    else chk = run_check(p, timed_out_local);
    have_check = true;
    const Residuals &L = chk.it[0], &A = chk.it[1];
    if (prm.log_level >= 2)
      printf("[b200pdlp] it %8d  pobj %+.8e dobj %+.8e  pfeas %.2e dfeas %.2e | avg pobj %+.8e dobj %+.8e pfeas %.2e dfeas %.2e  tau %.3e sigma %.3e\n",
             h->iter, L.pobj, L.dobj, L.pfeas, L.dfeas, A.pobj, A.dobj, A.pfeas, A.dfeas, h->tau, h->sigma);
    int choice = 0;
    const int t_code = check_decision(prm, tol_p, tol_d, h, chk, memo, &term_iterate, &choice);
    if (t_code >= 0) { term = t_code; trace_row(out, h, chk, 0); break; }
    bool dirty = false;
    if (choice) { do_restart(p, choice, chk, memo); restarts++; arm_step(h); dirty = true; }
    trace_row(out, h, chk, choice);
    const int next = next_check_iter(h->iter, interval, prm.iter_limit);
    h->stop_iter = next;
    fill_pow_tables(h);
    dirty = true;
    if (dirty) push_state(p);
    CUDA_OK(cudaEventRecord(ev0, s));
    bool have_ev1 = false;
    while (true) {
      const int need = next - h->iter;
      if (p->no_graph) {
        for (int q = 0; q < std::min(need + 4, p->graph_main_passes); q++) { enqueue_pass(p); p->launches += p->kernels_per_pass; }
      } else if (need >= p->graph_main_passes / 2 || need > p->graph_small_passes) {
        CUDA_OK(cudaGraphLaunch(p->graph_main, s));
        p->launches += (long long)p->graph_main_passes * p->kernels_per_pass;
      } else if (need > 1) {
        CUDA_OK(cudaGraphLaunch(p->graph_small, s));
        p->launches += (long long)p->graph_small_passes * p->kernels_per_pass;
      } else {
        enqueue_pass(p);
        p->launches += p->kernels_per_pass;
      }
      if (speculate) {
        if (!have_ev1) { CUDA_OK(cudaEventRecord(ev1, s)); have_ev1 = true; }
        const double el = std::chrono::duration<double>(clk::now() - t_loop).count();
        spec_flag = t_lim >= 0 && el > t_lim;
        enqueue_check_dev(p, spec_flag);
      }
      pull_state(p);
      if (h->iter >= next) { have_spec = speculate; break; }
      have_ev1 = false;
      if (h->step_iter - h->pow_base > kPowTab - p->graph_main_passes - 8) { fill_pow_tables(h); push_state(p); }
    }
    if (!have_ev1) CUDA_OK(cudaEventRecord(ev1, s));
    CUDA_OK(cudaEventSynchronize(ev1));
    float ms = 0.f;
    CUDA_OK(cudaEventElapsedTime(&ms, ev0, ev1));
    iter_ms += ms;
  }
  CUDA_OK(cudaEventRecord(evl1, s));
  CUDA_OK(cudaEventSynchronize(evl1));
  float loop_ms = 0.f;
  CUDA_OK(cudaEventElapsedTime(&loop_ms, evl0, evl1));
  const double solve_seconds = std::chrono::duration<double>(clk::now() - t_loop).count();
  out->loop_device_ms = loop_ms;
  lap("solve", "iterations");
  nvtxRangePop();
  NvtxRange nvtx_post("b200pdlp: postsolve + download");

  if (p->world > 1 && getenv("B200PDLP_DEBUG_MG")) {
    // diagnostics: per-rank barrier / exchange counts and checksums of what the postsolve is about to assemble
    unsigned long long ep[16] = {0};
    if (p->epochs.p) CUDA_OK(cudaMemcpy(ep, p->epochs.p, sizeof(ep), cudaMemcpyDeviceToHost));
    auto csum = [&](const double* d, int len) {
      std::vector<double> t(std::max(len, 1));
      if (len > 0) CUDA_OK(cudaMemcpy(t.data(), d, (size_t)len * sizeof(double), cudaMemcpyDeviceToHost));
      double a = 0.0; for (int i = 0; i < len; i++) a += t[i] * (1.0 + (i % 7)); return a;
    };
    fprintf(stderr, "[b200pdlp mg-debug] rank %d iter %d cur %d term %d term_iterate %d light_on %d | barrier0 %llu barrier1 %llu exchange %llu | "
            "x[cur] %.17g xavg %.17g y[cur] %.17g yavg %.17g ax[cur] %.17g axavg %.17g aty0 %.17g atyavg %.17g\n",
            p->rank, h->iter, h->cur, term, term_iterate, h->light_on, ep[0], ep[1], ep[10],
            csum(p->x[h->cur].p, p->nl), csum(p->xavg.p, p->nl), csum(p->y[h->cur].p, ml), csum(p->yavg.p, ml),
            csum(p->ax[h->cur].p, ml), csum(p->axavg.p, ml), csum(p->aty[0].p, p->nl), csum(p->atyavg.p, p->nl));
  }
  // ---- PDHG_PostSolve (cupdlp_solver.c:1281-1435)
  const int cur = h->cur;
  const bool use_avg = (term == B200PDLP_OPTIMAL && term_iterate == 1);
  const double* dx = use_avg ? p->xavg.p : p->x[cur].p;
  const double* dy = use_avg ? p->yavg.p : p->y[cur].p;
  const double* dax = use_avg ? p->axavg.p : p->ax[cur].p;
  if (p->world > 1 && h->accepted_last && !use_avg) {   // (only when the loop never ran a check, e.g. iter_limit <= 0)
    if (p->p2p) launch_reduce_part_p2p(s, nl, p->aty[0].p, p->peers, p->world, p->rank, p->seg_len, 1);
    else CUDA_OK(cudaMemcpyAsync(p->aty[0].p, p->red.p, (size_t)nl * sizeof(double), cudaMemcpyDeviceToDevice, s));
  }
  if (p->p2p) {
    int fault = 0;
    CUDA_OK(cudaMemcpyAsync(&fault, p->fault.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    if (fault) throw Error(B200PDLP_ERR_STATE, "P2P barrier timed out (a peer rank did not arrive)");
  }
  const double* daty = use_avg ? p->atyavg.p : p->aty[p->world == 1 ? cur : 0].p;
  if (dev_form) {
    // PDHG_PostSolve on the device (device_prep.cu post_*_kernel): un-permute, un-scale, sign conventions, slacks of
    // BOUND rows; four original-order vectors come back
    if (out->col_value && out->col_dual && out->row_value && out->row_dual) {
      const int n0 = f.n_orig;
      launch_postsolve(s, p->prep.arr, f.sense, have_check ? 1 : 0, dx, daty, dy, dax, p->cost.p, p->lower.p, p->upper.p,
                       p->colscale.p, p->rowscale.p, p->io_col.p, p->io_col.p + n0, p->io_row.p, p->io_row.p + m);
      p->launches += 2;
      CUDA_OK(cudaMemcpyAsync(out->col_value, p->io_col.p, (size_t)n0 * sizeof(double), cudaMemcpyDeviceToHost, s));
      CUDA_OK(cudaMemcpyAsync(out->col_dual, p->io_col.p + n0, (size_t)n0 * sizeof(double), cudaMemcpyDeviceToHost, s));
      CUDA_OK(cudaMemcpyAsync(out->row_value, p->io_row.p, (size_t)m * sizeof(double), cudaMemcpyDeviceToHost, s));
      CUDA_OK(cudaMemcpyAsync(out->row_dual, p->io_row.p + m, (size_t)m * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    CUDA_OK(cudaStreamSynchronize(s));
    lap("solve", "postsolve (device) + download");
  } else {
  std::vector<double> hx(n), hy(m, 0.0), hax(m, 0.0), haty(n);
  {
    // device order -> standard-form order
    std::vector<double> t(std::max<size_t>(std::max(n, std::max(ml, 1)), p->xfull.n));
    const bool dbg = p->world > 1 && getenv("B200PDLP_DEBUG_MG") != nullptr;
    // Logical shards share ONE CUDA context: a context-synchronising driver call on one rank's host thread (a pageable copy
    // that needs staging memory, a lazy module load, an allocation) waits for every running kernel, including a peer's
    // barrier kernel that is spinning for THIS rank's next launch -- a deadlock that only the barrier's timeout breaks
    // (and the assembly would then run on with stale segments).  So with local links every host-blocking copy
    // of the assembly sits between two host-side rendezvous, when no barrier kernel is in flight.  Separate processes
    // (CUDA IPC) have separate contexts and do not need this.
    const bool rendezvous = p->local_link && p->group;
    int dbg_stage = 0;
    auto dbg_segments = [&](const char* what) {
      if (!dbg) return;
      char line[1024]; int k = snprintf(line, sizeof line, "[b200pdlp mg-debug] rank %d stage %d %s segments:", p->rank, dbg_stage++, what);
      for (int g = 0; g < p->world && k < 900; g++) {
        double a = 0.0;
        for (int i = 0; i < p->seg_len; i++) a += t[(size_t)g * p->seg_len + i] * (1.0 + (i % 7));
        k += snprintf(line + k, sizeof line - k, " %.15g", a);
      }
      fprintf(stderr, "%s\n", line);
    };
    // barrier of the assembly; with local links the ranks also meet on the host before AND after it (see above): nobody
    // launches a kernel that spins for its peers while a peer's host may still sit in a blocking copy, and nobody starts a
    // blocking copy while a peer's barrier kernel is still in flight
    auto xchg = [&]() {
      if (rendezvous) { CUDA_OK(cudaStreamSynchronize(s)); p->group->arrive_and_wait(); }
      launch_p2p_exchange(s, p->outs.p + 60, 0, p->peers, p->world, p->rank, p->epochs.p, p->fault.p);
      p->launches++;
      if (rendezvous) { CUDA_OK(cudaStreamSynchronize(s)); p->group->arrive_and_wait(); }
    };
    auto down_col = [&](const double* d, std::vector<double>& h) {
      if (p->world == 1) {
        CUDA_OK(cudaMemcpyAsync(t.data(), d, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, s));
        CUDA_OK(cudaStreamSynchronize(s));
        for (int j = 0; j < n; j++) h[p->cperm[j]] = t[j];
      } else if (p->p2p && !p->comm) {
        // no NCCL communicator (logical shards of one process, or B200PDLP_NO_NCCL): all-gather through the peers' xfull,
        // with a barrier before anyone reads and one before anyone overwrites
        launch_push_shard(s, d, nl, p->peers, p->world, p->rank, p->seg_len);
        p->launches++;
        xchg();
        CUDA_OK(cudaMemcpyAsync(t.data(), p->xfull.p, p->xfull.n * sizeof(double), cudaMemcpyDeviceToHost, s));
        xchg();
        CUDA_OK(cudaStreamSynchronize(s));
        dbg_segments("columns");
        for (int j = 0; j < n; j++) h[p->cperm[j]] = t[seg_pos(p, j)];
      } else {   // all-gather the column shards, then unpack the segmented vector
        CUDA_OK(cudaMemcpyAsync(p->send.p, d, (size_t)nl * sizeof(double), cudaMemcpyDeviceToDevice, s));
        gather_shards(p);
        CUDA_OK(cudaMemcpyAsync(t.data(), p->xfull.p, p->xfull.n * sizeof(double), cudaMemcpyDeviceToHost, s));
        CUDA_OK(cudaStreamSynchronize(s));
        for (int j = 0; j < n; j++) h[p->cperm[j]] = t[seg_pos(p, j)];
      }
    };
    auto down_row = [&](const double* d, std::vector<double>& h) {
      if (ml) CUDA_OK(cudaMemcpyAsync(t.data(), d, (size_t)ml * sizeof(double), cudaMemcpyDeviceToHost, s));
      CUDA_OK(cudaStreamSynchronize(s));
      for (int i = 0; i < ml; i++) h[p->r0 + p->rperm[i]] = t[i];
      if (p->world > 1 && p->p2p && !p->comm) {
        // no NCCL communicator: every rank stores its rows (standard-form order) into slot `rank` of every peer's
        // receive buffer, seg_len rows at a time; all ranks run the same number of rounds
        int max_ml = 0;
        for (int g = 0; g < p->world; g++) max_ml = std::max(max_ml, p->row_bounds[g + 1] - p->row_bounds[g]);
        if (ml) CUDA_OK(cudaMemcpyAsync(p->redbuf.p, h.data() + p->r0, (size_t)ml * sizeof(double), cudaMemcpyHostToDevice, s));
        const int rounds = (max_ml + p->seg_len - 1) / p->seg_len;
        for (int c = 0; c < rounds; c++) {
          const int off = c * p->seg_len;
          launch_push_rows(s, p->redbuf.p + off, std::max(0, std::min(ml - off, p->seg_len)), p->peers, p->world, p->rank, p->seg_len);
          p->launches++;
          xchg();
          CUDA_OK(cudaMemcpyAsync(t.data(), p->recv.p, (size_t)p->world * p->seg_len * sizeof(double), cudaMemcpyDeviceToHost, s));
          xchg();
          CUDA_OK(cudaStreamSynchronize(s));
          dbg_segments("rows");
          for (int g = 0; g < p->world; g++) {
            const int mg = p->row_bounds[g + 1] - p->row_bounds[g];
            const int cnt = std::max(0, std::min(mg - off, p->seg_len));
            for (int i = 0; i < cnt; i++) h[p->row_bounds[g] + off + i] = t[(size_t)g * p->seg_len + i];
          }
        }
      } else if (p->world > 1) {   // other ranks' rows: zero-padded sum
        CUDA_OK(cudaMemcpyAsync(p->redbuf.p, h.data(), (size_t)m * sizeof(double), cudaMemcpyHostToDevice, s));
        allreduce_inplace(p, p->redbuf.p, m);
        CUDA_OK(cudaMemcpyAsync(h.data(), p->redbuf.p, (size_t)m * sizeof(double), cudaMemcpyDeviceToHost, s));
        CUDA_OK(cudaStreamSynchronize(s));
      }
    };
    down_col(dx, hx); down_col(daty, haty); down_row(dy, hy); down_row(dax, hax);
    if (p->p2p) {   // a barrier of the assembly that timed out leaves stale segments behind: an error, not a result
      int fault = 0;
      CUDA_OK(cudaMemcpyAsync(&fault, p->fault.p, sizeof(int), cudaMemcpyDeviceToHost, s));
      CUDA_OK(cudaStreamSynchronize(s));
      if (fault) throw Error(B200PDLP_ERR_STATE, "P2P barrier timed out while the solution was being assembled (a peer rank did not arrive)");
    }
  }
  lap("solve", "solution download");
  host_postsolve(f, have_check, hx, hy, hax, haty, out);
  }   // host postsolve
  fill_result(out, f, h, term, term_iterate, restarts, chk);
  out->kernel_launches = (int)std::min<long long>(p->launches - launches0, 2147483647LL);
  out->solve_seconds = solve_seconds;
  out->iter_device_ms = iter_ms;
  out->setup_seconds += std::chrono::duration<double>(t_loop - t_begin).count();
  lap("solve", "postsolve (host)");
}

// =================================================================================================== HiPDLP mode
// solveLpHiPdlp -> PDLPSolver::solve (/root/reference/highs/pdlp/hipdlp/pdhg.cc:494-707) on the device, single GPU.
// STATUS: runs on hardware (tests/test_gpu_hipdlp.py, tests/test_gpu_dropin.py, tests/test_gpu_hipdlp_device_prep.py,
// bench.py --solver hipdlp).  Tree mode on one GPU takes the device-resident prologue, initial point and postsolve by default;
// ordered mode keeps the host prologue (host_prep_hipdlp.cpp, the device prologue's tested twin).

// The device prologue (DevicePrologue::hipdlp) unless: B200PDLP_DEVICE_PREP=0 or params.device_prep = -1 (the host prologue on
// request), ordered mode (the standard form's max(n, m) <= ordered_max, decided with HiPDLP's classification: +-infinity
// thresholds, a slack column for every ranged and free row), or an empty matrix.
static bool use_device_prep_hipdlp(const b200pdlp_lp& lp, const b200pdlp_hipdlp_params& prm) {
  if (const char* e = getenv("B200PDLP_DEVICE_PREP")) { if (atoi(e) == 0) return false; }
  if (prm.device_prep == -1) return false;
  return device_prep_fits(lp, prm.ordered_max, std::numeric_limits<double>::infinity());
}

// the HiPDLP iterate set, its pinned state mirror and the scratch, all zeroed
static void hipdlp_buffers(b200pdlp_problem* p) {
  const int n = p->n, m = p->m;
  auto& h = p->hip;
  for (DevBuf<double>* b : {&h.x, &h.xn, &h.rx, &h.xa, &h.aty, &h.atyp, &h.atdy, &h.hslack, &h.sp, &h.sn}) b->alloc(n);
  for (DevBuf<double>* b : {&h.y, &h.yn, &h.ry, &h.ya, &h.axp, &h.dy}) b->alloc(m);
  h.state.alloc(1);
  h.hstate = static_cast<HipState*>(pinned_cache_alloc(sizeof(HipState), false));
  alloc_scratch(p, true);
}

// the whole HiPDLP prologue on the device: formulate, scale, unscaled norms, row index, orderings, both layouts, the
// row-major copy of the caller's matrix for the postsolve (device_prep.cu); the host learns sizes and scalars only
static void create_problem_hipdlp_device(const b200pdlp_lp& lp, const b200pdlp_hipdlp_params& prm, b200pdlp_problem* p) {
  NvtxRange nvtx("b200pdlp: HiPDLP prologue (device)");
  Laps lap;
  p->dev_form = true;
  DevicePrologue& P = p->prep;
  P.hipdlp = true;
  P.scaling_mode = prm.scaling_mode;
  P.ruiz_iterations = prm.ruiz_iterations;
  run_prologue(P, p->stream, lp, true);
  lap("setup", "device prologue (HiPDLP)");
  if (lap.on) fprintf(stderr, "[b200pdlp setup] ordered |c|^2, |b|^2 (side stream, under the layouts) %8.3f ms\n", P.sc.norms_ms);
  take_prologue(lp, P, p);
  adopt_matrix(p->A, P.A);
  adopt_matrix(p->AT, P.AT);
  apply_spmv_grid(p);
  hipdlp_buffers(p);
  alloc_postsolve_staging(p);
  CUDA_OK(cudaStreamSynchronize(p->stream));
  lap("setup", "vectors + scratch");
}

static void create_problem_hipdlp(const b200pdlp_lp& lp, const b200pdlp_hipdlp_params& prm, b200pdlp_problem* p) {
  open_problem(p, prm.device, 0, 1);
  if (use_device_prep_hipdlp(lp, prm)) { create_problem_hipdlp_device(lp, prm, p); return; }
  Laps lap;
  formulate_hipdlp(lp, p->form);
  scale_hipdlp(p->form, prm.scaling_mode, prm.ruiz_iterations);
  lap("setup", "formulate + scale (host)");
  StdForm& f = p->form;
  {
    HostLayout L;
    build_layout(f, 0, 1, prm.ordered_max, L);
    take_layout(p, std::move(L));
  }
  lap("setup", "layouts (host)");
  p->A.upload();
  p->AT.upload();
  const int n = p->n, m = p->m;
  const int* cperm = p->cperm.data();
  const int* rperm = p->rperm.data();
  upload_permuted(p->cost, f.cost, cperm, 0, n, n); upload_permuted(p->lower, f.lower, cperm, 0, n, n);
  upload_permuted(p->upper, f.upper, cperm, 0, n, n); upload_permuted(p->colscale, f.col_scale, cperm, 0, n, n);
  upload_permuted(p->rhs, f.rhs, rperm, 0, m, m); upload_permuted(p->hip.rup, f.row_upper, rperm, 0, m, m);
  upload_permuted(p->rowscale, f.row_scale, rperm, 0, m, m);
  hipdlp_buffers(p);
  CUDA_OK(cudaDeviceSynchronize());
  lap("setup", "upload + scratch");
}

// ---- HiPDLP on several GPUs.  Rank g computes whole rows of A (device rows [hip_r0, hip_r1)) and whole rows of A'
// (device columns [hip_c0, hip_c1)) in the one-GPU entry order, and every check sum runs over full vectors with the
// one-GPU kernels, so a G-rank solve returns the one-GPU bits (DESIGN section 5, "HiPDLP on several GPUs").
using HipBufs = b200pdlp_problem::HipBuffers;
using HipVec = DevBuf<double> HipBufs::*;
static bool hip_sharded(const b200pdlp_problem* p) { return !p->hip_peers.empty(); }

// what the solve loop reads of the standard form on every rank (rank 0 takes the whole form for the postsolve)
static StdForm hip_form_scalars(const StdForm& f) {
  StdForm s;
  s.hipdlp = true; s.scaled = f.scaled;
  s.n = f.n; s.m = f.m; s.nnz = f.nnz; s.neq = f.neq; s.n_orig = f.n_orig;
  s.sense = f.sense; s.offset = f.offset; s.norm_cost = f.norm_cost; s.norm_rhs = f.norm_rhs; s.amax = f.amax;
  return s;
}

// rank g's problem on `device`: A_g, A_g' (build_hipdlp_shard) and every vector full length in the one-GPU device order
static void create_problem_hipdlp_shard(const StdForm& f, const HipShards& S, int rank, int device, b200pdlp_problem* p) {
  open_problem(p, device, rank, S.world);
  p->form = hip_form_scalars(f);
  set_full_length_dims(p);
  p->ordered = S.ordered;
  p->hip_r0 = S.rb[rank]; p->hip_r1 = S.rb[rank + 1]; p->hip_c0 = S.cb[rank]; p->hip_c1 = S.cb[rank + 1];
  if (rank == 0) { p->rperm = S.rperm; p->cperm = S.cperm; }   // the postsolve's un-permutation
  build_hipdlp_shard(S, rank, p->A.host, p->AT.host);
  p->A.upload();
  p->AT.upload();
  const int n = f.n, m = f.m;
  upload_permuted(p->cost, f.cost, S.cperm.data(), 0, n, n); upload_permuted(p->lower, f.lower, S.cperm.data(), 0, n, n);
  upload_permuted(p->upper, f.upper, S.cperm.data(), 0, n, n); upload_permuted(p->colscale, f.col_scale, S.cperm.data(), 0, n, n);
  upload_permuted(p->rhs, f.rhs, S.rperm.data(), 0, m, m); upload_permuted(p->hip.rup, f.row_upper, S.rperm.data(), 0, m, m);
  upload_permuted(p->rowscale, f.row_scale, S.rperm.data(), 0, m, m);
  hipdlp_buffers(p);
  alloc_peer_words(p);
  CUDA_OK(cudaDeviceSynchronize());
}

// The same problems from the device prologue in block mode (DevicePrologue::world > 1): one prologue per device, shared by
// the ranks that live there.  Formulate, scaling, orderings, the partition and A_g / A_g' of `ranks` on the current device;
// returns with the stream idle.
static void run_hipdlp_shard_prologue(const b200pdlp_lp& lp, int scaling_mode, int ruiz_iterations, int world,
                                      const std::vector<int>& ranks, TempPrologue& T) {
  DevicePrologue& P = T.P;
  P.hipdlp = true;
  P.scaling_mode = scaling_mode;
  P.ruiz_iterations = ruiz_iterations;
  P.world = world;
  P.ranks = ranks;
  run_prologue(P, T.stream, lp, true);
}

// rank P.ranks[k]'s problem: it adopts its A_g / A_g' and takes its own copies of the full-length device-order vectors
static void create_problem_hipdlp_shard_device(const b200pdlp_lp& lp, TempPrologue& T, int k, b200pdlp_problem* p) {
  DevicePrologue& P = T.P;
  const int g = P.ranks[k];
  open_problem(p, T.device, g, P.world);
  p->dev_form = true;
  take_prologue(lp, P, p);
  p->hip_r0 = P.rb[g]; p->hip_r1 = P.rb[g + 1]; p->hip_c0 = P.cb[g]; p->hip_c1 = P.cb[g + 1];
  adopt_matrix(p->A, P.block_A[k]);
  adopt_matrix(p->AT, P.block_AT[k]);
  hipdlp_buffers(p);
  alloc_peer_words(p);
  if (g == 0) alloc_postsolve_staging(p);
  CUDA_OK(cudaStreamSynchronize(p->stream));
}

// rank 0 keeps the maps of the formulation and the row-major copy of the caller's matrix for the device postsolve; the
// device-order vectors were copied by every rank
static void hand_over_postsolve_maps(TempPrologue& T, b200pdlp_problem* p0) {
  DevProblemArrays& a = T.P.arr;
  for (double** v : {&a.cost, &a.lower, &a.upper, &a.colscale, &a.rhs, &a.rowscale, &a.rup}) { dev_cache_free(*v); *v = nullptr; }
  p0->prep.arr = a;
  a = DevProblemArrays();
}

static void hip_barrier(b200pdlp_problem* p) {
  PeerFlags pf{};
  for (size_t g = 0; g < p->hip_peers.size(); g++) pf.f[g] = p->hip_peers[g]->flags.p;
  launch_hip_barrier(p->stream, pf, p->world, p->rank, p->epochs.p, p->fault.p);
  p->launches++;
}
static PeerVec hip_peer_vec(const b200pdlp_problem* p, HipVec v, int offset = 0) {
  PeerVec r{};
  for (size_t g = 0; g < p->hip_peers.size(); g++) r.v[g] = (p->hip_peers[g]->hip.*v).p + offset;
  return r;
}
// this rank's columns (cols) or rows of the given vectors into every peer's copies
static void hip_gather(b200pdlp_problem* p, bool cols, std::initializer_list<HipVec> vs) {
  HipGather g{};
  g.lo = cols ? p->hip_c0 : p->hip_r0;
  g.hi = cols ? p->hip_c1 : p->hip_r1;
  for (HipVec v : vs) { g.src[g.nv] = (p->hip.*v).p; g.dst[g.nv] = hip_peer_vec(p, v); g.nv++; }
  launch_hip_gather(p->stream, g, p->world, p->rank);
  p->launches++;
}

static void hip_step(b200pdlp_problem* p, int k_offset, int is_major) {
  auto& h = p->hip;
  cudaStream_t s = p->stream;
  if (hip_sharded(p)) {
    // The reflected x and the blended y go straight into the peers' copies, and two barriers per step suffice.  A rank
    // stores into a peer's rx only after it has left the previous step's second barrier, which every rank reaches after
    // its A_g rx, the only reader of rx in a block.  It stores into a peer's y only after this step's first barrier, which
    // every rank reaches after the previous step's A_g' y, the only reader of other ranks' rows of y in a block.
    const int r0 = p->hip_r0, c0 = p->hip_c0;
    launch_hip_primal_shard(s, c0, p->hip_c1, h.state.p, k_offset, is_major, h.x.p, h.xa.p, p->cost.p, h.aty.p, p->lower.p,
                            p->upper.p, h.rx.p, h.xn.p, h.hslack.p, hip_peer_vec(p, &HipBufs::rx), p->world, p->rank);
    hip_barrier(p);
    launch_hip_dual_shard(s, p->A.dev, h.state.p, k_offset, is_major, h.rx.p, h.y.p + r0, h.ya.p + r0, p->rhs.p + r0,
                          h.rup.p + r0, h.yn.p + r0, h.ry.p + r0, hip_peer_vec(p, &HipBufs::y, r0), p->world, p->rank);
    hip_barrier(p);
    launch_spmv_plain(s, p->AT.dev, h.y.p, h.aty.p + c0);
    p->launches += 3;
    return;
  }
  launch_hip_primal(s, p->n, h.state.p, k_offset, is_major, h.x.p, h.xa.p, p->cost.p, h.aty.p, p->lower.p, p->upper.p,
                    h.rx.p, h.xn.p, h.hslack.p);
  launch_hip_dual(s, p->A.dev, h.state.p, k_offset, is_major, h.rx.p, h.y.p, h.ya.p, p->rhs.p, h.rup.p, h.yn.p, h.ry.p);
  launch_spmv_plain(s, p->AT.dev, h.y.p, h.aty.p);
  p->launches += 3;
}

// the scalars of one check (launch_hip_check) for the iterate (x, y), or with `major` for (xn, yn) together with the
// fixed-point error and the cached slacks of the major step that produced it.  Leaves them in p->houts[0..8] after ONE
// synchronisation.  Several GPUs: the iterate is gathered to every rank, each rank forms its rows of A x and its
// columns of A'y (and A'dy), those are gathered too, and every rank then sums full vectors with the one-GPU kernels,
// so all ranks see the one-GPU sums and take the same decisions.
static void hip_check(b200pdlp_problem* p, int major) {
  auto& h = p->hip;
  cudaStream_t s = p->stream;
  const HipVec xv = major ? &HipBufs::xn : &HipBufs::x, yv = major ? &HipBufs::yn : &HipBufs::y;
  const double* x = (h.*xv).p;
  const double* y = (h.*yv).p;
  const bool shard = hip_sharded(p);
  const int r0 = p->hip_r0, c0 = p->hip_c0;
  if (shard) {
    if (major) { hip_gather(p, true, {xv, &HipBufs::hslack}); hip_gather(p, false, {yv, &HipBufs::ry}); }
    else { hip_gather(p, true, {xv}); hip_gather(p, false, {yv}); }
    hip_barrier(p);
  }
  if (major) {
    launch_hip_diff(s, p->m, y, h.ry.p, h.dy.p);
    launch_spmv_plain(s, p->AT.dev, h.dy.p, h.atdy.p + c0);
    p->launches += 2;
  }
  launch_spmv_plain(s, p->A.dev, x, h.axp.p + r0);
  launch_spmv_plain(s, p->AT.dev, y, h.atyp.p + c0);
  if (shard) {
    if (major) hip_gather(p, true, {&HipBufs::atyp, &HipBufs::atdy});
    else hip_gather(p, true, {&HipBufs::atyp});
    hip_gather(p, false, {&HipBufs::axp});
    hip_barrier(p);
  }
  const int with_fpe = major, use_cached_slack = major;
  launch_hip_slack(s, p->n, use_cached_slack, h.hslack.p, p->cost.p, h.atyp.p, p->lower.p, p->upper.p, h.sp.p, h.sn.p);
  HipCheckArgs a{};
  a.n = p->n; a.m = p->m; a.neq = p->neq_local; a.scaled = p->form.scaled ? 1 : 0; a.offset = p->form.offset;
  a.x = x; a.y = y; a.ax = h.axp.p; a.aty = h.atyp.p; a.rx = h.rx.p; a.ry = h.ry.p; a.atdy = h.atdy.p;
  a.xa = h.xa.p; a.ya = h.ya.p; a.c = p->cost.p; a.lo = p->lower.p; a.up = p->upper.p; a.rlo = p->rhs.p;
  a.colscale = p->colscale.p; a.rowscale = p->rowscale.p; a.sp = h.sp.p; a.sn = h.sn.p;
  launch_hip_check(s, a, with_fpe, p->ordered ? 1 : 0, p->rs(kSlotChk, std::max(p->n, p->m)), p->outs.p);
  p->launches += 4;
  CUDA_OK(cudaMemcpyAsync(p->houts, p->outs.p, 9 * sizeof(double), cudaMemcpyDeviceToHost, s));
  int* hfault = reinterpret_cast<int*>(p->houts + 32);
  if (shard) CUDA_OK(cudaMemcpyAsync(hfault, p->fault.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  if (shard) {
    if (*hfault) throw Error(B200PDLP_ERR_STATE, "HiPDLP shards: a barrier timed out (a peer rank did not arrive)");
    // no rank starts the next step (which stores into its peers' rx) before every rank has finished reading rx here
    p->group->arrive_and_wait();
  }
}

// unscaleSolution + postprocess (pdhg.cc:1883-1897, :359-492) of a host-prologue form on the host: x, y in device order
// (cperm / rperm: device -> standard-form order), or nullptr when the run did not converge (the reference then returns
// x = y = 0), and the dual slacks sp, sn of the last check in device order -> the four vectors of `out`, when it has them
static void hip_host_postsolve(const b200pdlp_lp& lp, const StdForm& f, const int* cperm, const int* rperm, const double* x,
                               const double* y, const double* sp, const double* sn, b200pdlp_result* out) {
  const int n = f.n, m = f.m;
  std::vector<double> hx(std::max(n, 1), 0.0), hy(std::max(m, 1), 0.0), hsp(std::max(n, 1)), hsn(std::max(n, 1));
  if (x) {
    for (int i = 0; i < n; i++) hx[cperm[i]] = x[i];
    for (int i = 0; i < m; i++) hy[rperm[i]] = y[i];
  }
  for (int i = 0; i < n; i++) { hsp[cperm[i]] = sp[i]; hsn[cperm[i]] = sn[i]; }
  if (f.scaled) {
    for (int i = 0; i < n; i++) hx[i] /= f.col_scale[i];
    for (int i = 0; i < m; i++) hy[i] /= f.row_scale[i];
  }
  for (int i = 0; i < n; i++) { hsp[i] *= f.col_scale[i]; hsn[i] *= f.col_scale[i]; }
  if (out->col_value && out->col_dual && out->row_value && out->row_dual) {
    for (int j = 0; j < f.n_orig; j++) out->col_value[j] = hx[j];
    for (int i = 0; i < m; i++) {
      const double d = hy[f.row_new_idx[i]];
      out->row_dual[i] = f.row_class[i] == kLeq ? -d : d;
    }
    for (int i = 0; i < m; i++) out->row_value[i] = 0.0;
    for (int c = 0; c < lp.num_col; c++) {
      const double xv = hx[c];
      for (int q = lp.a_start[c]; q < lp.a_start[c + 1]; q++) out->row_value[lp.a_index[q]] += lp.a_value[q] * xv;
    }
    for (int j = 0; j < f.n_orig; j++) { double v = hsp[j] - hsn[j]; v *= f.sense; out->col_dual[j] = v; }
  }
}

static void solve_hipdlp_on_device(b200pdlp_problem* p, const b200pdlp_lp& lp, const b200pdlp_hipdlp_params& prm, b200pdlp_result* out) {
  NvtxRange nvtx("b200pdlp: solve (HiPDLP mode)");
  using clk = std::chrono::steady_clock;
  set_device(p);
  const auto t_begin = clk::now();
  const StdForm& f = p->form;
  auto& h = p->hip;
  cudaStream_t s = p->stream;
  const int n = p->n, m = p->m;
  const long long launches0 = p->launches;
  const bool shard = hip_sharded(p);
  const int r0 = p->hip_r0, c0 = p->hip_c0;
  CudaEvent evl0, evl1;
  if (!h.graph) {   // steps 2 .. 40 of a block: 38 minor steps and the closing major step (:629-632)
    const long long l0 = p->launches;
    cudaGraph_t g = nullptr;
    CUDA_OK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    for (int i = 2; i <= 39; i++) hip_step(p, i, 0);
    hip_step(p, 40, 1);
    CUDA_OK(cudaStreamEndCapture(s, &g));
    CUDA_OK(cudaGraphInstantiate(&h.graph, g, 0));
    CUDA_OK(cudaGraphDestroy(g));
    h.graph_launches = p->launches - l0;   // counted when replayed
    p->launches = l0;
  }
  if (shard) {
    // On one device a graph upload, a lazy kernel load or an allocation waits for every running kernel, a peer's spinning
    // barrier included (DESIGN section 5): all of them happen before any rank launches its first barrier.  The kernels
    // were loaded when the ranks were linked; the initial-point kernel and the copy / fill operations are loaded here by
    // running them once.
    CUDA_OK(cudaGraphUpload(h.graph, s));
    launch_hip_init_point(s, n, p->lower.p, p->upper.p, h.x.p, h.xa.p);
    CUDA_OK(cudaMemsetAsync(h.dy.p, 0, (size_t)std::max(m, 1) * sizeof(double), s));
    CUDA_OK(cudaMemcpyAsync(h.dy.p, h.ry.p, (size_t)std::max(m, 1) * sizeof(double), cudaMemcpyDeviceToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));
    p->group->arrive_and_wait();
  }
  // PDLPSolver::powerMethod (pdhg.cc:1529-1671) on the device: 20 iterations of q <- A A'q / |A A'q| from the ones vector,
  // lambda = |A'q|^2; no host round trip inside (the norm stays on the device), one read-back at the end.  Several GPUs:
  // every rank holds q and z whole, forms its columns of w and its rows of z, and gathers them; the norms are then the
  // one-GPU sums over full vectors.
  double op_norm_sq = 1.0;
  if (n > 0 && m > 0) {
    double* xq = h.dy.p;      // m-vectors: q (dy), z (axp); n-vector: w = A'q (atdy)
    double* zq = h.axp.p;
    double* wq = h.atdy.p;
    // several GPUs: A'z goes to a second buffer, so that a rank's next A'q cannot overwrite a peer's A'z while that peer
    // still sums it (no barrier lies between the two)
    const HipVec wzv = shard ? &HipBufs::atyp : &HipBufs::atdy;
    double* wz = (h.*wzv).p;
    double* sc = p->outs.p + 16;
    launch_fill(s, m, xq, 1.0);
    for (int it = 0; it < 20; it++) {
      launch_spmv_plain(s, p->AT.dev, xq, wq + c0);
      if (shard) { hip_gather(p, true, {&HipBufs::atdy}); hip_barrier(p); }
      launch_spmv_plain(s, p->A.dev, wq, zq + r0);
      if (shard) { hip_gather(p, false, {&HipBufs::axp}); hip_barrier(p); }
      launch_hip_dot(s, m, zq, zq, p->ordered ? 1 : 0, p->rs(kSlotChk, m), sc);
      launch_hip_div_norm(s, m, zq, sc);
      launch_spmv_plain(s, p->AT.dev, zq, wz + c0);
      if (shard) { hip_gather(p, true, {wzv}); hip_barrier(p); }
      launch_hip_dot(s, n, wz, wz, p->ordered ? 1 : 0, p->rs(kSlotChk, n), sc + 1);
      CUDA_OK(cudaMemcpyAsync(xq, zq, (size_t)m * sizeof(double), cudaMemcpyDeviceToDevice, s));
      p->launches += 6;
    }
    CUDA_OK(cudaMemcpyAsync(p->houts + 16, sc + 1, sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    op_norm_sq = p->houts[16];
  }
  HipController ctl;   // step sizes, fixed-point error, convergence test, restart criteria, PID weight (host_prep_hipdlp.cpp)
  ctl.init(f.norm_cost, f.norm_rhs, op_norm_sq, prm.tolerance, prm.step_size_strategy);
  // x = xa = proj_[l,u](0) (a kernel on the device-order bounds, upper first, then lower), y = ya = 0; A'y (:512-552)
  {
    launch_hip_init_point(s, n, p->lower.p, p->upper.p, h.x.p, h.xa.p);
    CUDA_OK(cudaMemsetAsync(h.y.p, 0, (size_t)std::max(m, 1) * sizeof(double), s));
    CUDA_OK(cudaMemsetAsync(h.ya.p, 0, (size_t)std::max(m, 1) * sizeof(double), s));
    for (DevBuf<double>* b : {&h.xn, &h.rx, &h.hslack, &h.sp, &h.sn, &h.atdy}) CUDA_OK(cudaMemsetAsync(b->p, 0, (size_t)std::max(n, 1) * sizeof(double), s));
    for (DevBuf<double>* b : {&h.yn, &h.ry, &h.dy}) CUDA_OK(cudaMemsetAsync(b->p, 0, (size_t)std::max(m, 1) * sizeof(double), s));
    launch_spmv_plain(s, p->AT.dev, h.y.p, h.aty.p + c0);
    CUDA_OK(cudaStreamSynchronize(s));
    if (shard) p->group->arrive_and_wait();   // nobody gathers into a peer's vectors before that peer has set them
  }
  auto push_state = [&]() {
    h.hstate->primal_step = ctl.primal_step; h.hstate->dual_step = ctl.dual_step; h.hstate->halpern_iteration = ctl.halpern_iteration;
    CUDA_OK(cudaMemcpyAsync(h.state.p, h.hstate, sizeof(HipState), cudaMemcpyHostToDevice, s));
  };
  const double t_lim = (prm.time_limit >= 0 && std::isfinite(prm.time_limit)) ? prm.time_limit : -1.0;   // < 0: none
  int term = B200PDLP_TIMELIMIT_OR_ITERLIMIT;
  bool converged = false, timed_out = false;
  const auto t_loop = clk::now();
  CUDA_OK(cudaEventRecord(evl0, s));
  hip_check(p, 0);   // iteration 0 (:566-572)
  const double* sol_x = h.x.p;
  const double* sol_y = h.y.p;
  if (ctl.converged(p->houts)) { converged = true; }
  else {
    while (ctl.iters < prm.iter_limit) {
      bool over = t_lim >= 0 && std::chrono::duration<double>(clk::now() - t_loop).count() > t_lim;
      if (shard) over = p->group->arrive_and_wait(p->rank, over);   // rank 0's clock decides for every rank
      if (over) { timed_out = true; break; }
      push_state();
      hip_step(p, 1, 1);
      if (ctl.pending_restart_fpe) {   // the restart's reference fixed-point error is that of the first step after it (:600-608)
        hip_check(p, 1);
        ctl.restart_reference(p->houts);
      }
      CUDA_OK(cudaGraphLaunch(h.graph, s));
      p->launches += h.graph_launches;
      hip_check(p, 1);
      const bool restart = ctl.after_block(p->houts);
      if (prm.log_level >= 2)
        printf("[b200pdlp hipdlp] it %8d  pobj %+.8e dobj %+.8e  pfeas %.2e dfeas %.2e  fpe %.3e  weight %.3e\n", ctl.iters,
               ctl.pobj, ctl.dobj, ctl.pfeas, ctl.dfeas, ctl.fpe, ctl.primal_weight);
      if (ctl.pfeas < ctl.tol * (1.0 + f.norm_rhs) && ctl.dfeas < ctl.tol * (1.0 + f.norm_cost) && ctl.relgap < ctl.tol) {
        converged = true; sol_x = h.xn.p; sol_y = h.yn.p; break;
      }
      if (restart) {   // anchors and iterates <- the PDHG iterate of the last major step (:664-688)
        // (several GPUs: xn and yn were gathered by the check, so every rank copies them whole and holds full anchors)
        CUDA_OK(cudaMemcpyAsync(h.xa.p, h.xn.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s));
        CUDA_OK(cudaMemcpyAsync(h.ya.p, h.yn.p, (size_t)std::max(m, 1) * sizeof(double), cudaMemcpyDeviceToDevice, s));
        CUDA_OK(cudaMemcpyAsync(h.x.p, h.xn.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s));
        CUDA_OK(cudaMemcpyAsync(h.y.p, h.yn.p, (size_t)std::max(m, 1) * sizeof(double), cudaMemcpyDeviceToDevice, s));
        launch_spmv_plain(s, p->AT.dev, h.y.p, h.aty.p + c0);
        p->launches++;
      }
    }
  }
  const int iters = ctl.iters, restarts = ctl.restarts;
  const double pfeas = ctl.pfeas, dfeas = ctl.dfeas, pobj = ctl.pobj, dobj = ctl.dobj, relgap = ctl.relgap;
  if (converged) term = B200PDLP_OPTIMAL;
  CUDA_OK(cudaEventRecord(evl1, s));
  CUDA_OK(cudaEventSynchronize(evl1));
  // the postsolve's pageable copies wait for every kernel of the context: no barrier kernel may still be in flight
  if (shard) p->group->arrive_and_wait();
  float loop_ms = 0.f;
  CUDA_OK(cudaEventElapsedTime(&loop_ms, evl0, evl1));
  out->loop_device_ms = loop_ms;
  out->iter_device_ms = loop_ms;
  const double solve_seconds = std::chrono::duration<double>(clk::now() - t_loop).count();
  // unscaleSolution + postprocess (pdhg.cc:1883-1897, :359-492): the iterate is copied out ONLY on convergence --
  // an iteration-limited run returns x = y = 0, like the reference
  // (several GPUs: rank 0 holds the whole iterate and slacks after the final check; the other ranks return no vectors)
  if (p->dev_form && p->rank == 0) {
    // on the device (launch_hip_postsolve), one download of the four original-order vectors
    const int n0 = f.n_orig;
    double* cv = p->io_col.p;
    double* cd = cv + std::max(n0, 1);
    double* rv = p->io_row.p;
    double* rd = rv + std::max(m, 1);
    launch_hip_postsolve(s, p->prep.arr, f.sense, converged ? 1 : 0, f.scaled ? 1 : 0, sol_x, sol_y, h.sp.p, h.sn.p, p->colscale.p,
                         p->rowscale.p, cv, cd, rv, rd);
    CUDA_OK(cudaGetLastError());
    if (out->col_value && out->col_dual && out->row_value && out->row_dual) {
      auto dn = [&](double* dst, const double* src, int len) {
        if (len > 0) CUDA_OK(cudaMemcpyAsync(dst, src, (size_t)len * sizeof(double), cudaMemcpyDeviceToHost, s));
      };
      dn(out->col_value, cv, n0); dn(out->col_dual, cd, n0); dn(out->row_value, rv, m); dn(out->row_dual, rd, m);
    }
    CUDA_OK(cudaStreamSynchronize(s));
  } else if (!p->dev_form && p->rank == 0) {
    // one download of the device-order vectors, then the host postsolve
    std::vector<double> dx, dy, dsp, dsn;
    auto down = [&](const double* d, std::vector<double>& v, int len) {
      v.resize(std::max(len, 1));
      if (len > 0) CUDA_OK(cudaMemcpyAsync(v.data(), d, (size_t)len * sizeof(double), cudaMemcpyDeviceToHost, s));
    };
    if (converged) { down(sol_x, dx, n); down(sol_y, dy, m); }
    down(h.sp.p, dsp, n); down(h.sn.p, dsn, n);
    CUDA_OK(cudaStreamSynchronize(s));
    hip_host_postsolve(lp, f, p->cperm.data(), p->rperm.data(), converged ? dx.data() : nullptr,
                       converged ? dy.data() : nullptr, dsp.data(), dsn.data(), out);
  }
  if (getenv("B200PDLP_TIMING"))
    fprintf(stderr, "[b200pdlp solve] postsolve (%s) %8.3f ms\n", p->dev_form ? "device" : "host",
            std::chrono::duration<double, std::milli>(clk::now() - t_loop).count() - 1e3 * solve_seconds);
  out->value_valid = 1; out->dual_valid = 1;
  out->term_code = term;
  out->term_iterate = timed_out ? 2 : 0;   // 2: the time limit, not the iteration limit, ended the run
  out->iters = iters; out->passes = iters; out->restarts = restarts;
  out->kernel_launches = (int)std::min<long long>(p->launches - launches0, 2147483647LL);
  out->primal_obj = pobj; out->dual_obj = dobj; out->primal_feas = pfeas; out->dual_feas = dfeas;
  out->gap = pobj - dobj; out->rel_gap = relgap;
  out->solve_seconds = solve_seconds;
  out->setup_seconds += std::chrono::duration<double>(t_loop - t_begin).count();
  out->form_cols = n; out->form_rows = m; out->form_nnz = f.nnz; out->form_neq = f.neq;
}

}  // namespace b200

// ============================================================================ C ABI
template <class F>
static int guarded(F&& fn) {
  try {
    fn();
    return B200PDLP_OK;
  } catch (const b200::Error& e) {
    g_last_error = e.what();
    return e.code;
  } catch (const std::bad_alloc&) {
    g_last_error = "host allocation failed";
    return B200PDLP_ERR_ALLOC;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    return B200PDLP_ERR_STATE;
  }
}

// fn(i) for i < count, one host thread each.  After every thread has joined, the first failure is rethrown with its code
// and "<label> <id>: " before its message (id = ids[i], or i).
template <class F>
static void run_per_rank(int count, const char* label, F&& fn, const int* ids = nullptr) {
  std::vector<int> codes((size_t)count, B200PDLP_OK);
  std::vector<std::string> msgs((size_t)count);
  std::vector<std::thread> th;
  for (int i = 0; i < count; i++)
    th.emplace_back([&, i] {
      codes[i] = guarded([&] { fn(i); });
      if (codes[i] != B200PDLP_OK) msgs[i] = g_last_error;   // thread-local: hand it to the caller's thread
    });
  for (auto& t : th) t.join();
  for (int i = 0; i < count; i++)
    if (codes[i] != B200PDLP_OK) throw Error(codes[i], std::string(label) + " " + std::to_string(ids ? ids[i] : i) + ": " + msgs[i]);
}

// owning handle of a problem: deleted with its own device selected
struct ProblemDeleter {
  void operator()(b200pdlp_problem* p) const { cudaSetDevice(p->device); delete p; }
};
using ProblemPtr = std::unique_ptr<b200pdlp_problem, ProblemDeleter>;

static void check_params(const b200pdlp_params& prm) {
  if (prm.device_scaling != 0 && prm.device_scaling != -1)
    throw Error(B200PDLP_ERR_ARG, "b200pdlp: params.device_scaling must be 0 (default) or -1 (host prologue)");
}

// what check_lp checks without reading an array: the sizes, and the arrays the sizes call for are present
static bool lp_fields_ok(const b200pdlp_lp* lp) {
  return lp && lp->num_col >= 0 && lp->num_row >= 0 && lp->a_start && (lp->num_col == 0 || (lp->col_cost && lp->col_lower && lp->col_upper)) &&
         (lp->num_row == 0 || (lp->row_lower && lp->row_upper));
}

// deep: also the O(n) / O(nnz) validation of a_start and a_index (the device prologue does both in its first sweep)
static void check_lp(const b200pdlp_lp* lp, bool deep = true) {
  if (!lp_fields_ok(lp) || (lp->a_start[lp->num_col] > 0 && (!lp->a_index || !lp->a_value)))
    throw Error(B200PDLP_ERR_ARG, "b200pdlp: malformed b200pdlp_lp");
  if (lp->sense != 1.0 && lp->sense != -1.0) throw Error(B200PDLP_ERR_ARG, "b200pdlp: sense must be +1 or -1");
  // formulate() indexes per-row arrays with a_index and walks a_start: validate both once (O(nnz), a few ms at 8M nonzeros)
  if (lp->a_start[0] != 0 || lp->a_start[lp->num_col] < 0) throw Error(B200PDLP_ERR_ARG, "b200pdlp: a_start[0] must be 0 and a_start[num_col] >= 0");
  if (!deep) return;
  for (int j = 0; j < lp->num_col; j++)
    if (lp->a_start[j + 1] < lp->a_start[j]) throw Error(B200PDLP_ERR_ARG, "b200pdlp: a_start must be non-decreasing");
  const int nnz = lp->a_start[lp->num_col], m = lp->num_row;
  unsigned bad = 0;
  for (int q = 0; q < nnz; q++) bad |= (unsigned)lp->a_index[q] >= (unsigned)m;
  if (bad) throw Error(B200PDLP_ERR_ARG, "b200pdlp: a_index entry outside [0, num_row)");
}

// the public entry points select the problem's device; the caller's current device is restored on every exit path
struct DeviceGuard {
  int prev = -1;
  DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; cudaGetLastError(); } }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// b200pdlp_solve_hipdlp_multi's device prologue: one host thread per distinct device in `dev` runs the block-mode prologue
// for the ranks on that device and creates their problems (probs[g], already allocated).  Every thread is joined, and its
// device idle, before this returns: on one device an allocation or a lazy module load of a prologue would otherwise wait
// behind a peer's spinning barrier (DESIGN section 5).
static void create_hipdlp_shards_device(const b200pdlp_lp& lp, const b200pdlp_hipdlp_params& prm, const std::vector<int>& dev,
                                        std::vector<b200pdlp_problem*>& probs) {
  const int world = (int)dev.size();
  std::vector<int> devices;   // distinct, in the order of their first rank
  for (int d : dev)
    if (std::find(devices.begin(), devices.end(), d) == devices.end()) devices.push_back(d);
  run_per_rank((int)devices.size(), "device", [&](int i) {
    std::vector<int> ranks;
    for (int g = 0; g < world; g++)
      if (dev[g] == devices[i]) ranks.push_back(g);
    CUDA_OK(cudaSetDevice(devices[i]));
    TempPrologue T;
    run_hipdlp_shard_prologue(lp, prm.scaling_mode, prm.ruiz_iterations, world, ranks, T);
    for (size_t k = 0; k < ranks.size(); k++) create_problem_hipdlp_shard_device(lp, T, (int)k, probs[ranks[k]]);
    if (ranks[0] == 0) hand_over_postsolve_maps(T, probs[0]);
    CUDA_OK(cudaDeviceSynchronize());
  }, devices.data());   // (T has released the standard form, the orderings and the other temporaries of this device)
}

// ====================================================================================== batch of small LPs, one GPU
// b200pdlp_solve_batch: every member is an ordered-mode problem, solved by one CTA of batch_round_kernel (batch_kernels.cu).
// The host runs each member's prologue (formulate, scale, build_layout with identity orderings) on its threads, packs every
// member into a few pooled buffers, then drives ROUNDS: one launch, one read-back of the control blocks and states, the
// decisions of every member that checked (the same functions solve_on_device calls), one upload.  Each member returns the
// bits b200pdlp_solve returns for it alone.

// fn(i) for i < count on up to one host thread per core; after all have run, the failure of the lowest index is rethrown
// with "member i: " before its message
template <class F>
static void for_members(int count, F&& fn) {
  std::vector<int> codes((size_t)count, B200PDLP_OK);
  std::vector<std::string> msgs((size_t)count);
  std::atomic<int> next{0};
  auto work = [&] {
    for (int i; (i = next++) < count;) {
      codes[i] = guarded([&] { fn(i); });
      if (codes[i] != B200PDLP_OK) msgs[i] = g_last_error;
    }
  };
  const int T = std::max(1, std::min<int>(count, (int)std::thread::hardware_concurrency()));
  std::vector<std::thread> th;
  for (int t = 1; t < T; t++) th.emplace_back(work);
  work();
  for (auto& t : th) t.join();
  for (int i = 0; i < count; i++)
    if (codes[i] != B200PDLP_OK) throw Error(codes[i], "member " + std::to_string(i) + ": " + msgs[i]);
}

// a batch member's standard form must be an ordered-mode problem (max(n, m) <= ordered_max): checked before any device work
static void check_batch_member(const b200pdlp_lp* lp, const b200pdlp_params& prm, int i) {
  const int rc = guarded([&] {
    check_lp(lp);
    const int omax = prm.ordered_max == 0 ? 4096 : prm.ordered_max;
    if (omax < 0) throw Error(B200PDLP_ERR_ARG, "ordered_max < 0: a batch solves ordered-mode problems only");
    const int n = std_form_cols(*lp, 1e20);
    if (std::max(n, lp->num_row) > omax)
      throw Error(B200PDLP_ERR_ARG, "standard form " + std::to_string(lp->num_row) + " x " + std::to_string(n) +
                                        " exceeds ordered_max = " + std::to_string(omax));
  });
  if (rc != B200PDLP_OK) throw Error(rc, "b200pdlp_solve_batch: member " + std::to_string(i) + ": " + g_last_error);
}

struct BatchRun {   // one member's host control over the rounds
  StdForm f;        // b200pdlp_solve_batch_device fills the scalars only: dimensions, sense, offset, norms, amax
  double cost_sq = 0.0, rhs_sq = 0.0;   // |c|^2 and |b|^2 of the scaled form, index order: what sets beta
  RestartMemo memo;
  CheckResult chk;
  int term = B200PDLP_TIMELIMIT_OR_ITERLIMIT, term_iterate = 0, restarts = 0;
  bool have_check = false;
  double tol_p = 0.0, tol_d = 0.0;
};

struct BatchHost : BatchRun {   // one member of b200pdlp_solve_batch on the host
  HostLayout L;
  std::vector<double> x0, y0;
  size_t vec = 0, sl_a = 0, sl_at = 0, e_a = 0, e_at = 0;   // offsets in the pools
};

// pinned host array, returned to the pinned cache
template <class T>
struct PinnedArray {
  T* p = nullptr;
  explicit PinnedArray(size_t count) { p = static_cast<T*>(pinned_cache_alloc(std::max<size_t>(count, 1) * sizeof(T), false)); }
  ~PinnedArray() { if (p) pinned_cache_free(p); }
  PinnedArray(const PinnedArray&) = delete;
  PinnedArray& operator=(const PinnedArray&) = delete;
};

struct StreamHolder {
  cudaStream_t s = nullptr;
  StreamHolder() { CUDA_OK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); }
  ~StreamHolder() { if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); } }
  StreamHolder(const StreamHolder&) = delete;
  StreamHolder& operator=(const StreamHolder&) = delete;
};

// doubles of a member's vector block: cost, lower, upper, colscale, then x0 x1 aty0 aty1 xsum xavg atyavg xlr (n each);
// rhs, rowscale, then y0 y1 ax0 ax1 ysum yavg axavg ylr (m each)
static size_t batch_vec_len(int n, int m) { return (size_t)12 * n + (size_t)10 * m; }

// doubles of a HiPDLP member's vector block: cost, lower, upper, colscale, then x xa xn rx aty hslack atyp atdy sp sn (n each);
// rlo, rup, rowscale, then y ya yn ry axp dy (m each)
static size_t hip_batch_vec_len(int n, int m) { return (size_t)14 * n + (size_t)9 * m; }

// the vectors of a member's block `v` (batch_vec_len) as BatchMember pointers
static void batch_member_vectors(BatchMember& M, double* v, int n, int m) {
  double* w = v + 12 * (size_t)n;
  M.n = n; M.m = m;
  M.cost = v; M.lower = v + n; M.upper = v + 2 * n; M.colscale = v + 3 * n;
  M.x0 = v + 4 * n; M.x1 = v + 5 * n; M.aty0 = v + 6 * n; M.aty1 = v + 7 * n;
  M.xsum = v + 8 * n; M.xavg = v + 9 * n; M.atyavg = v + 10 * n; M.xlr = v + 11 * n;
  M.rhs = w; M.rowscale = w + m;
  M.y0 = w + 2 * m; M.y1 = w + 3 * m; M.ax0 = w + 4 * m; M.ax1 = w + 5 * m;
  M.ysum = w + 6 * m; M.yavg = w + 7 * m; M.axavg = w + 8 * m; M.ylr = w + 9 * m;
}

struct BatchLoop {
  std::chrono::steady_clock::time_point t_loop;   // the start of the rounds (the time limit counts from here)
  long long rounds = 0;
  double iter_ms = 0.0, solve_seconds = 0.0;
  float loop_ms = 0.f;
};

// The rounds of a batch, for both entry points: each member's initial state from its form's scalars, then per round one
// upload of the control blocks and states, one launch, one read-back and the decisions of every member that checked (the
// functions solve_on_device calls), until no member is active.  hst: `count` pinned states, the final ones on return.
static BatchLoop batch_rounds(cudaStream_t s, int count, const b200pdlp_params& prm, const BatchMember* dmem,
                              const std::vector<BatchRun*>& R, PdhgState* hst, b200pdlp_result* outs) {
  using clk = std::chrono::steady_clock;
  // ---- initial states: PDHG_Init_Step_Sizes (cupdlp_step.c:312-375); a fixed step takes tau, sigma after round 0's power method
  PinnedArray<BatchCtl> hctl((size_t)count);
  for (int i = 0; i < count; i++) {
    const BatchRun& r = *R[i];
    PdhgState* h = hst + i;
    memset(h, 0, sizeof(PdhgState));
    h->adaptive = prm.adaptive_step != 0;
    const double a = r.cost_sq, b = r.rhs_sq;
    h->beta = std::fmin(a, b) > 1e-6 ? a / b : 1.0;
    if (h->adaptive) {
      h->tau = (1.0 / r.f.amax) / std::sqrt(h->beta);
      h->sigma = h->tau * h->beta;
    }
    arm_step(h);
    fill_pow_tables(h);
    h->stop_iter = 0;   // the first check is due at once (iteration 0)
    BatchCtl& c = hctl.p[i];
    memset(&c, 0, sizeof(BatchCtl));
    c.active = 1; c.first = 1; c.fixed_step = !h->adaptive; c.no_check = prm.iter_limit <= 0;
    outs[i].trace_len = 0;
  }
  DevBuf<PdhgState> dst;
  DevBuf<BatchCtl> dctl;
  dst.alloc(count, false); dctl.alloc(count, false);

  const int interval = prm.check_interval > 0 ? prm.check_interval : 40;
  const double t_lim = (prm.time_limit >= 0 && std::isfinite(prm.time_limit)) ? prm.time_limit : -1.0;   // < 0: none
  CudaEvent evl0, evl1, ev0, ev1;
  BatchLoop L;
  int active = count;
  CUDA_OK(cudaEventRecord(evl0, s));
  L.t_loop = clk::now();
  while (active > 0) {
    NvtxRange nvtx("b200pdlp: batch round");
    const bool timed_out = t_lim >= 0 && std::chrono::duration<double>(clk::now() - L.t_loop).count() > t_lim;
    CUDA_OK(cudaMemcpyAsync(dctl.p, hctl.p, (size_t)count * sizeof(BatchCtl), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaMemcpyAsync(dst.p, hst, (size_t)count * sizeof(PdhgState), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaEventRecord(ev0, s));
    launch_batch_round(s, count, dmem, dst.p, dctl.p);
    CUDA_OK(cudaEventRecord(ev1, s));
    CUDA_OK(cudaMemcpyAsync(hctl.p, dctl.p, (size_t)count * sizeof(BatchCtl), cudaMemcpyDeviceToHost, s));
    // the scalars of every state (the power tables are the host's own)
    CUDA_OK(cudaMemcpy2DAsync(hst, sizeof(PdhgState), dst.p, sizeof(PdhgState), offsetof(PdhgState, pow_red), count,
                              cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    float ms = 0.f;
    CUDA_OK(cudaEventElapsedTime(&ms, ev0, ev1));
    L.iter_ms += ms;
    const bool first = L.rounds == 0;
    L.rounds++;
    for (int i = 0; i < count; i++) {
      BatchCtl& c = hctl.p[i];
      if (!c.active) continue;
      BatchRun& b = *R[i];
      PdhgState* h = hst + i;
      b200pdlp_result* out = outs + i;
      if (!c.checked) {
        if (first && c.no_check) { c.active = 0; active--; continue; }   // iter_limit <= 0: no check at all
        fill_pow_tables(h);   // the tables ran out before the check iteration: refill, the next round goes on
        continue;
      }
      if (first && c.fixed_step) {
        const double lambda = c.outs[kBatchLambda];
        h->tau = 0.8 / std::sqrt(lambda);
        h->sigma = h->tau;
        h->tau /= std::sqrt(h->beta);
        h->sigma *= std::sqrt(h->beta);
        arm_step(h);
      }
      CheckResult& chk = b.chk;
      double dscale[2], pscale[2];
      assemble_check_a(b.f, c.outs, chk, dscale, pscale);
      assemble_check_b(b.f, c.outs, chk, dscale, pscale);
      chk.timed_out = timed_out;
      b.have_check = true;
      int choice = 0;
      const int t_code = check_decision(prm, b.tol_p, b.tol_d, h, chk, b.memo, &b.term_iterate, &choice);
      if (t_code >= 0) {
        b.term = t_code;
        trace_row(out, h, chk, 0);
        c.active = 0;
        active--;
        continue;
      }
      if (choice) {
        restart_steps(h, choice, chk, b.memo, c.outs[choice == 1 ? kBatchDxAvg : kBatchDxCur],
                      c.outs[choice == 1 ? kBatchDyAvg : kBatchDyCur]);
        b.restarts++;
        arm_step(h);
        c.restart = choice;
      }
      trace_row(out, h, chk, choice);
      h->stop_iter = next_check_iter(h->iter, interval, prm.iter_limit);
      fill_pow_tables(h);
    }
  }
  CUDA_OK(cudaEventRecord(evl1, s));
  CUDA_OK(cudaEventSynchronize(evl1));
  CUDA_OK(cudaEventElapsedTime(&L.loop_ms, evl0, evl1));
  L.solve_seconds = std::chrono::duration<double>(clk::now() - L.t_loop).count();
  return L;
}

// the per-member fields of a batch result besides the vectors; the timings and kernel_launches are the batch's
static void batch_result(b200pdlp_result* out, const BatchRun& b, const PdhgState* h, const BatchLoop& L, double setup_seconds) {
  fill_result(out, b.f, h, b.term, b.term_iterate, b.restarts, b.chk);
  out->kernel_launches = (int)std::min<long long>(L.rounds, 2147483647LL);
  out->setup_seconds = setup_seconds;
  out->solve_seconds = L.solve_seconds;
  out->loop_device_ms = L.loop_ms;
  out->iter_device_ms = L.iter_ms;
}

static void solve_batch(int count, const b200pdlp_lp* lps, const b200pdlp_params& prm, const b200pdlp_warm* warms,
                        b200pdlp_result* outs) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  Laps lap;
  device_count_checked();
  if (prm.device >= 0) CUDA_OK(cudaSetDevice(prm.device));
  StreamHolder sh;
  cudaStream_t s = sh.s;
  std::vector<BatchHost> B((size_t)count);
  {
    NvtxRange nvtx("b200pdlp: batch prologue (host threads)");
    for_members(count, [&](int i) {
      BatchHost& b = B[i];
      formulate(lps[i], b.f);
      scale(b.f, prm.scaling != 0);
      build_layout(b.f, 0, 1, prm.ordered_max, b.L);
      if (!b.L.ordered || !b.L.A.segs.empty() || !b.L.AT.segs.empty())
        throw Error(B200PDLP_ERR_STATE, "the layout is not an ordered-mode layout");
      host_start_point(b.f, warms ? &warms[i] : nullptr, b.x0, b.y0);
      b.tol_p = prm.tol_primal * (1.0 + b.f.norm_rhs);
      b.tol_d = prm.tol_dual * (1.0 + b.f.norm_cost);
      for (int j = 0; j < b.f.n; j++) b.cost_sq += b.f.cost[j] * b.f.cost[j];
      for (int r = 0; r < b.f.m; r++) b.rhs_sq += b.f.rhs[r] * b.f.rhs[r];
    });
  }
  lap("batch", "prologue (host threads)");

  // ---- pooled device buffers: vectors, slice descriptors, column ids and values of A and A'; one descriptor per member
  size_t nvec = 0, nsl = 0, nent = 0;
  for (BatchHost& b : B) {
    b.vec = nvec; nvec += batch_vec_len(b.f.n, b.f.m);
    b.sl_a = nsl; nsl += b.L.A.slices.size();
    b.sl_at = nsl; nsl += b.L.AT.slices.size();
    b.e_a = nent; nent += b.L.A.col.size();
    b.e_at = nent; nent += b.L.AT.col.size();
  }
  std::vector<double> hvec(std::max<size_t>(nvec, 1), 0.0), hval(std::max<size_t>(nent, 1), 0.0);
  std::vector<int> hcol(std::max<size_t>(nent, 1), 0);
  std::vector<int4> hsl(std::max<size_t>(nsl, 1));
  for_members(count, [&](int i) {
    const BatchHost& b = B[i];
    const StdForm& f = b.f;
    const int n = f.n, m = f.m;
    double* v = hvec.data() + b.vec;
    // identity orderings (ordered mode): standard-form order is device order
    std::copy(f.cost.begin(), f.cost.end(), v);
    std::copy(f.lower.begin(), f.lower.end(), v + n);
    std::copy(f.upper.begin(), f.upper.end(), v + 2 * n);
    std::copy(f.col_scale.begin(), f.col_scale.end(), v + 3 * n);
    std::copy(b.x0.begin(), b.x0.end(), v + 4 * n);
    for (int j = 0; j < n; j++) v[8 * n + j] = proj_zero(f, j);   // xsum
    double* w = v + 12 * n;
    std::copy(f.rhs.begin(), f.rhs.end(), w);
    std::copy(f.row_scale.begin(), f.row_scale.end(), w + m);
    std::copy(b.y0.begin(), b.y0.end(), w + 2 * m);
    static_assert(sizeof(SellMatrix::Slice) == sizeof(int4), "descriptor layout");
    memcpy(hsl.data() + b.sl_a, b.L.A.slices.data(), b.L.A.slices.size() * sizeof(int4));
    memcpy(hsl.data() + b.sl_at, b.L.AT.slices.data(), b.L.AT.slices.size() * sizeof(int4));
    std::copy(b.L.A.col.begin(), b.L.A.col.end(), hcol.begin() + b.e_a);
    std::copy(b.L.AT.col.begin(), b.L.AT.col.end(), hcol.begin() + b.e_at);
    std::copy(b.L.A.val.begin(), b.L.A.val.end(), hval.begin() + b.e_a);
    std::copy(b.L.AT.val.begin(), b.L.AT.val.end(), hval.begin() + b.e_at);
  });
  DevBuf<double> dvec, dval;
  DevBuf<int> dcol;
  DevBuf<int4> dsl;
  DevBuf<BatchMember> dmem;
  dvec.alloc(hvec.size(), false); dval.alloc(hval.size(), false); dcol.alloc(hcol.size(), false); dsl.alloc(hsl.size(), false);
  dmem.alloc(count, false);
  std::vector<BatchMember> hmem((size_t)count);
  for (int i = 0; i < count; i++) {
    const BatchHost& b = B[i];
    BatchMember& M = hmem[i];
    batch_member_vectors(M, dvec.p + b.vec, b.f.n, b.f.m);
    M.neq = b.L.neq_local;
    M.a_slices = dsl.p + b.sl_a; M.a_col = dcol.p + b.e_a; M.a_val = dval.p + b.e_a;
    M.at_slices = dsl.p + b.sl_at; M.at_col = dcol.p + b.e_at; M.at_val = dval.p + b.e_at;
  }
  CUDA_OK(cudaMemcpyAsync(dvec.p, hvec.data(), hvec.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(dval.p, hval.data(), hval.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(dcol.p, hcol.data(), hcol.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(dsl.p, hsl.data(), hsl.size() * sizeof(int4), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(dmem.p, hmem.data(), (size_t)count * sizeof(BatchMember), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaStreamSynchronize(s));
  lap("batch", "pools + upload");

  std::vector<BatchRun*> R((size_t)count);
  for (int i = 0; i < count; i++) R[i] = &B[i];
  PinnedArray<PdhgState> hst((size_t)count);
  const BatchLoop loop = batch_rounds(s, count, prm, dmem.p, R, hst.p, outs);
  lap("batch", "rounds");

  // ---- PDHG_PostSolve of every member, on the host
  NvtxRange nvtx_post("b200pdlp: batch postsolve + download");
  CUDA_OK(cudaMemcpyAsync(hvec.data(), dvec.p, hvec.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  const double setup_seconds = std::chrono::duration<double>(loop.t_loop - t_begin).count();
  for_members(count, [&](int i) {
    BatchHost& b = B[i];
    const StdForm& f = b.f;
    const PdhgState* h = hst.p + i;
    const int n = f.n, m = f.m, cur = h->cur;
    const bool use_avg = b.term == B200PDLP_OPTIMAL && b.term_iterate == 1;
    const double* v = hvec.data() + b.vec;
    const double* w = v + 12 * n;
    const double* dx = use_avg ? v + 9 * n : v + (4 + cur) * n;
    const double* daty = use_avg ? v + 10 * n : v + (6 + cur) * n;
    const double* dy = use_avg ? w + 7 * m : w + (2 + cur) * m;
    const double* dax = use_avg ? w + 8 * m : w + (4 + cur) * m;
    std::vector<double> hx(n), hy(m), hax(m), haty(n);
    for (int j = 0; j < n; j++) { hx[b.L.cperm[j]] = dx[j]; haty[b.L.cperm[j]] = daty[j]; }
    for (int r = 0; r < m; r++) { hy[b.L.rperm[r]] = dy[r]; hax[b.L.rperm[r]] = dax[r]; }
    b200pdlp_result* out = outs + i;
    host_postsolve(f, b.have_check, hx, hy, hax, haty, out);
    batch_result(out, b, h, loop, setup_seconds);
  });
  lap("batch", "postsolve (host threads)");
}

// ------------------------------------------------------------------------------ batch of small LPs already on the GPU
// b200pdlp_solve_batch_device: every array of every member is device memory.  The prologue and the postsolve run on the
// device, one CTA per member (batch_prep.cu); the rounds are solve_batch's (batch_rounds).  The host reads one sizing record
// and one scalar record per member, never an array, and the members return solve_batch's bits.

// the checks of a member that read no array (the device checks the arrays: batch_size_kernel)
// (both device-pointer batches; who: the entry point, for the message)
static void check_batch_device_member(const b200pdlp_lp* lp, int ordered_max, int i, const char* who) {
  const int rc = guarded([&] {
    if (!lp_fields_ok(lp)) throw Error(B200PDLP_ERR_ARG, "b200pdlp: malformed b200pdlp_lp");
    if (lp->sense != 1.0 && lp->sense != -1.0) throw Error(B200PDLP_ERR_ARG, "b200pdlp: sense must be +1 or -1");
    if (ordered_max < 0) throw Error(B200PDLP_ERR_ARG, "ordered_max < 0: a batch solves ordered-mode problems only");
  });
  if (rc != B200PDLP_OK) throw Error(rc, std::string(who) + ": member " + std::to_string(i) + ": " + g_last_error);
}

// ptr (NULL: not given) must be device or managed memory of `device`
static void check_device_array(const void* ptr, int device, int i, const char* field, const char* who) {
  if (!ptr) return;
  cudaPointerAttributes a{};
  const cudaError_t e = cudaPointerGetAttributes(&a, ptr);
  if (e != cudaSuccess) cudaGetLastError();
  if (e != cudaSuccess || !((a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device))
    throw Error(B200PDLP_ERR_ARG, std::string(who) + ": member " + std::to_string(i) + ": " + field +
                                      " is not device memory of device " + std::to_string(device));
}

// every array pointer of the batch (warms: NULL for none) must be device memory of `device`: the lowest failing member, field
static void check_device_arrays(int count, const b200pdlp_lp* lps, const b200pdlp_warm* warms, const b200pdlp_result* outs,
                                int device, const char* who) {
  for (int i = 0; i < count; i++) {
    const b200pdlp_lp& lp = lps[i];
    check_device_array(lp.a_start, device, i, "a_start", who);
    check_device_array(lp.a_index, device, i, "a_index", who);
    check_device_array(lp.a_value, device, i, "a_value", who);
    check_device_array(lp.col_cost, device, i, "col_cost", who);
    check_device_array(lp.col_lower, device, i, "col_lower", who);
    check_device_array(lp.col_upper, device, i, "col_upper", who);
    check_device_array(lp.row_lower, device, i, "row_lower", who);
    check_device_array(lp.row_upper, device, i, "row_upper", who);
    if (warms) {
      check_device_array(warms[i].col_value, device, i, "warm col_value", who);
      check_device_array(warms[i].row_value, device, i, "warm row_value", who);
      check_device_array(warms[i].row_dual, device, i, "warm row_dual", who);
    }
    check_device_array(outs[i].col_value, device, i, "result col_value", who);
    check_device_array(outs[i].col_dual, device, i, "result col_dual", who);
    check_device_array(outs[i].row_value, device, i, "result row_value", who);
    check_device_array(outs[i].row_dual, device, i, "result row_dual", who);
  }
}

// A device-resident batch after its prologue: the descriptors (pool pointers set), the sizing and scalar records, the pools
struct DeviceBatch {
  std::vector<BatchPrep> hp;
  std::vector<BatchSize> size;
  std::vector<double> rec;   // [count][kPrepRec]
  DevBuf<BatchPrep> prep;
  DevBuf<BatchSize> dsize;
  DevBuf<double> drec;
  DevBuf<int> rows;          // the sizing's row maps and row lengths: 4 m + 1 per member
  DevBuf<int> ints, col;     // the form's index arrays: 3 nnz + n + m + 1 per member; the layouts' column ids
  DevBuf<double> dbls, vec, val;   // the form's values and the scaling factors: nnz + 2 n + m; batch_vec_len; the layouts' values
  DevBuf<int4> slices;
  std::vector<HipBatchPrep> hx;    // HiPDLP members only: their arrays in `ints`
  DevBuf<HipBatchPrep> dhx;
};

// which prologue a device batch runs: formulate + scale (PDLP mode), or formulate_hipdlp + scale_hipdlp (HiPDLP mode)
struct PrepMode {
  bool hip = false;
  int scaling = 0;           // PDLP: b200pdlp_params::scaling; HiPDLP: scaling_mode
  int ruiz_iterations = 0;   // HiPDLP only
};

static const char* prep_error_text(int err) {
  switch (err) {
    case kPrepStart0: return "b200pdlp: a_start[0] must be 0 and a_start[num_col] >= 0";
    case kPrepDecreasing: return "b200pdlp: a_start must be non-decreasing";
    case kPrepIndex: return "b200pdlp: a_index entry outside [0, num_row)";
    default: return "b200pdlp: malformed b200pdlp_lp";
  }
}

// Validation and sizing (one read-back of `count` records), the pools, then the prologue (one read-back of the scalar
// records), on stream s of the current device.  lps[i] / warms[i]: host structs whose arrays are device memory.
static void device_batch_prologue(cudaStream_t s, int count, const b200pdlp_lp* lps, const b200pdlp_warm* warms,
                                  const PrepMode& mode, int ordered_max, const char* who, DeviceBatch& D, Laps& lap) {
  const int omax = ordered_max == 0 ? 4096 : ordered_max;
  D.hp.assign((size_t)count, BatchPrep{});
  size_t nrows = 0;
  for (int i = 0; i < count; i++) nrows += 4 * (size_t)lps[i].num_row + 1;
  D.rows.alloc(nrows, false);
  nrows = 0;
  for (int i = 0; i < count; i++) {
    const b200pdlp_lp& lp = lps[i];
    BatchPrep& P = D.hp[i];
    const int m = lp.num_row;
    P.n0 = lp.num_col; P.m = m; P.sense = lp.sense;
    P.a_start = lp.a_start; P.a_index = lp.a_index; P.a_value = lp.a_value;
    P.col_cost = lp.col_cost; P.col_lower = lp.col_lower; P.col_upper = lp.col_upper;
    P.row_lower = lp.row_lower; P.row_upper = lp.row_upper;
    if (warms && warms[i].col_value && warms[i].row_value && warms[i].row_dual) {
      P.warm_x = warms[i].col_value; P.warm_rv = warms[i].row_value; P.warm_rd = warms[i].row_dual;
    }
    int* q = D.rows.p + nrows;
    P.row_class = q; P.row_new_idx = q + m; P.slack = q + 2 * m; P.rptr = q + 3 * m;
    nrows += 4 * (size_t)m + 1;
  }
  D.prep.alloc(count, false); D.dsize.alloc(count, false); D.drec.alloc((size_t)count * kPrepRec, false);
  CUDA_OK(cudaMemcpyAsync(D.prep.p, D.hp.data(), (size_t)count * sizeof(BatchPrep), cudaMemcpyHostToDevice, s));
  if (mode.hip) launch_hip_batch_size(s, count, D.prep.p, D.dsize.p);
  else launch_batch_size(s, count, D.prep.p, D.dsize.p);
  CUDA_OK(cudaGetLastError());
  D.size.resize((size_t)count);
  CUDA_OK(cudaMemcpyAsync(D.size.data(), D.dsize.p, (size_t)count * sizeof(BatchSize), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  for (int i = 0; i < count; i++) {   // the lowest failing member
    const BatchSize& z = D.size[i];
    const std::string at = std::string(who) + ": member " + std::to_string(i) + ": ";
    if (z.err != kPrepOk) throw Error(B200PDLP_ERR_ARG, at + prep_error_text(z.err));
    if (std::max(z.n, lps[i].num_row) > omax)
      throw Error(B200PDLP_ERR_ARG, at + "standard form " + std::to_string(lps[i].num_row) + " x " + std::to_string(z.n) +
                                        " exceeds ordered_max = " + std::to_string(omax));
    if (z.pad_a >= 2000000000 || z.pad_at >= 2000000000)
      throw Error(B200PDLP_ERR_ARG, at + "b200pdlp: matrix too large for 32-bit slice offsets");
  }
  lap("batch device", "validation + sizing");

  // ---- the pools: each member's slices of them
  size_t ni = 0, nd = 0, nv = 0, nsl = 0, ne = 0;
  for (int i = 0; i < count; i++) {
    const BatchSize& z = D.size[i];
    const size_t n = z.n, m = lps[i].num_row, nnz = z.nnz;
    ni += 3 * nnz + n + m + 1;
    if (mode.hip) ni += m + 1 + (nnz - n) + 2 * (size_t)lps[i].num_col;   // optr, opos (nnz0), sortcols
    nd += nnz + 2 * n + m;
    nv += mode.hip ? hip_batch_vec_len(z.n, lps[i].num_row) : batch_vec_len(z.n, lps[i].num_row);
    nsl += (m + 31) / 32 + (n + 31) / 32;
    ne += (size_t)z.pad_a + 32 + (size_t)z.pad_at + 32;
  }
  D.ints.alloc(ni, false); D.dbls.alloc(nd, false); D.vec.alloc(nv, false); D.slices.alloc(nsl, false);
  D.col.alloc(ne, false); D.val.alloc(ne, false);
  CUDA_OK(cudaMemsetAsync(D.vec.p, 0, std::max<size_t>(nv, 1) * sizeof(double), s));   // the iterates' other halves, sums
  ni = nd = nv = nsl = ne = 0;
  if (mode.hip) D.hx.assign((size_t)count, HipBatchPrep{});
  for (int i = 0; i < count; i++) {
    const BatchSize& z = D.size[i];
    BatchPrep& P = D.hp[i];
    const int n = z.n, m = lps[i].num_row, nnz = z.nnz;
    P.n = n; P.nnz = nnz; P.neq = z.neq;
    int* q = D.ints.p + ni;
    P.cbeg = q; P.cidx = q + n + 1; P.pcol = P.cidx + nnz; P.rpos = P.pcol + nnz; P.rwork = P.rpos + nnz;
    ni += 3 * (size_t)nnz + n + m + 1;
    if (mode.hip) {
      const int n0 = lps[i].num_col;
      HipBatchPrep& X = D.hx[i];
      X.optr = D.ints.p + ni; X.opos = X.optr + m + 1; X.sortcols = X.opos + (nnz - n + n0);
      ni += (size_t)m + 1 + (nnz - n + n0) + n0;
    }
    double* d = D.dbls.p + nd;
    P.cval = d; P.cs = d + nnz; P.cs_next = P.cs + n; P.rs = P.cs_next + n;
    nd += (size_t)nnz + 2 * (size_t)n + m;
    P.vec = D.vec.p + nv;
    nv += mode.hip ? hip_batch_vec_len(n, m) : batch_vec_len(n, m);
    P.a_slices = D.slices.p + nsl; nsl += (m + 31) / 32;
    P.at_slices = D.slices.p + nsl; nsl += (n + 31) / 32;
    P.a_col = D.col.p + ne; P.a_val = D.val.p + ne; ne += (size_t)z.pad_a + 32;
    P.at_col = D.col.p + ne; P.at_val = D.val.p + ne; ne += (size_t)z.pad_at + 32;
    P.rec = D.drec.p + (size_t)kPrepRec * i;
  }
  CUDA_OK(cudaMemcpyAsync(D.prep.p, D.hp.data(), (size_t)count * sizeof(BatchPrep), cudaMemcpyHostToDevice, s));
  D.rec.assign((size_t)count * kPrepRec, 0.0);
  if (mode.hip) {
    D.dhx.alloc(count, false);
    CUDA_OK(cudaMemcpyAsync(D.dhx.p, D.hx.data(), (size_t)count * sizeof(HipBatchPrep), cudaMemcpyHostToDevice, s));
    launch_hip_batch_prep(s, count, D.prep.p, D.dhx.p, mode.scaling, mode.ruiz_iterations);
    CUDA_OK(cudaGetLastError());
    // rec[0..1] of every member: |c|^2 and |b|^2 of the unscaled form
    CUDA_OK(cudaMemcpy2DAsync(D.rec.data(), kPrepRec * sizeof(double), D.drec.p, kPrepRec * sizeof(double), 2 * sizeof(double),
                              count, cudaMemcpyDeviceToHost, s));
  } else {
    launch_batch_prep(s, count, D.prep.p, mode.scaling != 0);
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaMemcpyAsync(D.rec.data(), D.drec.p, D.rec.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  }
  CUDA_OK(cudaStreamSynchronize(s));
  lap("batch device", "prologue (device)");
}

static void solve_batch_device(int count, const b200pdlp_lp* lps, const b200pdlp_params& prm, const b200pdlp_warm* warms,
                               b200pdlp_result* outs) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  Laps lap;
  device_count_checked();
  if (prm.device >= 0) CUDA_OK(cudaSetDevice(prm.device));
  int device = 0;
  CUDA_OK(cudaGetDevice(&device));
  check_device_arrays(count, lps, warms, outs, device, "b200pdlp_solve_batch_device");
  StreamHolder sh;
  cudaStream_t s = sh.s;
  DeviceBatch D;
  {
    NvtxRange nvtx("b200pdlp: batch prologue (device)");
    PrepMode mode;
    mode.scaling = prm.scaling;
    device_batch_prologue(s, count, lps, warms, mode, prm.ordered_max, "b200pdlp_solve_batch_device", D, lap);
  }
  std::vector<BatchRun> runs((size_t)count);
  std::vector<BatchRun*> R((size_t)count);
  std::vector<BatchMember> hmem((size_t)count);
  for (int i = 0; i < count; i++) {
    BatchRun& b = runs[i];
    const BatchPrep& P = D.hp[i];
    const double* r = D.rec.data() + (size_t)kPrepRec * i;
    StdForm& f = b.f;
    f.n = P.n; f.m = P.m; f.nnz = P.nnz; f.neq = P.neq; f.n_orig = P.n0;
    f.sense = lps[i].sense; f.offset = lps[i].offset;
    f.norm_cost = std::sqrt(r[0]); f.norm_rhs = std::sqrt(r[1]); f.amax = r[2];
    b.cost_sq = r[3]; b.rhs_sq = r[4];
    b.tol_p = prm.tol_primal * (1.0 + f.norm_rhs);
    b.tol_d = prm.tol_dual * (1.0 + f.norm_cost);
    R[i] = &b;
    BatchMember& M = hmem[i];
    batch_member_vectors(M, P.vec, P.n, P.m);
    M.neq = P.neq;
    M.a_slices = P.a_slices; M.a_col = P.a_col; M.a_val = P.a_val;
    M.at_slices = P.at_slices; M.at_col = P.at_col; M.at_val = P.at_val;
  }
  DevBuf<BatchMember> dmem;
  dmem.alloc(count, false);
  CUDA_OK(cudaMemcpyAsync(dmem.p, hmem.data(), (size_t)count * sizeof(BatchMember), cudaMemcpyHostToDevice, s));
  PinnedArray<PdhgState> hst((size_t)count);
  const BatchLoop loop = batch_rounds(s, count, prm, dmem.p, R, hst.p, outs);
  lap("batch device", "rounds");

  // ---- PDHG_PostSolve of every member on the device, into the caller's vectors
  NvtxRange nvtx_post("b200pdlp: batch postsolve (device)");
  std::vector<BatchPost> hpost((size_t)count);
  for (int i = 0; i < count; i++) {
    const BatchRun& b = runs[i];
    BatchPost& q = hpost[i];
    q.col_value = outs[i].col_value; q.col_dual = outs[i].col_dual; q.row_value = outs[i].row_value; q.row_dual = outs[i].row_dual;
    q.sel = (b.term == B200PDLP_OPTIMAL && b.term_iterate == 1) ? 2 : hst.p[i].cur;
    q.have_check = b.have_check;
  }
  DevBuf<BatchPost> dpost;
  dpost.alloc(count, false);
  CUDA_OK(cudaMemcpyAsync(dpost.p, hpost.data(), (size_t)count * sizeof(BatchPost), cudaMemcpyHostToDevice, s));
  launch_batch_post(s, count, D.prep.p, dpost.p);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaStreamSynchronize(s));
  const double setup_seconds = std::chrono::duration<double>(loop.t_loop - t_begin).count();
  for (int i = 0; i < count; i++) batch_result(outs + i, runs[i], hst.p + i, loop, setup_seconds);
  lap("batch device", "postsolve (device)");
}

// ---- b200pdlp_debug_batch_prep_compare: the device prologue and postsolve against their host twins
static const int kBatchPrepItems = 27;

template <class T>
static std::vector<T> download_vec(const T* d, size_t count) {
  std::vector<T> h(count);
  if (count) CUDA_OK(cudaMemcpy(h.data(), d, count * sizeof(T), cudaMemcpyDeviceToHost));
  return h;
}
// elements of a[0..count) whose bytes differ from b's
template <class T>
static double bit_mismatches(const T* a, const T* b, size_t count) {
  double k = 0;
  for (size_t i = 0; i < count; i++) k += memcmp(a + i, b + i, sizeof(T)) != 0;
  return k;
}
// a fixed pseudo-random value in [-1, 1) for (member, index)
static double batch_probe(int i, int k) {
  unsigned long long h = (0x9E3779B97F4A7C15ull * (unsigned long long)(i + 1)) ^ (0x94D049BB133111EBull * (unsigned long long)(k + 3));
  h ^= h >> 31; h *= 0xD6E8FEB86659FD93ull; h ^= h >> 32;
  return (double)(h >> 11) * 0x1p-52 - 1.0;
}

// host LPs uploaded as they are: dl[i] is lps[i] with its arrays in ri / rd
struct RawLps {
  DevBuf<int> ri;
  DevBuf<double> rd;
  std::vector<b200pdlp_lp> dl;
};
static void upload_raw_lps(int count, const b200pdlp_lp* lps, RawLps& R) {
  DevBuf<int>& ri = R.ri;
  DevBuf<double>& rd = R.rd;
  std::vector<b200pdlp_lp>& dl = R.dl;
  size_t ni = 0, nd = 0;
  for (int i = 0; i < count; i++) {
    const b200pdlp_lp& lp = lps[i];
    const size_t nnz = lp.a_start[lp.num_col];
    ni += lp.num_col + 1 + nnz;
    nd += nnz + 3 * (size_t)lp.num_col + 2 * (size_t)lp.num_row;
  }
  ri.alloc(ni, false); rd.alloc(nd, false);
  dl.assign(lps, lps + count);
  ni = nd = 0;
  for (int i = 0; i < count; i++) {
    const b200pdlp_lp& lp = lps[i];
    b200pdlp_lp& d = dl[i];
    const int n0 = lp.num_col, m = lp.num_row, nnz = lp.a_start[n0];
    auto up_i = [&](const int* src, size_t len) { int* p = ri.p + ni; if (len) CUDA_OK(cudaMemcpy(p, src, len * sizeof(int), cudaMemcpyHostToDevice)); ni += len; return p; };
    auto up_d = [&](const double* src, size_t len) { double* p = rd.p + nd; if (len) CUDA_OK(cudaMemcpy(p, src, len * sizeof(double), cudaMemcpyHostToDevice)); nd += len; return p; };
    d.a_start = up_i(lp.a_start, n0 + 1); d.a_index = up_i(lp.a_index, nnz); d.a_value = up_d(lp.a_value, nnz);
    d.col_cost = up_d(lp.col_cost, n0); d.col_lower = up_d(lp.col_lower, n0); d.col_upper = up_d(lp.col_upper, n0);
    d.row_lower = up_d(lp.row_lower, m); d.row_upper = up_d(lp.row_upper, m);
  }
}

static void batch_prep_compare(int count, const b200pdlp_lp* lps, int scaling, double* report) {
  device_count_checked();
  RawLps raw;
  upload_raw_lps(count, lps, raw);
  StreamHolder sh;
  DeviceBatch D;
  Laps lap;
  PrepMode mode;
  mode.scaling = scaling;
  device_batch_prologue(sh.s, count, raw.dl.data(), nullptr, mode, std::numeric_limits<int>::max(), "b200pdlp_debug_batch_prep_compare",
                        D, lap);
  std::vector<StdForm> F((size_t)count);
  for (int i = 0; i < count; i++) {
    const BatchPrep& P = D.hp[i];
    StdForm& f = F[i];
    HostLayout L;
    formulate(lps[i], f);
    scale(f, scaling != 0);
    build_layout(f, 0, 1, std::numeric_limits<int>::max(), L);
    std::vector<double> x0, y0;
    host_start_point(f, nullptr, x0, y0);
    double* rep = report + (size_t)kBatchPrepItems * i;
    for (int k = 0; k < kBatchPrepItems; k++) rep[k] = 0.0;
    rep[0] = (P.n != f.n) + (P.m != f.m) + (P.nnz != f.nnz) + (P.neq != f.neq);
    if (rep[0] != 0.0) {   // nothing else lines up
      for (int k = 1; k < kBatchPrepItems; k++) rep[k] = -1.0;
      continue;
    }
    const int n = f.n, m = f.m;
    const std::vector<double> v = download_vec(P.vec, batch_vec_len(n, m));
    const double* w = v.data() + 12 * (size_t)n;
    rep[1] = bit_mismatches(v.data(), f.cost.data(), n);
    rep[2] = bit_mismatches(v.data() + n, f.lower.data(), n);
    rep[3] = bit_mismatches(v.data() + 2 * n, f.upper.data(), n);
    rep[4] = bit_mismatches(w, f.rhs.data(), m);
    rep[5] = bit_mismatches(v.data() + 3 * n, f.col_scale.data(), n);
    rep[6] = bit_mismatches(w + m, f.row_scale.data(), m);
    rep[7] = bit_mismatches(download_vec(P.row_new_idx, m).data(), f.row_new_idx.data(), m);
    rep[8] = bit_mismatches(download_vec(P.row_class, m).data(), reinterpret_cast<const int*>(f.row_class.data()), m);
    static_assert(sizeof(RowClass) == sizeof(int), "row classes are ints");
    auto sell = [&](const SellMatrix& H, const int4* sl, const int* col, const double* val, double* r) {
      const size_t ns = H.slices.size(), ne = H.col.size();
      const std::vector<int4> ds = download_vec(sl, ns);
      r[0] = bit_mismatches(reinterpret_cast<const int4*>(H.slices.data()), ds.data(), ns);
      if (r[0] != 0.0) { r[1] = r[2] = -1.0; return; }
      r[1] = bit_mismatches(download_vec(col, ne).data(), H.col.data(), ne);
      r[2] = bit_mismatches(download_vec(val, ne).data(), H.val.data(), ne);
    };
    sell(L.A, P.a_slices, P.a_col, P.a_val, rep + 9);
    sell(L.AT, P.at_slices, P.at_col, P.at_val, rep + 12);
    rep[15] = bit_mismatches(v.data() + 4 * n, x0.data(), n);
    rep[16] = bit_mismatches(w + 2 * m, y0.data(), m);
    std::vector<double> xsum(n);
    for (int j = 0; j < n; j++) xsum[j] = proj_zero(f, j);
    rep[17] = bit_mismatches(v.data() + 8 * n, xsum.data(), n);
    const double* r = D.rec.data() + (size_t)kPrepRec * i;
    double cost_sq = 0.0, rhs_sq = 0.0;
    for (int j = 0; j < n; j++) cost_sq += f.cost[j] * f.cost[j];
    for (int q = 0; q < m; q++) rhs_sq += f.rhs[q] * f.rhs[q];
    const double got[5] = {std::sqrt(r[0]), std::sqrt(r[1]), r[2], r[3], r[4]};
    const double want[5] = {f.norm_cost, f.norm_rhs, f.amax, cost_sq, rhs_sq};
    for (int k = 0; k < 5; k++) rep[18 + k] = bit_mismatches(got + k, want + k, 1);
  }
  // the postsolve of a probe iterate (x, A'y, y, A x in half 0 of every block, a check assumed) into fresh device vectors
  std::vector<BatchPost> hpost((size_t)count);
  std::vector<std::vector<double>> probes((size_t)count);
  size_t nout = 0;
  for (int i = 0; i < count; i++) nout += 2 * (size_t)D.hp[i].n0 + 2 * (size_t)D.hp[i].m;
  DevBuf<double> dout;
  dout.alloc(nout, false);
  nout = 0;
  for (int i = 0; i < count; i++) {
    const BatchPrep& P = D.hp[i];
    const int n = P.n, m = P.m, n0 = P.n0;
    std::vector<double>& pr = probes[i];   // x, A'y (n each), y, A x (m each)
    pr.resize(2 * (size_t)n + 2 * (size_t)m);
    for (size_t k = 0; k < pr.size(); k++) pr[k] = batch_probe(i, (int)k);
    double* v = P.vec;
    double* w = v + 12 * (size_t)n;
    CUDA_OK(cudaMemcpy(v + 4 * (size_t)n, pr.data(), n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(v + 6 * (size_t)n, pr.data() + n, n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(w + 2 * (size_t)m, pr.data() + 2 * n, m * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(w + 4 * (size_t)m, pr.data() + 2 * n + m, m * sizeof(double), cudaMemcpyHostToDevice));
    double* o = dout.p + nout;
    hpost[i] = BatchPost{o, o + n0, o + 2 * n0, o + 2 * n0 + m, 0, 1};
    nout += 2 * (size_t)n0 + 2 * (size_t)m;
  }
  DevBuf<BatchPost> dpost;
  dpost.alloc(count, false);
  dpost.upload(hpost.data(), count);
  launch_batch_post(sh.s, count, D.prep.p, dpost.p);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaStreamSynchronize(sh.s));
  for (int i = 0; i < count; i++) {
    double* rep = report + (size_t)kBatchPrepItems * i;
    if (rep[0] != 0.0) continue;
    const StdForm& f = F[i];
    const int n = f.n, m = f.m, n0 = f.n_orig;
    const std::vector<double>& pr = probes[i];
    std::vector<double> hx(pr.begin(), pr.begin() + n), haty(pr.begin() + n, pr.begin() + 2 * n);
    std::vector<double> hy(pr.begin() + 2 * n, pr.begin() + 2 * n + m), hax(pr.begin() + 2 * n + m, pr.end());
    std::vector<double> cv(n0), cd(n0), rv(m), rdual(m);
    b200pdlp_result res{};
    res.col_value = cv.data(); res.col_dual = cd.data(); res.row_value = rv.data(); res.row_dual = rdual.data();
    host_postsolve(f, true, hx, hy, hax, haty, &res);
    const BatchPost& q = hpost[i];
    rep[23] = bit_mismatches(download_vec(q.col_value, n0).data(), cv.data(), n0);
    rep[24] = bit_mismatches(download_vec(q.col_dual, n0).data(), cd.data(), n0);
    rep[25] = bit_mismatches(download_vec(q.row_value, m).data(), rv.data(), m);
    rep[26] = bit_mismatches(download_vec(q.row_dual, m).data(), rdual.data(), m);
  }
}

// ----------------------------------------------------------------------------------- batch of small LPs, HiPDLP mode
// b200pdlp_solve_hipdlp_batch: every member is an ordered-mode HiPDLP problem, solved by one CTA of hip_batch_round_kernel
// (batch_kernels.cu).  The host prologue (formulate_hipdlp, scale_hipdlp, build_layout) runs on host threads; the members are
// packed into pooled buffers, one descriptor each.  A round is one block of 40 Halpern steps for every unfinished member
// (round 0: the power method, the initial point and the iteration-0 check): one upload of the control blocks and states, one
// launch, one read-back, then each member's HipController decisions in the order solve_hipdlp_on_device takes them.  The
// PID weight's log / exp / log10 stay on the host.  Each member returns the bits b200pdlp_solve_hipdlp returns for it alone.

// a member's standard form under HiPDLP's classification (std_form_cols with infinite thresholds, as use_device_prep_hipdlp)
// must be an ordered-mode problem: checked before any device work
static void check_hipdlp_batch_member(const b200pdlp_lp* lp, const b200pdlp_hipdlp_params& prm, int i) {
  const int rc = guarded([&] {
    check_lp(lp);
    const int omax = prm.ordered_max == 0 ? 4096 : prm.ordered_max;
    if (omax < 0) throw Error(B200PDLP_ERR_ARG, "ordered_max < 0: a batch solves ordered-mode problems only");
    const int n = std_form_cols(*lp, std::numeric_limits<double>::infinity());
    if (std::max(n, lp->num_row) > omax)
      throw Error(B200PDLP_ERR_ARG, "standard form " + std::to_string(lp->num_row) + " x " + std::to_string(n) +
                                        " exceeds ordered_max = " + std::to_string(omax));
  });
  if (rc != B200PDLP_OK) throw Error(rc, "b200pdlp_solve_hipdlp_batch: member " + std::to_string(i) + ": " + g_last_error);
}

struct HipBatchRun {   // one member's host control over the rounds
  StdForm f;           // b200pdlp_solve_hipdlp_batch_device fills the scalars only: dimensions, sense, offset, norms, scaled
  HipController ctl;
  bool converged = false, timed_out = false;
  int sol = 0;   // converged: 0 at the iteration-0 check (x, y), 1 after a block (xn, yn)
};

struct HipBatchHost : HipBatchRun {   // one member of b200pdlp_solve_hipdlp_batch on the host
  HostLayout L;
  size_t vec = 0, sl_a = 0, sl_at = 0, e_a = 0, e_at = 0;   // offsets in the pools
};

// the HipBatchMember of a member with block `v` (hip_batch_vec_len) and the given layouts
static HipBatchMember hip_batch_member(const StdForm& f, int neq, double* v, const int4* a_slices, const int* a_col,
                                       const double* a_val, const int4* at_slices, const int* at_col, const double* at_val) {
  const int n = f.n, m = f.m;
  double* w = v + 14 * (size_t)n;
  HipBatchMember M;
  M.n = n; M.m = m; M.neq = neq; M.scaled = f.scaled ? 1 : 0; M.offset = f.offset;
  M.a_slices = a_slices; M.a_col = a_col; M.a_val = a_val;
  M.at_slices = at_slices; M.at_col = at_col; M.at_val = at_val;
  M.cost = v; M.lower = v + n; M.upper = v + 2 * n; M.colscale = v + 3 * n;
  M.x = v + 4 * n; M.xa = v + 5 * n; M.xn = v + 6 * n; M.rx = v + 7 * n; M.aty = v + 8 * n; M.hslack = v + 9 * n;
  M.atyp = v + 10 * n; M.atdy = v + 11 * n; M.sp = v + 12 * n; M.sn = v + 13 * n;
  M.rlo = w; M.rup = w + m; M.rowscale = w + 2 * m;
  M.y = w + 3 * m; M.ya = w + 4 * m; M.yn = w + 5 * m; M.ry = w + 6 * m; M.axp = w + 7 * m; M.dy = w + 8 * m;
  return M;
}

// The rounds of a HiPDLP batch, for both entry points: one upload of the control blocks and states, one launch, one
// read-back, then each member's HipController decisions in the order solve_hipdlp_on_device takes them, until no member is
// active or the time limit has passed.
static BatchLoop hip_batch_rounds(cudaStream_t s, int count, const b200pdlp_hipdlp_params& prm, const HipBatchMember* dmem,
                                  const std::vector<HipBatchRun*>& B) {
  using clk = std::chrono::steady_clock;
  DevBuf<HipState> dst;
  DevBuf<HipBatchCtl> dctl;
  dst.alloc(count, false); dctl.alloc(count, false);
  PinnedArray<HipState> hst((size_t)count);
  PinnedArray<HipBatchCtl> hctl((size_t)count);
  memset(hst.p, 0, (size_t)count * sizeof(HipState));
  for (int i = 0; i < count; i++) {
    HipBatchCtl& c = hctl.p[i];
    memset(&c, 0, sizeof(HipBatchCtl));
    c.active = 1; c.first = 1;
  }
  const double t_lim = (prm.time_limit >= 0 && std::isfinite(prm.time_limit)) ? prm.time_limit : -1.0;   // < 0: none
  CudaEvent evl0, evl1, ev0, ev1;
  BatchLoop L;
  int active = count;
  CUDA_OK(cudaEventRecord(evl0, s));
  L.t_loop = clk::now();
  while (active > 0) {
    NvtxRange nvtx("b200pdlp: HiPDLP batch round");
    // solve_hipdlp_on_device reads its clock before every block.  There a restart decided after the last block copies the
    // iterates before that test; here the copy is the first thing of the next round, so a member that times out never
    // makes it.  That cannot show: the copy writes x, xa, y, ya and A'y only, an unconverged run returns x = y = 0, and the
    // slacks sp / sn the postsolve reads are those of the last check in both solves.
    if (L.rounds > 0 && t_lim >= 0 && std::chrono::duration<double>(clk::now() - L.t_loop).count() > t_lim) {
      for (int i = 0; i < count; i++)
        if (hctl.p[i].active) { B[i]->timed_out = true; hctl.p[i].active = 0; }
      break;
    }
    CUDA_OK(cudaMemcpyAsync(dctl.p, hctl.p, (size_t)count * sizeof(HipBatchCtl), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaMemcpyAsync(dst.p, hst.p, (size_t)count * sizeof(HipState), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaEventRecord(ev0, s));
    launch_hip_batch_round(s, count, dmem, dst.p, dctl.p);
    CUDA_OK(cudaEventRecord(ev1, s));
    CUDA_OK(cudaMemcpyAsync(hctl.p, dctl.p, (size_t)count * sizeof(HipBatchCtl), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    float ms = 0.f;
    CUDA_OK(cudaEventElapsedTime(&ms, ev0, ev1));
    L.iter_ms += ms;
    const bool first = L.rounds == 0;
    L.rounds++;
    for (int i = 0; i < count; i++) {
      HipBatchCtl& c = hctl.p[i];
      if (!c.active) continue;
      HipBatchRun& b = *B[i];
      HipController& ctl = b.ctl;
      const StdForm& f = b.f;
      bool done = false, restart = false;
      if (first) {   // iteration 0 (:566-572)
        const double op_norm_sq = (f.n > 0 && f.m > 0) ? c.outs[kHipBatchLambda] : 1.0;
        ctl.init(f.norm_cost, f.norm_rhs, op_norm_sq, prm.tolerance, prm.step_size_strategy);
        if (ctl.converged(c.outs)) { b.converged = true; b.sol = 0; done = true; }
        else done = ctl.iters >= prm.iter_limit;
      } else {
        if (c.fpe) ctl.restart_reference(c.outs + kHipBatchFpe);
        restart = ctl.after_block(c.outs);
        if (ctl.pfeas < ctl.tol * (1.0 + f.norm_rhs) && ctl.dfeas < ctl.tol * (1.0 + f.norm_cost) && ctl.relgap < ctl.tol) {
          b.converged = true; b.sol = 1; done = true;
        } else {
          done = ctl.iters >= prm.iter_limit;
        }
      }
      if (done) { c.active = 0; active--; continue; }
      c.first = 0;
      c.restart = restart ? 1 : 0;
      c.fpe = ctl.pending_restart_fpe ? 1 : 0;
      HipState& st = hst.p[i];
      st.primal_step = ctl.primal_step; st.dual_step = ctl.dual_step; st.halpern_iteration = ctl.halpern_iteration;
    }
  }
  CUDA_OK(cudaEventRecord(evl1, s));
  CUDA_OK(cudaEventSynchronize(evl1));
  CUDA_OK(cudaEventElapsedTime(&L.loop_ms, evl0, evl1));
  L.solve_seconds = std::chrono::duration<double>(clk::now() - L.t_loop).count();
  return L;
}

// the fields of a HiPDLP batch result besides the vectors; the timings and kernel_launches are the batch's
static void hip_batch_result(b200pdlp_result* out, const HipBatchRun& b, const BatchLoop& L, double setup_seconds) {
  const StdForm& f = b.f;
  const HipController& ctl = b.ctl;
  out->value_valid = 1; out->dual_valid = 1;
  out->term_code = b.converged ? B200PDLP_OPTIMAL : B200PDLP_TIMELIMIT_OR_ITERLIMIT;
  out->term_iterate = b.timed_out ? 2 : 0;
  out->iters = ctl.iters; out->passes = ctl.iters; out->restarts = ctl.restarts;
  out->kernel_launches = (int)std::min<long long>(L.rounds, 2147483647LL);
  out->primal_obj = ctl.pobj; out->dual_obj = ctl.dobj; out->primal_feas = ctl.pfeas; out->dual_feas = ctl.dfeas;
  out->gap = ctl.pobj - ctl.dobj; out->rel_gap = ctl.relgap;
  out->setup_seconds = setup_seconds;
  out->solve_seconds = L.solve_seconds;
  out->loop_device_ms = L.loop_ms;
  out->iter_device_ms = L.iter_ms;
  out->form_cols = f.n; out->form_rows = f.m; out->form_nnz = f.nnz; out->form_neq = f.neq;
}

static void solve_hipdlp_batch(int count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params& prm, b200pdlp_result* outs) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  Laps lap;
  device_count_checked();
  if (prm.device >= 0) CUDA_OK(cudaSetDevice(prm.device));
  StreamHolder sh;
  cudaStream_t s = sh.s;
  std::vector<HipBatchHost> B((size_t)count);
  {
    NvtxRange nvtx("b200pdlp: HiPDLP batch prologue (host threads)");
    for_members(count, [&](int i) {
      HipBatchHost& b = B[i];
      formulate_hipdlp(lps[i], b.f);
      scale_hipdlp(b.f, prm.scaling_mode, prm.ruiz_iterations);
      build_layout(b.f, 0, 1, prm.ordered_max, b.L);
      if (!b.L.ordered || !b.L.A.segs.empty() || !b.L.AT.segs.empty())
        throw Error(B200PDLP_ERR_STATE, "the layout is not an ordered-mode layout");
    });
  }
  lap("batch", "HiPDLP prologue (host threads)");

  // ---- pooled device buffers: vectors, slice descriptors, column ids and values of A and A'; one descriptor per member
  size_t nvec = 0, nsl = 0, nent = 0;
  for (HipBatchHost& b : B) {
    b.vec = nvec; nvec += hip_batch_vec_len(b.f.n, b.f.m);
    b.sl_a = nsl; nsl += b.L.A.slices.size();
    b.sl_at = nsl; nsl += b.L.AT.slices.size();
    b.e_a = nent; nent += b.L.A.col.size();
    b.e_at = nent; nent += b.L.AT.col.size();
  }
  std::vector<double> hvec(std::max<size_t>(nvec, 1), 0.0), hval(std::max<size_t>(nent, 1), 0.0);
  std::vector<int> hcol(std::max<size_t>(nent, 1), 0);
  std::vector<int4> hsl(std::max<size_t>(nsl, 1));
  for_members(count, [&](int i) {
    const HipBatchHost& b = B[i];
    const StdForm& f = b.f;
    const int n = f.n, m = f.m;
    const int* cperm = b.L.cperm.data();
    const int* rperm = b.L.rperm.data();
    double* v = hvec.data() + b.vec;
    double* w = v + 14 * n;
    for (int j = 0; j < n; j++) {   // device order, as create_problem_hipdlp uploads them
      v[j] = f.cost[cperm[j]]; v[n + j] = f.lower[cperm[j]]; v[2 * n + j] = f.upper[cperm[j]]; v[3 * n + j] = f.col_scale[cperm[j]];
    }
    for (int r = 0; r < m; r++) { w[r] = f.rhs[rperm[r]]; w[m + r] = f.row_upper[rperm[r]]; w[2 * m + r] = f.row_scale[rperm[r]]; }
    static_assert(sizeof(SellMatrix::Slice) == sizeof(int4), "descriptor layout");
    memcpy(hsl.data() + b.sl_a, b.L.A.slices.data(), b.L.A.slices.size() * sizeof(int4));
    memcpy(hsl.data() + b.sl_at, b.L.AT.slices.data(), b.L.AT.slices.size() * sizeof(int4));
    std::copy(b.L.A.col.begin(), b.L.A.col.end(), hcol.begin() + b.e_a);
    std::copy(b.L.AT.col.begin(), b.L.AT.col.end(), hcol.begin() + b.e_at);
    std::copy(b.L.A.val.begin(), b.L.A.val.end(), hval.begin() + b.e_a);
    std::copy(b.L.AT.val.begin(), b.L.AT.val.end(), hval.begin() + b.e_at);
  });
  DevBuf<double> dvec, dval;
  DevBuf<int> dcol;
  DevBuf<int4> dsl;
  DevBuf<HipBatchMember> dmem;
  dvec.alloc(hvec.size(), false); dval.alloc(hval.size(), false); dcol.alloc(hcol.size(), false); dsl.alloc(hsl.size(), false);
  dmem.alloc(count, false);
  std::vector<HipBatchMember> hmem((size_t)count);
  for (int i = 0; i < count; i++) {
    const HipBatchHost& b = B[i];
    hmem[i] = hip_batch_member(b.f, b.L.neq_local, dvec.p + b.vec, dsl.p + b.sl_a, dcol.p + b.e_a, dval.p + b.e_a,
                               dsl.p + b.sl_at, dcol.p + b.e_at, dval.p + b.e_at);
  }
  CUDA_OK(cudaMemcpyAsync(dvec.p, hvec.data(), hvec.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(dval.p, hval.data(), hval.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(dcol.p, hcol.data(), hcol.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(dsl.p, hsl.data(), hsl.size() * sizeof(int4), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(dmem.p, hmem.data(), (size_t)count * sizeof(HipBatchMember), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaStreamSynchronize(s));
  lap("batch", "pools + upload");

  std::vector<HipBatchRun*> R((size_t)count);
  for (int i = 0; i < count; i++) R[i] = &B[i];
  const BatchLoop loop = hip_batch_rounds(s, count, prm, dmem.p, R);
  lap("batch", "rounds");

  // ---- the host postsolve of every member (hip_host_postsolve, as the single solve's host prologue path), one download
  NvtxRange nvtx_post("b200pdlp: HiPDLP batch postsolve + download");
  CUDA_OK(cudaMemcpyAsync(hvec.data(), dvec.p, hvec.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  const double setup_seconds = std::chrono::duration<double>(loop.t_loop - t_begin).count();
  for_members(count, [&](int i) {
    const HipBatchHost& b = B[i];
    const StdForm& f = b.f;
    const int n = f.n, m = f.m;
    const double* v = hvec.data() + b.vec;
    const double* w = v + 14 * n;
    const double* x = b.converged ? v + (b.sol ? 6 : 4) * n : nullptr;   // xn or x
    const double* y = b.converged ? w + (b.sol ? 5 : 3) * m : nullptr;   // yn or y
    b200pdlp_result* out = outs + i;
    hip_host_postsolve(lps[i], f, b.L.cperm.data(), b.L.rperm.data(), x, y, v + 12 * n, v + 13 * n, out);
    hip_batch_result(out, b, loop, setup_seconds);
  });
  lap("batch", "postsolve (host threads)");
}

// ------------------------------------------------------------------ HiPDLP batch of small LPs already on the GPU
// b200pdlp_solve_hipdlp_batch_device: solve_hipdlp_batch for LPs whose arrays are device memory.  The prologue and the
// postsolve run on the device, one CTA per member (batch_prep.cu hip_batch_*_kernel); the rounds are solve_hipdlp_batch's
// (hip_batch_rounds).  The host reads one sizing record and |c|^2, |b|^2 per member, never an array.

static void solve_hipdlp_batch_device(int count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params& prm, b200pdlp_result* outs) {
  using clk = std::chrono::steady_clock;
  const char* who = "b200pdlp_solve_hipdlp_batch_device";
  const auto t_begin = clk::now();
  Laps lap;
  device_count_checked();
  if (prm.device >= 0) CUDA_OK(cudaSetDevice(prm.device));
  int device = 0;
  CUDA_OK(cudaGetDevice(&device));
  check_device_arrays(count, lps, nullptr, outs, device, who);
  StreamHolder sh;
  cudaStream_t s = sh.s;
  DeviceBatch D;
  PrepMode mode;
  mode.hip = true; mode.scaling = prm.scaling_mode; mode.ruiz_iterations = prm.ruiz_iterations;
  {
    NvtxRange nvtx("b200pdlp: HiPDLP batch prologue (device)");
    device_batch_prologue(s, count, lps, nullptr, mode, prm.ordered_max, who, D, lap);
  }
  const bool scaled = (prm.scaling_mode & 7) != 0;   // scale_hipdlp: any of its passes is switched on
  std::vector<HipBatchRun> runs((size_t)count);
  std::vector<HipBatchRun*> R((size_t)count);
  std::vector<HipBatchMember> hmem((size_t)count);
  for (int i = 0; i < count; i++) {
    HipBatchRun& b = runs[i];
    const BatchPrep& P = D.hp[i];
    const double* r = D.rec.data() + (size_t)kPrepRec * i;
    StdForm& f = b.f;
    f.hipdlp = true;
    f.n = P.n; f.m = P.m; f.nnz = P.nnz; f.neq = P.neq; f.n_orig = P.n0;
    f.sense = lps[i].sense; f.offset = lps[i].offset;
    f.norm_cost = std::sqrt(r[0]); f.norm_rhs = std::sqrt(r[1]);
    f.scaled = scaled;
    R[i] = &b;
    hmem[i] = hip_batch_member(f, P.neq, P.vec, P.a_slices, P.a_col, P.a_val, P.at_slices, P.at_col, P.at_val);
  }
  DevBuf<HipBatchMember> dmem;
  dmem.alloc(count, false);
  CUDA_OK(cudaMemcpyAsync(dmem.p, hmem.data(), (size_t)count * sizeof(HipBatchMember), cudaMemcpyHostToDevice, s));
  const BatchLoop loop = hip_batch_rounds(s, count, prm, dmem.p, R);
  lap("batch device", "rounds");

  // ---- the postsolve of every member on the device, into the caller's vectors
  NvtxRange nvtx_post("b200pdlp: HiPDLP batch postsolve (device)");
  std::vector<HipBatchPost> hpost((size_t)count);
  for (int i = 0; i < count; i++) {
    HipBatchPost& q = hpost[i];
    q.col_value = outs[i].col_value; q.col_dual = outs[i].col_dual; q.row_value = outs[i].row_value; q.row_dual = outs[i].row_dual;
    q.sol = runs[i].converged ? runs[i].sol : -1;
    q.pad = 0;
  }
  DevBuf<HipBatchPost> dpost;
  dpost.alloc(count, false);
  CUDA_OK(cudaMemcpyAsync(dpost.p, hpost.data(), (size_t)count * sizeof(HipBatchPost), cudaMemcpyHostToDevice, s));
  launch_hip_batch_post(s, count, D.prep.p, D.dhx.p, dpost.p, scaled ? 1 : 0);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaStreamSynchronize(s));
  const double setup_seconds = std::chrono::duration<double>(loop.t_loop - t_begin).count();
  for (int i = 0; i < count; i++) hip_batch_result(outs + i, runs[i], loop, setup_seconds);
  lap("batch device", "postsolve (device)");
}

// ---- b200pdlp_debug_hipdlp_batch_prep_compare: the HiPDLP device prologue and postsolve against their host twins
static const int kHipBatchPrepItems = 24;

static void hipdlp_batch_prep_compare(int count, const b200pdlp_lp* lps, int scaling_mode, int ruiz_iterations, double* report) {
  device_count_checked();
  RawLps raw;
  upload_raw_lps(count, lps, raw);
  StreamHolder sh;
  DeviceBatch D;
  Laps lap;
  PrepMode mode;
  mode.hip = true; mode.scaling = scaling_mode; mode.ruiz_iterations = ruiz_iterations;
  device_batch_prologue(sh.s, count, raw.dl.data(), nullptr, mode, std::numeric_limits<int>::max(),
                        "b200pdlp_debug_hipdlp_batch_prep_compare", D, lap);
  const bool scaled = (scaling_mode & 7) != 0;
  std::vector<StdForm> F((size_t)count);
  std::vector<HostLayout> Ls((size_t)count);
  for (int i = 0; i < count; i++) {
    const BatchPrep& P = D.hp[i];
    StdForm& f = F[i];
    HostLayout& L = Ls[i];
    formulate_hipdlp(lps[i], f);
    scale_hipdlp(f, scaling_mode, ruiz_iterations);
    build_layout(f, 0, 1, std::numeric_limits<int>::max(), L);
    double* rep = report + (size_t)kHipBatchPrepItems * i;
    for (int k = 0; k < kHipBatchPrepItems; k++) rep[k] = 0.0;
    rep[0] = (P.n != f.n) + (P.m != f.m) + (P.nnz != f.nnz) + (P.neq != f.neq);
    if (rep[0] != 0.0) {   // nothing else lines up
      for (int k = 1; k < kHipBatchPrepItems; k++) rep[k] = -1.0;
      continue;
    }
    const int n = f.n, m = f.m;
    const std::vector<double> v = download_vec(P.vec, hip_batch_vec_len(n, m));
    const double* w = v.data() + 14 * (size_t)n;
    rep[1] = bit_mismatches(v.data(), f.cost.data(), n);
    rep[2] = bit_mismatches(v.data() + n, f.lower.data(), n);
    rep[3] = bit_mismatches(v.data() + 2 * n, f.upper.data(), n);
    rep[4] = bit_mismatches(w, f.rhs.data(), m);
    rep[5] = bit_mismatches(w + m, f.row_upper.data(), m);
    rep[6] = bit_mismatches(v.data() + 3 * n, f.col_scale.data(), n);
    rep[7] = bit_mismatches(w + 2 * m, f.row_scale.data(), m);
    rep[8] = bit_mismatches(download_vec(P.row_new_idx, m).data(), f.row_new_idx.data(), m);
    rep[9] = bit_mismatches(download_vec(P.row_class, m).data(), reinterpret_cast<const int*>(f.row_class.data()), m);
    auto sell = [&](const SellMatrix& H, const int4* sl, const int* col, const double* val, double* r) {
      const size_t ns = H.slices.size(), ne = H.col.size();
      const std::vector<int4> ds = download_vec(sl, ns);
      r[0] = bit_mismatches(reinterpret_cast<const int4*>(H.slices.data()), ds.data(), ns);
      if (r[0] != 0.0) { r[1] = r[2] = -1.0; return; }
      r[1] = bit_mismatches(download_vec(col, ne).data(), H.col.data(), ne);
      r[2] = bit_mismatches(download_vec(val, ne).data(), H.val.data(), ne);
    };
    sell(L.A, P.a_slices, P.a_col, P.a_val, rep + 10);
    sell(L.AT, P.at_slices, P.at_col, P.at_val, rep + 13);
    const double* r = D.rec.data() + (size_t)kPrepRec * i;
    const double got[2] = {std::sqrt(r[0]), std::sqrt(r[1])};
    const double want[2] = {f.norm_cost, f.norm_rhs};
    for (int k = 0; k < 2; k++) rep[16 + k] = bit_mismatches(got + k, want + k, 1);
    rep[18] = scaled != f.scaled;
    for (int j = 0; j < n; j++) rep[19] += L.cperm[j] != j;   // the batch assumes identity orderings
    for (int q = 0; q < m; q++) rep[19] += L.rperm[q] != q;
  }
  // the postsolve of a probe iterate (x, y, sp, sn; a converged member at the iteration-0 check) into fresh device vectors
  std::vector<HipBatchPost> hpost((size_t)count);
  std::vector<std::vector<double>> probes((size_t)count);
  size_t nout = 0;
  for (int i = 0; i < count; i++) nout += 2 * (size_t)D.hp[i].n0 + 2 * (size_t)D.hp[i].m;
  DevBuf<double> dout;
  dout.alloc(nout, false);
  nout = 0;
  for (int i = 0; i < count; i++) {
    const BatchPrep& P = D.hp[i];
    const int n = P.n, m = P.m, n0 = P.n0;
    std::vector<double>& pr = probes[i];   // x, sp, sn (n each), y (m)
    pr.resize(3 * (size_t)n + m);
    for (size_t k = 0; k < pr.size(); k++) pr[k] = batch_probe(i, (int)k);
    double* v = P.vec;
    double* w = v + 14 * (size_t)n;
    CUDA_OK(cudaMemcpy(v + 4 * (size_t)n, pr.data(), n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(v + 12 * (size_t)n, pr.data() + n, 2 * (size_t)n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(w + 3 * (size_t)m, pr.data() + 3 * n, m * sizeof(double), cudaMemcpyHostToDevice));
    double* o = dout.p + nout;
    hpost[i] = HipBatchPost{o, o + n0, o + 2 * n0, o + 2 * n0 + m, 0, 0};
    nout += 2 * (size_t)n0 + 2 * (size_t)m;
  }
  DevBuf<HipBatchPost> dpost;
  dpost.alloc(count, false);
  dpost.upload(hpost.data(), count);
  launch_hip_batch_post(sh.s, count, D.prep.p, D.dhx.p, dpost.p, scaled ? 1 : 0);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaStreamSynchronize(sh.s));
  for (int i = 0; i < count; i++) {
    double* rep = report + (size_t)kHipBatchPrepItems * i;
    if (rep[0] != 0.0) continue;
    const StdForm& f = F[i];
    const HostLayout& L = Ls[i];
    const int n = f.n, m = f.m, n0 = f.n_orig;
    const double* pr = probes[i].data();
    // (at least one element each: hip_host_postsolve writes nothing when a vector pointer is NULL)
    std::vector<double> cv(std::max(n0, 1)), cd(std::max(n0, 1)), rv(std::max(m, 1)), rdual(std::max(m, 1));
    b200pdlp_result res{};
    res.col_value = cv.data(); res.col_dual = cd.data(); res.row_value = rv.data(); res.row_dual = rdual.data();
    hip_host_postsolve(lps[i], f, L.cperm.data(), L.rperm.data(), pr, pr + 3 * n, pr + n, pr + 2 * n, &res);
    const HipBatchPost& q = hpost[i];
    rep[20] = bit_mismatches(download_vec(q.col_value, n0).data(), cv.data(), n0);
    rep[21] = bit_mismatches(download_vec(q.col_dual, n0).data(), cd.data(), n0);
    rep[22] = bit_mismatches(download_vec(q.row_value, m).data(), rv.data(), m);
    rep[23] = bit_mismatches(download_vec(q.row_dual, m).data(), rdual.data(), m);
  }
}

// ====================================================================================== KKT assessment of a batch
// b200pdlp_kkt_check_batch / _device: kkt_batch.cu's kernel assesses every member at once (one CTA each); the host reads one
// record per member and runs finalize_kkt on it, so the derived fields and the status rules are those of the single checks.

// the checks of a member that read no array: its lengths, and no NULL array whose length is positive (the matrix arrays,
// whose length is a_start[num_col], are checked with the other array checks)
static void check_kkt_batch_member(const b200pdlp_lp& lp, const b200pdlp_solution& x, int i, const char* who) {
  const std::string at = std::string(who) + ": member " + std::to_string(i) + ": ";
  if (lp.num_col < 0 || lp.num_row < 0) throw Error(B200PDLP_ERR_ARG, at + "num_col < 0 or num_row < 0");
  const bool cols = lp.num_col > 0, rows = lp.num_row > 0;
  if (!lp.a_start || (cols && !(lp.col_cost && lp.col_lower && lp.col_upper && x.col_value && x.col_dual)) ||
      (rows && !(lp.row_lower && lp.row_upper && x.row_value && x.row_dual)))
    throw Error(B200PDLP_ERR_ARG, at + "NULL array of positive length");
}

// the array checks of kkt_batch_check_kernel on host arrays (a BatchPrepErr)
static int kkt_batch_host_arrays(const b200pdlp_lp& lp) {
  if (lp.a_start[0] != 0) return kPrepStart0;
  for (int j = 0; j < lp.num_col; j++)
    if (lp.a_start[j + 1] < lp.a_start[j]) return kPrepDecreasing;
  const int nnz = lp.a_start[lp.num_col];
  if (nnz > 0 && (!lp.a_index || !lp.a_value)) return kPrepNull;
  for (int p = 0; p < nnz; p++)
    if ((unsigned)lp.a_index[p] >= (unsigned)lp.num_row) return kPrepIndex;
  return kPrepOk;
}

// device_arrays: every array of lps / sols is device memory of the device (b200pdlp_kkt_check_batch_device).  Otherwise they
// are host arrays that have passed kkt_batch_host_arrays, and the call uploads them with the members' descriptors in one copy.
static void kkt_check_batch(int count, const b200pdlp_lp* lps, const b200pdlp_solution* sols, const KktTolerances& t,
                            int device, bool device_arrays, const char* who, b200pdlp_kkt_info* inout, Laps& lap) {
  device_count_checked();
  if (device >= 0) CUDA_OK(cudaSetDevice(device));
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  NvtxRange nvtx("b200pdlp: KKT check batch");
  StreamHolder sh;
  cudaStream_t s = sh.s;
  std::vector<KktBatchMember> hm((size_t)count);
  for (int i = 0; i < count; i++) {
    const b200pdlp_lp& lp = lps[i];
    const b200pdlp_solution& x = sols[i];
    KktBatchMember& M = hm[i];
    M.n = lp.num_col; M.m = lp.num_row; M.sense = lp.sense;
    M.a_start = lp.a_start; M.a_index = lp.a_index; M.a_value = lp.a_value;
    M.col_cost = lp.col_cost; M.col_lower = lp.col_lower; M.col_upper = lp.col_upper;
    M.row_lower = lp.row_lower; M.row_upper = lp.row_upper;
    M.col_value = x.col_value; M.col_dual = x.col_dual; M.row_value = x.row_value; M.row_dual = x.row_dual;
  }
  const size_t head = (size_t)count * sizeof(KktBatchMember);
  DevBuf<char> pack;   // the descriptors, then (host arrays) every member's doubles and ints
  std::vector<int> nnz((size_t)count);
  if (device_arrays) {
    for (int i = 0; i < count; i++) {
      const b200pdlp_lp& lp = lps[i];
      const b200pdlp_solution& x = sols[i];
      check_device_array(lp.a_start, dev, i, "a_start", who);
      check_device_array(lp.a_index, dev, i, "a_index", who);
      check_device_array(lp.a_value, dev, i, "a_value", who);
      check_device_array(lp.col_cost, dev, i, "col_cost", who);
      check_device_array(lp.col_lower, dev, i, "col_lower", who);
      check_device_array(lp.col_upper, dev, i, "col_upper", who);
      check_device_array(lp.row_lower, dev, i, "row_lower", who);
      check_device_array(lp.row_upper, dev, i, "row_upper", who);
      check_device_array(x.col_value, dev, i, "col_value", who);
      check_device_array(x.col_dual, dev, i, "col_dual", who);
      check_device_array(x.row_value, dev, i, "row_value", who);
      check_device_array(x.row_dual, dev, i, "row_dual", who);
    }
    // the array checks on the device, and nnz for the workspace: one record per member
    pack.alloc(head, false);
    DevBuf<KktBatchSize> dsize;
    dsize.alloc(count, false);
    CUDA_OK(cudaMemcpyAsync(pack.p, hm.data(), head, cudaMemcpyHostToDevice, s));
    launch_kkt_batch_check(s, count, reinterpret_cast<const KktBatchMember*>(pack.p), dsize.p);
    CUDA_OK(cudaGetLastError());
    std::vector<KktBatchSize> sz((size_t)count);
    CUDA_OK(cudaMemcpyAsync(sz.data(), dsize.p, (size_t)count * sizeof(KktBatchSize), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    for (int i = 0; i < count; i++) {   // the lowest failing member
      if (sz[i].err != kPrepOk)
        throw Error(B200PDLP_ERR_ARG, std::string(who) + ": member " + std::to_string(i) + ": " + prep_error_text(sz[i].err));
      nnz[i] = sz[i].nnz;
    }
    lap("kkt batch", "validation");
  } else {
    for (int i = 0; i < count; i++) nnz[i] = lps[i].a_start[lps[i].num_col];
  }

  // ---- the workspace: rptr [m + 1], rpos and colof [nnz] (ints); rres [m], cres [n] (doubles)
  size_t ni = 0, nd = 0;
  for (int i = 0; i < count; i++) {
    ni += (size_t)hm[i].m + 1 + 2 * (size_t)nnz[i];
    nd += (size_t)hm[i].n + hm[i].m;
  }
  DevBuf<int> wi;
  DevBuf<double> wd;
  DevBuf<KktBatchRec> drec;
  wi.alloc(ni, false); wd.alloc(nd, false); drec.alloc(count, false);
  ni = nd = 0;
  for (int i = 0; i < count; i++) {
    KktBatchMember& M = hm[i];
    M.rptr = wi.p + ni; M.rpos = M.rptr + M.m + 1; M.colof = M.rpos + nnz[i];
    ni += (size_t)M.m + 1 + 2 * (size_t)nnz[i];
    M.rres = wd.p + nd; M.cres = M.rres + M.m;
    nd += (size_t)M.n + M.m;
  }
  if (device_arrays) {
    CUDA_OK(cudaMemcpyAsync(pack.p, hm.data(), head, cudaMemcpyHostToDevice, s));
  } else {
    // one packed copy (per-array copies would cost more than the kernel): the descriptors, the doubles, the ints
    size_t dbl = 0, ints = 0;
    for (int i = 0; i < count; i++) {
      dbl += (size_t)nnz[i] + 5 * (size_t)hm[i].n + 4 * (size_t)hm[i].m;
      ints += (size_t)hm[i].n + 1 + nnz[i];
    }
    const size_t bytes = head + 8 * dbl + 4 * ints;
    pack.alloc(bytes, false);
    PinnedArray<char> stage(bytes);
    double* hd = reinterpret_cast<double*>(stage.p + head);
    int* hi = reinterpret_cast<int*>(stage.p + head + 8 * dbl);
    const double* dd = reinterpret_cast<const double*>(pack.p + head);
    const int* di = reinterpret_cast<const int*>(pack.p + head + 8 * dbl);
    size_t od = 0, oi = 0;
    auto put_d = [&](const double* src, size_t len) {
      if (len) memcpy(hd + od, src, len * sizeof(double));
      od += len;
      return dd + od - len;
    };
    auto put_i = [&](const int* src, size_t len) {
      if (len) memcpy(hi + oi, src, len * sizeof(int));
      oi += len;
      return di + oi - len;
    };
    for (int i = 0; i < count; i++) {
      KktBatchMember& M = hm[i];
      const size_t n = M.n, m = M.m, z = nnz[i];
      M.a_start = put_i(M.a_start, n + 1); M.a_index = put_i(M.a_index, z); M.a_value = put_d(M.a_value, z);
      M.col_cost = put_d(M.col_cost, n); M.col_lower = put_d(M.col_lower, n); M.col_upper = put_d(M.col_upper, n);
      M.row_lower = put_d(M.row_lower, m); M.row_upper = put_d(M.row_upper, m);
      M.col_value = put_d(M.col_value, n); M.col_dual = put_d(M.col_dual, n);
      M.row_value = put_d(M.row_value, m); M.row_dual = put_d(M.row_dual, m);
    }
    memcpy(stage.p, hm.data(), head);
    CUDA_OK(cudaMemcpyAsync(pack.p, stage.p, bytes, cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));   // (`stage` goes back to the pinned cache at the end of this block)
  }
  lap("kkt batch", "upload");
  launch_kkt_batch(s, count, reinterpret_cast<const KktBatchMember*>(pack.p), t, drec.p);
  CUDA_OK(cudaGetLastError());
  if (lap.on) CUDA_OK(cudaStreamSynchronize(s));
  lap("kkt batch", "kernel");
  PinnedArray<KktBatchRec> rec((size_t)count);
  CUDA_OK(cudaMemcpyAsync(rec.p, drec.p, (size_t)count * sizeof(KktBatchRec), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  lap("kkt batch", "read-back");
  // inout is written only now, when nothing can fail any more
  std::vector<b200pdlp_kkt_info> out(inout, inout + count);
  for (int i = 0; i < count; i++) {
    out[i].norm_bounds = rec.p[i].norm_bounds;
    out[i].norm_costs = rec.p[i].norm_costs;
    finalize_kkt(rec.p[i].sums, lps[i].offset, t, &out[i]);
  }
  std::copy(out.begin(), out.end(), inout);
}

static int kkt_check_batch_entry(bool device_arrays, int count, const b200pdlp_lp* lps, const b200pdlp_solution* sols,
                                 const b200pdlp_kkt_tolerances* tol, int device, b200pdlp_kkt_info* inout) {
  DeviceGuard dg;
  const char* who = device_arrays ? "b200pdlp_kkt_check_batch_device" : "b200pdlp_kkt_check_batch";
  return guarded([&] {
    Laps lap;
    if (count < 0) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": count < 0");
    if (count == 0) return;
    if (!lps || !sols || !tol || !inout) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": null argument");
    for (int i = 0; i < count; i++) check_kkt_batch_member(lps[i], sols[i], i, who);
    if (!device_arrays) {   // the array checks of host arrays: on the host, before any device work
      for (int i = 0; i < count; i++) {
        const int err = kkt_batch_host_arrays(lps[i]);
        if (err != kPrepOk)
          throw Error(B200PDLP_ERR_ARG, std::string(who) + ": member " + std::to_string(i) + ": " + prep_error_text(err));
      }
      lap("kkt batch", "validation");
    }
    kkt_check_batch(count, lps, sols, tolerances_of(tol), device, device_arrays, who, inout, lap);
  });
}


extern "C" {

const char* b200pdlp_last_error(void) { return g_last_error.c_str(); }
int b200pdlp_version(void) { return B200PDLP_VERSION; }
int b200pdlp_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

void b200pdlp_default_params(b200pdlp_params* p) {
  memset(p, 0, sizeof(*p));
  p->iter_limit = 2147483647;                 // kHighsIInf (HighsOptions.h:1341)
  p->tol_primal = p->tol_dual = p->tol_gap = 1e-7;
  p->time_limit = -1.0;                       // none (0 = already over: the first check ends the run)
  p->scaling = 1; p->adaptive_step = 1; p->restart = 1;
  p->log_level = 0; p->check_interval = 40; p->device = -1; p->graph_passes = 0;
}

int b200pdlp_problem_create(const b200pdlp_lp* lp, const b200pdlp_params* params, int32_t rank, int32_t world, b200pdlp_problem** out) {
  DeviceGuard dg;
  return guarded([&] {
    if (!params || !out || world < 1 || rank < 0 || rank >= world) throw Error(B200PDLP_ERR_ARG, "b200pdlp_problem_create: bad arguments");
    check_params(*params);
    check_lp(lp, false);
    check_lp(lp, !use_device_prep(*lp, *params, world));
    auto* p = new b200pdlp_problem();
    try {
      p->prep.keep_form = true;   // persistent handle: the accessors below may ask for the standard form
      if (use_device_prep(*lp, *params, world)) create_problem_device(*lp, *params, p);
      else create_problem(*lp, *params, rank, world, p);
    } catch (...) { delete p; throw; }
    *out = p;
  });
}

void b200pdlp_problem_destroy(b200pdlp_problem* p) {
  if (!p) return;
  DeviceGuard dg;
  cudaSetDevice(p->device);
  delete p;
}

int b200pdlp_problem_dims(const b200pdlp_problem* p, int32_t dims[8]) {
  return guarded([&] {
    if (!p || !dims) throw Error(B200PDLP_ERR_ARG, "null argument");
    dims[0] = p->n; dims[1] = p->m; dims[2] = p->form.nnz; dims[3] = p->form.neq;
    dims[4] = p->ml; dims[5] = p->r0; dims[6] = p->csr_local.nnz; dims[7] = p->form.n_orig;
  });
}

int b200pdlp_problem_get_vector(const b200pdlp_problem* p, int32_t which, double* dst, int32_t cap) {
  if (!p || !dst) return B200PDLP_ERR_ARG;
  if (p->dev_form) {
    DeviceGuard dg;
    const int rc = guarded([&] { set_device(p); ensure_host_form(const_cast<b200pdlp_problem*>(p)); });
    if (rc != B200PDLP_OK) return rc;
  }
  const std::vector<double>* v = nullptr;
  switch (which) {
    case 0: v = &p->form.cost; break;
    case 1: v = &p->form.lower; break;
    case 2: v = &p->form.upper; break;
    case 3: v = &p->form.rhs; break;
    case 4: v = &p->form.col_scale; break;
    case 5: v = &p->form.row_scale; break;
    default: return B200PDLP_ERR_ARG;
  }
  if (!v) return B200PDLP_ERR_ARG;
  const int k = std::min<int>(cap, (int)v->size());
  memcpy(dst, v->data(), (size_t)k * sizeof(double));
  return k;
}

int b200pdlp_problem_get_csr(const b200pdlp_problem* p, int32_t* rowptr, int32_t* col, double* val) {
  if (!p || !rowptr || !col || !val) return B200PDLP_ERR_ARG;
  if (p->dev_form) {
    DeviceGuard dg;
    const int rc = guarded([&] { set_device(p); ensure_host_form(const_cast<b200pdlp_problem*>(p)); });
    if (rc != B200PDLP_OK) return rc;
  }
  Csr lazy;
  if (p->csr_local.rowptr.empty()) {
    // device-filled layouts keep no host copy: rebuild it from the (downloaded) scaled form on demand
    StdForm& f = const_cast<StdForm&>(p->form);
    if (f.rptr.empty()) build_row_index(f);
    build_row_major(f, p->r0, p->r1, lazy);
  }
  const Csr& a = p->csr_local.rowptr.empty() ? lazy : p->csr_local;
  memcpy(rowptr, a.rowptr.data(), (size_t)(a.nrows + 1) * sizeof(int));
  memcpy(col, a.col.data(), (size_t)a.nnz * sizeof(int));
  memcpy(val, a.val.data(), (size_t)a.nnz * sizeof(double));
  return B200PDLP_OK;
}

int b200pdlp_spmv_ax(b200pdlp_problem* p, const double* x, double* ax) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !x || !ax) throw Error(B200PDLP_ERR_ARG, "null argument");
    set_device(p);
    ensure_host_maps(p);
    const size_t full = p->world == 1 ? (size_t)p->n : p->xfull.n;
    std::vector<double> t(std::max<size_t>(full, std::max(p->ml, 1)), 0.0);
    for (int j = 0; j < p->n; j++) t[seg_pos(p, j)] = x[p->cperm[j]];
    double* dx = p->world == 1 ? p->xavg.p : p->xfull.p;   // whole x supplied by the caller: no gather needed
    CUDA_OK(cudaMemcpyAsync(dx, t.data(), full * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    launch_spmv_plain(p->stream, p->A.dev, dx, p->axavg.p);
    p->launches++;
    CUDA_OK(cudaStreamSynchronize(p->stream));
    if (p->ml) CUDA_OK(cudaMemcpy(t.data(), p->axavg.p, (size_t)p->ml * sizeof(double), cudaMemcpyDeviceToHost));
    for (int i = 0; i < p->ml; i++) ax[p->rperm[i]] = t[i];
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_spmv_aty(b200pdlp_problem* p, const double* y, double* aty) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !y || !aty) throw Error(B200PDLP_ERR_ARG, "null argument");
    set_device(p);
    ensure_host_maps(p);
    const size_t full = p->world == 1 ? (size_t)p->n : p->part.n;
    std::vector<double> t(std::max<size_t>(full, std::max(p->ml, 1)), 0.0);
    for (int i = 0; i < p->ml; i++) t[i] = y[p->rperm[i]];
    if (p->ml) CUDA_OK(cudaMemcpyAsync(p->yavg.p, t.data(), (size_t)p->ml * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    // local partial A_g^T y (no reduction over ranks)
    if (p->world == 1) launch_spmv_plain(p->stream, p->AT.dev, p->yavg.p, p->atyavg.p);
    else launch_spmv_partial_aty(p->stream, p->AT.dev, nullptr, p->yavg.p, p->yavg.p, p->part.p, p->at_outpos.p);
    p->launches++;
    CUDA_OK(cudaStreamSynchronize(p->stream));
    CUDA_OK(cudaMemcpy(t.data(), p->world == 1 ? p->atyavg.p : p->part.p, full * sizeof(double), cudaMemcpyDeviceToHost));
    for (int j = 0; j < p->n; j++) aty[p->cperm[j]] = t[seg_pos(p, j)];
    CUDA_OK(cudaGetLastError());
  });
}

// ---- kernel-level entry points (SURVEY.md 8(b): _primal_step, _dual_step, _residuals): one fused kernel of the hot
// path on host vectors in standard-form order (H2D, kernel, D2H), single GPU.  They use the problem's iterate buffers as
// scratch, so a solve on the same handle starts from scratch afterwards (it always does).
static void kernel_api_state(b200pdlp_problem* p, double tau, double sigma) {
  PdhgState* h = p->hstate;
  memset(h, 0, sizeof(PdhgState));
  h->adaptive = 1; h->beta = 1.0;
  h->tau = h->tau_try = tau; h->sigma = h->sigma_try = sigma;
  h->stop_iter = 2147483647;
  push_state(p);
}
static double sum_partials(b200pdlp_problem* p, const ReduceScratch& r, int nb) {   // what K4 does with one accumulator
  std::vector<double> t((size_t)std::max(nb, 1));
  if (r.terms) {
    std::vector<double> terms((size_t)r.len);
    CUDA_OK(cudaMemcpy(terms.data(), r.terms, (size_t)r.len * sizeof(double), cudaMemcpyDeviceToHost));
    double s = 0.0;
    for (double v : terms) s += v;
    return s;
  }
  CUDA_OK(cudaMemcpy(t.data(), r.partials, (size_t)nb * sizeof(double), cudaMemcpyDeviceToHost));
  double s = 0.0;
  for (int i = 0; i < nb; i++) s += t[i];
  return s;
}

int b200pdlp_primal_step(b200pdlp_problem* p, const double* x, const double* aty, double tau, double* x_new, double* dx2) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !x || !aty || !x_new) throw Error(B200PDLP_ERR_ARG, "null argument");
    if (p->world != 1) throw Error(B200PDLP_ERR_ARG, "kernel-level entry points are single-GPU");
    set_device(p);
    ensure_host_maps(p);
    const int n = p->n;
    std::vector<double> t(n);
    for (int j = 0; j < n; j++) t[j] = x[p->cperm[j]];
    CUDA_OK(cudaMemcpyAsync(p->x[0].p, t.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    CUDA_OK(cudaStreamSynchronize(p->stream));
    for (int j = 0; j < n; j++) t[j] = aty[p->cperm[j]];
    CUDA_OK(cudaMemcpyAsync(p->aty[0].p, t.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice, p->stream));
    kernel_api_state(p, tau, tau);
    const ReduceScratch r1 = p->rs(kSlotK1, n);
    launch_primal_step(p->stream, n, p->state.p, p->x[0].p, p->x[1].p, p->aty[0].p, p->aty[1].p, p->cost.p, p->lower.p,
                       p->upper.p, p->xsum.p, r1);
    p->launches++;
    CUDA_OK(cudaMemcpyAsync(t.data(), p->x[1].p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
    CUDA_OK(cudaStreamSynchronize(p->stream));
    for (int j = 0; j < n; j++) x_new[p->cperm[j]] = t[j];
    if (dx2) *dx2 = sum_partials(p, r1, primal_step_grid(n));
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_dual_step(b200pdlp_problem* p, const double* x_new, const double* y, const double* ax, double sigma,
                       double* y_new, double* ax_new, double* dy2) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !x_new || !y || !ax || !y_new || !ax_new) throw Error(B200PDLP_ERR_ARG, "null argument");
    if (p->world != 1) throw Error(B200PDLP_ERR_ARG, "kernel-level entry points are single-GPU");
    set_device(p);
    ensure_host_maps(p);
    const int n = p->n, m = p->m;
    std::vector<double> t(std::max(n, m));
    cudaStream_t s = p->stream;
    for (int j = 0; j < n; j++) t[j] = x_new[p->cperm[j]];
    CUDA_OK(cudaMemcpyAsync(p->x[1].p, t.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));
    for (int i = 0; i < m; i++) t[i] = y[p->rperm[i]];
    CUDA_OK(cudaMemcpyAsync(p->y[0].p, t.data(), (size_t)m * sizeof(double), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));
    for (int i = 0; i < m; i++) t[i] = ax[p->rperm[i]];
    CUDA_OK(cudaMemcpyAsync(p->ax[0].p, t.data(), (size_t)m * sizeof(double), cudaMemcpyHostToDevice, s));
    kernel_api_state(p, sigma, sigma);
    const ReduceScratch r2 = p->rs(kSlotK2, m);
    launch_spmv_dual(s, p->A.dev, p->state.p, p->x[0].p, p->x[1].p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->rhs.p,
                     p->ysum.p, p->neq_local, 0, r2);
    p->launches++;
    CUDA_OK(cudaMemcpyAsync(t.data(), p->y[1].p, (size_t)m * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    for (int i = 0; i < m; i++) y_new[p->rperm[i]] = t[i];
    CUDA_OK(cudaMemcpyAsync(t.data(), p->ax[1].p, (size_t)m * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    for (int i = 0; i < m; i++) ax_new[p->rperm[i]] = t[i];
    if (dy2) *dy2 = sum_partials(p, r2, p->A.grid());
    CUDA_OK(cudaGetLastError());
  });
}

// out[10]: pobj, dobj, pfeas, dfeas, gap, relgap, primal-ray objective, primal-ray residual, dual-ray objective,
// dual-ray residual of the iterate (x, y) (PDHG_Compute_Residuals / _Infeas_Residuals); A x and A'y are formed here
int b200pdlp_residuals(b200pdlp_problem* p, const double* x, const double* y, double out[10]) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !x || !y || !out) throw Error(B200PDLP_ERR_ARG, "null argument");
    if (p->world != 1) throw Error(B200PDLP_ERR_ARG, "kernel-level entry points are single-GPU");
    set_device(p);
    ensure_host_maps(p);
    const int n = p->n, m = p->m;
    std::vector<double> t(std::max(n, m));
    cudaStream_t s = p->stream;
    for (int j = 0; j < n; j++) t[j] = x[p->cperm[j]];
    CUDA_OK(cudaMemcpyAsync(p->x[0].p, t.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));
    for (int i = 0; i < m; i++) t[i] = y[p->rperm[i]];
    CUDA_OK(cudaMemcpyAsync(p->y[0].p, t.data(), (size_t)m * sizeof(double), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));
    // the check machinery with sums = the iterate itself: "average" == current
    PdhgState* h = p->hstate;
    memset(h, 0, sizeof(PdhgState));
    h->sum_step = 1.0; h->beta = 1.0;
    push_state(p);
    CUDA_OK(cudaMemcpyAsync(p->xsum.p, p->x[0].p, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, s));
    CUDA_OK(cudaMemcpyAsync(p->ysum.p, p->y[0].p, (size_t)m * sizeof(double), cudaMemcpyDeviceToDevice, s));
    full_ax(p, p->x[0].p, p->ax[0].p);
    full_aty(p, p->y[0].p, p->aty[0].p);
    const CheckResult c = run_check(p, false);
    const Residuals& R = c.it[0];
    out[0] = R.pobj; out[1] = R.dobj; out[2] = R.pfeas; out[3] = R.dfeas; out[4] = R.gap; out[5] = R.relgap;
    out[6] = R.pinf_obj; out[7] = R.pinf_res; out[8] = R.dinf_obj; out[9] = R.dinf_res;
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_bench_spmv(b200pdlp_problem* p, int32_t which, int32_t reps, float* ms_total) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !ms_total || reps < 1) throw Error(B200PDLP_ERR_ARG, "bad argument");
    set_device(p);
    cudaEvent_t e0, e1;
    CUDA_OK(cudaEventCreate(&e0));
    CUDA_OK(cudaEventCreate(&e1));
    CUDA_OK(cudaEventRecord(e0, p->stream));
    for (int r = 0; r < reps; r++) {
      if (which == 0) launch_spmv_plain(p->stream, p->A.dev, p->world == 1 ? p->xavg.p : p->xfull.p, p->axavg.p);
      else if (p->world == 1) launch_spmv_plain(p->stream, p->AT.dev, p->yavg.p, p->atyavg.p);
      else launch_spmv_partial_aty(p->stream, p->AT.dev, nullptr, p->yavg.p, p->yavg.p, p->part.p, p->at_outpos.p);
    }
    p->launches += reps;
    CUDA_OK(cudaEventRecord(e1, p->stream));
    CUDA_OK(cudaEventSynchronize(e1));
    CUDA_OK(cudaEventElapsedTime(ms_total, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_bench_pass(b200pdlp_problem* p, int32_t reps, float ms[4]) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !ms || reps < 1) throw Error(B200PDLP_ERR_ARG, "bad argument");
    set_device(p);
    cudaStream_t s = p->stream;
    PdhgState* st = p->state.p;
    p->kernels_per_pass = p->world == 1 ? 4 : (p->p2p ? 5 : 6);
    pull_state(p);
    p->hstate->stop_iter = 2147483647;
    fill_pow_tables(p->hstate);
    push_state(p);
    cudaEvent_t ev[5];
    for (auto& e : ev) CUDA_OK(cudaEventCreate(&e));
    double acc[4] = {0, 0, 0, 0};
    for (int r = 0; r < reps; r++) {
      if (r % 64 == 63) { pull_state(p); fill_pow_tables(p->hstate); push_state(p); }
      if (p->world == 1) {
        const ReduceScratch r1 = p->rs(kSlotK1, p->n), r2 = p->rs(kSlotK2, p->ml), r3 = p->rs(kSlotK3, p->n);
        CUDA_OK(cudaEventRecord(ev[0], s));
        launch_primal_step(s, p->n, st, p->x[0].p, p->x[1].p, p->aty[0].p, p->aty[1].p, p->cost.p, p->lower.p,
                           p->upper.p, p->xsum.p, r1);
        CUDA_OK(cudaEventRecord(ev[1], s));
        launch_spmv_dual(s, p->A.dev, st, p->x[0].p, p->x[1].p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p,
                         p->rhs.p, p->ysum.p, p->neq_local, 0, r2);
        CUDA_OK(cudaEventRecord(ev[2], s));
        launch_spmv_primal(s, p->AT.dev, st, p->y[0].p, p->y[1].p, p->x[0].p, p->x[1].p, p->aty[0].p,
                           p->aty[1].p, r3);
        CUDA_OK(cudaEventRecord(ev[3], s));
        launch_step_rule(s, st, r1, primal_step_grid(p->n), r2, p->A.grid(), r3, p->AT.grid(), nullptr);
      } else {
        // ms[0] = primal shard + all-gather, ms[1] = A x + dual, ms[2] = partial A'y, ms[3] = reduce-scatter + step rule
        const ReduceScratch r1 = p->rs(kSlotK1, p->nl), r2 = p->rs(kSlotK2, p->ml);
        if (p->p2p) {
          CUDA_OK(cudaEventRecord(ev[0], s));
          launch_primal_shard_p2p(s, p->nl, st, p->x[0].p, p->x[1].p, p->aty[0].p, p->peers, p->world, p->rank,
                                  p->seg_len, p->cost.p, p->lower.p, p->upper.p, p->xsum.p, r1);
          launch_p2p_barrier(s, 0, st, r1.partials, primal_shard_p2p_grid(p->nl), p->peers, p->world, p->rank, p->seg_len,
                             p->shard_len, p->epochs.p, p->fault.p);
          CUDA_OK(cudaEventRecord(ev[1], s));
          launch_spmv_dual_mg(s, p->A.dev, st, p->xfull.p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->rhs.p,
                              p->ysum.p, p->neq_local, r2);
          CUDA_OK(cudaEventRecord(ev[2], s));
          launch_spmv_partial_aty(s, p->AT.dev, st, p->y[0].p, p->y[1].p, p->part.p, p->at_outpos.p);
          CUDA_OK(cudaEventRecord(ev[3], s));
          launch_p2p_barrier(s, 1, st, r2.partials, p->A.grid(), p->peers, p->world, p->rank, p->seg_len, p->shard_len,
                             p->epochs.p, p->fault.p);
          CUDA_OK(cudaEventRecord(ev[4], s));
          CUDA_OK(cudaEventSynchronize(ev[4]));
          p->launches += p->kernels_per_pass;
          for (int k = 0; k < 4; k++) { float t = 0.f; CUDA_OK(cudaEventElapsedTime(&t, ev[k], ev[k + 1])); acc[k] += t; }
          continue;
        }
        CUDA_OK(cudaEventRecord(ev[0], s));
        launch_primal_shard(s, p->nl, st, p->x[0].p, p->x[1].p, p->aty[0].p, p->red.p, p->cost.p, p->lower.p,
                            p->upper.p, p->xsum.p, p->send.p, r1);
        launch_stash_scalars(s, 1, st, r1.partials, primal_shard_grid(p->nl), p->send.p + p->shard_len, 1, 0);
        gather_shards(p);
        CUDA_OK(cudaEventRecord(ev[1], s));
        launch_spmv_dual_mg(s, p->A.dev, st, p->xfull.p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->rhs.p,
                            p->ysum.p, p->neq_local, r2);
        launch_stash_scalars(s, 2, st, r2.partials, p->A.grid(), p->part.p + p->shard_len, p->world, p->seg_len);
        CUDA_OK(cudaEventRecord(ev[2], s));
        launch_spmv_partial_aty(s, p->AT.dev, st, p->y[0].p, p->y[1].p, p->part.p, p->at_outpos.p);
        CUDA_OK(cudaEventRecord(ev[3], s));
        reduce_scatter_part(p);
        launch_step_rule_mg(s, st, p->xfull.p, p->world, p->seg_len, p->shard_len, p->red.p);
      }
      CUDA_OK(cudaEventRecord(ev[4], s));
      CUDA_OK(cudaEventSynchronize(ev[4]));
      p->launches += p->kernels_per_pass;
      for (int k = 0; k < 4; k++) {
        float t = 0.f;
        CUDA_OK(cudaEventElapsedTime(&t, ev[k], ev[k + 1]));
        acc[k] += t;
      }
    }
    for (auto& e : ev) cudaEventDestroy(e);
    for (int k = 0; k < 4; k++) ms[k] = (float)acc[k];
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_problem_solve(b200pdlp_problem* p, const b200pdlp_params* params, const b200pdlp_warm* warm, b200pdlp_result* out) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !params || !out) throw Error(B200PDLP_ERR_ARG, "null argument");
    out->setup_seconds = 0.0;
    solve_on_device(p, *params, warm, out);
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_solve(const b200pdlp_lp* lp, const b200pdlp_params* params, const b200pdlp_warm* warm, b200pdlp_result* out) {
  DeviceGuard dg;
  return guarded([&] {
    if (!params || !out) throw Error(B200PDLP_ERR_ARG, "null argument");
    check_params(*params);
    check_lp(lp, false);
    check_lp(lp, !use_device_prep(*lp, *params, 1));
    const auto t0 = std::chrono::steady_clock::now();
    ProblemPtr p(new b200pdlp_problem());
    if (use_device_prep(*lp, *params, 1)) create_problem_device(*lp, *params, p.get());
    else create_problem(*lp, *params, 0, 1, p.get());
    out->setup_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    solve_on_device(p.get(), *params, warm, out);
    CUDA_OK(cudaGetLastError());
    Laps lap;
    p.reset();
    lap("solve", "teardown");
  });
}

int b200pdlp_solve_batch(int32_t count, const b200pdlp_lp* lps, const b200pdlp_params* params, const b200pdlp_warm* warms,
                         b200pdlp_result* outs) {
  DeviceGuard dg;
  return guarded([&] {
    if (count < 0) throw Error(B200PDLP_ERR_ARG, "b200pdlp_solve_batch: count < 0");
    if (count == 0) return;
    if (!lps || !params || !outs) throw Error(B200PDLP_ERR_ARG, "b200pdlp_solve_batch: null argument");
    check_params(*params);
    for (int i = 0; i < count; i++) check_batch_member(&lps[i], *params, i);
    solve_batch(count, lps, *params, warms, outs);
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_solve_batch_device(int32_t count, const b200pdlp_lp* lps, const b200pdlp_params* params, const b200pdlp_warm* warms,
                                b200pdlp_result* outs) {
  DeviceGuard dg;
  return guarded([&] {
    if (count < 0) throw Error(B200PDLP_ERR_ARG, "b200pdlp_solve_batch_device: count < 0");
    if (count == 0) return;
    if (!lps || !params || !outs) throw Error(B200PDLP_ERR_ARG, "b200pdlp_solve_batch_device: null argument");
    check_params(*params);
    for (int i = 0; i < count; i++) check_batch_device_member(&lps[i], params->ordered_max, i, "b200pdlp_solve_batch_device");
    solve_batch_device(count, lps, *params, warms, outs);
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_debug_batch_prep_compare(int32_t count, const b200pdlp_lp* lps, int32_t scaling, double* report) {
  DeviceGuard dg;
  return guarded([&] {
    if (count < 0 || (count > 0 && (!lps || !report))) throw Error(B200PDLP_ERR_ARG, "b200pdlp_debug_batch_prep_compare: bad arguments");
    for (int i = 0; i < count; i++) check_lp(&lps[i]);
    if (count > 0) batch_prep_compare(count, lps, scaling, report);
  });
}

int b200pdlp_solve_hipdlp_batch(int32_t count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params* params,
                                b200pdlp_result* outs) {
  DeviceGuard dg;
  return guarded([&] {
    if (count < 0) throw Error(B200PDLP_ERR_ARG, "b200pdlp_solve_hipdlp_batch: count < 0");
    if (count == 0) return;
    if (!lps || !params || !outs) throw Error(B200PDLP_ERR_ARG, "b200pdlp_solve_hipdlp_batch: null argument");
    for (int i = 0; i < count; i++) check_hipdlp_batch_member(&lps[i], *params, i);
    solve_hipdlp_batch(count, lps, *params, outs);
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_solve_hipdlp_batch_device(int32_t count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params* params,
                                       b200pdlp_result* outs) {
  DeviceGuard dg;
  return guarded([&] {
    const char* who = "b200pdlp_solve_hipdlp_batch_device";
    if (count < 0) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": count < 0");
    if (count == 0) return;
    if (!lps || !params || !outs) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": null argument");
    for (int i = 0; i < count; i++) check_batch_device_member(&lps[i], params->ordered_max, i, who);
    solve_hipdlp_batch_device(count, lps, *params, outs);
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_kkt_check_batch(int32_t count, const b200pdlp_lp* lps, const b200pdlp_solution* sols,
                             const b200pdlp_kkt_tolerances* tol, int32_t device, b200pdlp_kkt_info* inout) {
  return kkt_check_batch_entry(false, count, lps, sols, tol, device, inout);
}

int b200pdlp_kkt_check_batch_device(int32_t count, const b200pdlp_lp* lps, const b200pdlp_solution* sols,
                                    const b200pdlp_kkt_tolerances* tol, int32_t device, b200pdlp_kkt_info* inout) {
  return kkt_check_batch_entry(true, count, lps, sols, tol, device, inout);
}

int b200pdlp_debug_hipdlp_batch_prep_compare(int32_t count, const b200pdlp_lp* lps, int32_t scaling_mode, int32_t ruiz_iterations,
                                             double* report) {
  DeviceGuard dg;
  return guarded([&] {
    if (count < 0 || (count > 0 && (!lps || !report)))
      throw Error(B200PDLP_ERR_ARG, "b200pdlp_debug_hipdlp_batch_prep_compare: bad arguments");
    for (int i = 0; i < count; i++) check_lp(&lps[i]);
    if (count > 0) hipdlp_batch_prep_compare(count, lps, scaling_mode, ruiz_iterations, report);
  });
}

// One process, several GPUs (what a HiGHS process would do: Highs::run() is not an MPI program): one problem per
// device, wired to each other with b200pdlp_p2p_link_local (peer access instead of CUDA IPC, no NCCL), one host
// thread per rank.  The standard form is formulated and scaled once and copied to the other ranks.
int b200pdlp_solve_multi(const b200pdlp_lp* lp, const b200pdlp_params* params, const b200pdlp_warm* warm,
                         b200pdlp_result* out, int32_t ngpus, const int32_t* devices) {
  if (ngpus <= 1) return b200pdlp_solve(lp, params, warm, out);
  // fixed-step mode needs the power method, which is single-GPU (power_method): fall back instead of failing
  if (params && params->adaptive_step == 0) return b200pdlp_solve(lp, params, warm, out);
  DeviceGuard dg;
  std::vector<ProblemPtr> owned;
  const int rc = guarded([&] {
    check_lp(lp);
    if (!params || !out || ngpus > kMaxPeers) throw Error(B200PDLP_ERR_ARG, "b200pdlp_solve_multi: bad arguments");
    check_params(*params);
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<b200pdlp_problem*> probs((size_t)ngpus, nullptr);
    for (int g = 0; g < ngpus; g++) {
      b200pdlp_params prm = *params;
      prm.device = devices ? devices[g] : g;
      owned.emplace_back(probs[g] = new b200pdlp_problem());
      create_problem(*lp, prm, g, ngpus, probs[g], g == 0 ? nullptr : &probs[0]->form);
    }
    const int lrc = b200pdlp_p2p_link_local(probs.data(), ngpus);
    if (lrc != B200PDLP_OK) throw Error(lrc, g_last_error);
    const double setup = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    // every rank assembles the complete solution; ranks > 0 write theirs into scratch
    const size_t n = (size_t)std::max(lp->num_col, 1), m = (size_t)std::max(lp->num_row, 1);
    std::vector<std::vector<double>> scratch((size_t)ngpus);
    std::vector<b200pdlp_result> res((size_t)ngpus);
    for (int g = 0; g < ngpus; g++) {
      res[g] = *out;
      res[g].setup_seconds = 0.0;
      if (g > 0) {
        scratch[g].assign(2 * n + 2 * m, 0.0);
        res[g].col_value = scratch[g].data(); res[g].col_dual = scratch[g].data() + n;
        res[g].row_value = scratch[g].data() + 2 * n; res[g].row_dual = scratch[g].data() + 2 * n + m;
        res[g].trace = nullptr; res[g].trace_cap = 0;
      }
    }
    run_per_rank(ngpus, "rank", [&](int g) {
      b200pdlp_params prm = *params;
      prm.device = probs[g]->device;
      solve_on_device(probs[g], prm, warm, &res[g]);
      CUDA_OK(cudaGetLastError());
    });
    *out = res[0];
    out->setup_seconds += setup;
  });
  for (ProblemPtr& p : owned) p->p2p = false;
  return rc;
}

int b200pdlp_hipdlp_controller_replay(double norm_cost, double norm_rhs, double op_norm_sq, double tolerance, int32_t strategy,
                                       int32_t nblocks, const double* sums, const double* restart_sums, double* out) {
  if (nblocks < 0 || (nblocks > 0 && (!sums || !restart_sums || !out))) return B200PDLP_ERR_ARG;
  HipController ctl;
  ctl.init(norm_cost, norm_rhs, op_norm_sq, tolerance, strategy);
  for (int b = 0; b < nblocks; b++) {
    if (ctl.pending_restart_fpe) ctl.restart_reference(restart_sums + 3 * (size_t)b);
    const bool restart = ctl.after_block(sums + 9 * (size_t)b);
    double* o = out + 8 * (size_t)b;
    o[0] = restart ? 1.0 : 0.0; o[1] = ctl.primal_weight; o[2] = ctl.primal_step; o[3] = ctl.dual_step; o[4] = ctl.fpe;
    o[5] = (ctl.pfeas < ctl.tol * (1.0 + norm_rhs) && ctl.dfeas < ctl.tol * (1.0 + norm_cost) && ctl.relgap < ctl.tol) ? 1.0 : 0.0;
    o[6] = ctl.iters; o[7] = ctl.halpern_iteration;
  }
  return B200PDLP_OK;
}

void b200pdlp_hipdlp_default_params(b200pdlp_hipdlp_params* p) {
  memset(p, 0, sizeof(*p));
  p->tolerance = 1e-7;
  p->iter_limit = 2147483647;
  p->scaling_mode = 5;
  p->ruiz_iterations = 10;
  p->step_size_strategy = 3;
  p->time_limit = -1.0;
  p->device = -1;
}

int b200pdlp_solve_hipdlp(const b200pdlp_lp* lp, const b200pdlp_hipdlp_params* params, b200pdlp_result* out) {
  DeviceGuard dg;
  return guarded([&] {
    check_lp(lp);
    if (!params || !out) throw Error(B200PDLP_ERR_ARG, "null argument");
    const auto t0 = std::chrono::steady_clock::now();
    ProblemPtr p(new b200pdlp_problem());
    create_problem_hipdlp(*lp, *params, p.get());
    out->setup_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    solve_hipdlp_on_device(p.get(), *lp, *params, out);
    CUDA_OK(cudaGetLastError());
  });
}

// The HiPDLP mode on several devices of this process: the prologue once per device (device prologue in block mode) or once
// on the host (ordered mode, device_prep = -1), then one problem per rank (its blocks of the one-GPU device orders), wired by
// peer pointers, one host thread per rank, no NCCL.
int b200pdlp_solve_hipdlp_multi(const b200pdlp_lp* lp, const b200pdlp_hipdlp_params* params, b200pdlp_result* out,
                                int32_t ngpus, const int32_t* devices) {
  if (ngpus <= 1) return b200pdlp_solve_hipdlp(lp, params, out);
  DeviceGuard dg;
  return guarded([&] {
    check_lp(lp);
    if (!params || !out || ngpus > kMaxPeers) throw Error(B200PDLP_ERR_ARG, "b200pdlp_solve_hipdlp_multi: bad arguments");
    const int ndev = device_count_checked();
    std::vector<int> dev(ngpus);
    for (int g = 0; g < ngpus; g++) {
      dev[g] = devices ? devices[g] : g;
      if (dev[g] < 0 || dev[g] >= ndev) throw Error(B200PDLP_ERR_ARG, "b200pdlp_solve_hipdlp_multi: no such device");
    }
    for (int a : dev)   // every rank stores into every other rank's memory
      for (int b : dev)
        if (a != b) {
          int ok = 0;
          CUDA_OK(cudaDeviceCanAccessPeer(&ok, a, b));
          if (!ok) throw Error(B200PDLP_ERR_ARG, "b200pdlp_solve_hipdlp_multi: devices cannot access each other");
        }
    const auto t0 = std::chrono::steady_clock::now();
    Laps lap;
    std::vector<ProblemPtr> owned;
    std::vector<b200pdlp_problem*> probs;
    for (int g = 0; g < ngpus; g++) { owned.emplace_back(new b200pdlp_problem()); probs.push_back(owned.back().get()); }
    if (use_device_prep_hipdlp(*lp, *params)) {
      create_hipdlp_shards_device(*lp, *params, dev, probs);
      lap("setup", "HiPDLP shards: device prologue");
    } else {
      StdForm f;
      formulate_hipdlp(*lp, f);
      scale_hipdlp(f, params->scaling_mode, params->ruiz_iterations);
      HipShards S;
      plan_hipdlp_shards(f, ngpus, params->ordered_max, S);
      for (int g = 0; g < ngpus; g++) create_problem_hipdlp_shard(f, S, g, dev[g], probs[g]);
      probs[0]->form = std::move(f);
      lap("setup", "HiPDLP shards: host prologue");
    }
    auto group = std::make_shared<LocalGroup>();
    group->world = ngpus;
    for (b200pdlp_problem* p : probs) {
      set_device(p);
      preload_hipdlp_shard_kernels();
      for (b200pdlp_problem* q : probs)
        if (q->device != p->device) {
          const cudaError_t pe = cudaDeviceEnablePeerAccess(q->device, 0);
          if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) CUDA_OK(pe);
          cudaGetLastError();
        }
      p->hip_peers = probs;
      p->group = group;
      p->local_link = true;
    }
    const double setup = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    // rank 0 writes the caller's arrays; the other ranks' results carry no vectors
    std::vector<b200pdlp_result> res((size_t)ngpus, *out);
    for (int g = 0; g < ngpus; g++) {
      res[g].setup_seconds = 0.0;
      if (g > 0) { res[g].col_value = res[g].col_dual = res[g].row_value = res[g].row_dual = nullptr; res[g].trace = nullptr; res[g].trace_cap = 0; }
    }
    run_per_rank(ngpus, "rank", [&](int g) {
      solve_hipdlp_on_device(probs[g], *lp, *params, &res[g]);
      CUDA_OK(cudaGetLastError());
    });
    *out = res[0];
    out->setup_seconds += setup;
  });
}

int b200pdlp_hipdlp_shard_layout_eval(b200pdlp_form* fh, int32_t rank, int32_t world, int32_t ordered_max, const double* x,
                                      const double* y, double* ax, double* aty, double stats[7]) {
  return guarded([&] {
    if (!fh || !x || !y || !ax || !aty || !stats) throw Error(B200PDLP_ERR_ARG, "null argument");
    if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world) throw Error(B200PDLP_ERR_ARG, "bad rank/world");
    StdForm& f = fh->f;
    if (!f.hipdlp) throw Error(B200PDLP_ERR_ARG, "b200pdlp_hipdlp_shard_layout_eval needs a HiPDLP form");
    HipShards S;
    plan_hipdlp_shards(f, world, ordered_max, S);
    SellMatrix A, AT;
    build_hipdlp_shard(S, rank, A, AT);
    const int n = f.n, m = f.m;
    const int r0 = S.rb[rank], r1 = S.rb[rank + 1], c0 = S.cb[rank], c1 = S.cb[rank + 1];
    std::vector<double> xin((size_t)std::max(n, 1), 0.0), yin((size_t)std::max(m, 1), 0.0);
    std::vector<double> rows((size_t)std::max(r1 - r0, 1)), cols((size_t)std::max(c1 - c0, 1));
    for (int j = 0; j < n; j++) xin[j] = x[S.cperm[j]];
    for (int i = 0; i < m; i++) yin[i] = y[S.rperm[i]];
    sell_apply_host(A, xin.data(), rows.data());
    sell_apply_host(AT, yin.data(), cols.data());
    for (int i = r0; i < r1; i++) ax[S.rperm[i]] = rows[i - r0];
    for (int j = c0; j < c1; j++) aty[S.cperm[j]] = cols[j - c0];
    stats[0] = r0; stats[1] = r1; stats[2] = c0; stats[3] = c1; stats[4] = S.ordered ? 1 : 0;
    stats[5] = (double)A.long_rows.size(); stats[6] = (double)AT.long_rows.size();
  });
}

int b200pdlp_nccl_unique_id(uint8_t id[128]) {
  return guarded([&] {
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId u;
    NCCL_OK(nccl().GetUniqueId(&u));
    memcpy(id, &u, 128);
  });
}

int b200pdlp_comm_init(b200pdlp_problem* p, const uint8_t id[128]) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !id) throw Error(B200PDLP_ERR_ARG, "null argument");
    set_device(p);
    ncclUniqueId u;
    memcpy(&u, id, 128);
    NCCL_OK(nccl().CommInitRank(&p->comm, p->world, u, p->rank));
  });
}

int b200pdlp_p2p_timeline(b200pdlp_problem* p, double out_us[8]) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !out_us || !p->p2p) throw Error(B200PDLP_ERR_ARG, "p2p_timeline needs the fused multi-GPU path");
    set_device(p);
    unsigned long long h[16];
    CUDA_OK(cudaMemcpy(h, p->epochs.p, sizeof(h), cudaMemcpyDeviceToHost));
    const double c = h[9] ? 1e-3 / (double)h[9] : 0.0;
    // per-pass averages in us: primal-shard phase, barrier 0 total, barrier 0 wait, Ax+A'y phase, barrier 1 total,
    // barrier 1 wait, passes counted
    out_us[0] = h[3] * c; out_us[1] = h[4] * c; out_us[2] = h[5] * c; out_us[3] = h[6] * c; out_us[4] = h[7] * c;
    out_us[5] = h[8] * c; out_us[6] = (double)h[9]; out_us[7] = 0.0;
    unsigned long long z[8] = {0};   // [2..9] only: [0],[1],[10] are live barrier epochs
    CUDA_OK(cudaMemcpy(p->epochs.p + 2, z, sizeof(z), cudaMemcpyHostToDevice));
  });
}

int b200pdlp_p2p_export(b200pdlp_problem* p, uint8_t handles[B200PDLP_IPC_BYTES]) {
  DeviceGuard dg;
  return guarded([&] {
    static_assert(4 * sizeof(cudaIpcMemHandle_t) == B200PDLP_IPC_BYTES, "IPC blob size");
    if (!p || !handles || p->world < 2) throw Error(B200PDLP_ERR_ARG, "p2p_export needs a multi-GPU problem");
    set_device(p);
    cudaIpcMemHandle_t h[4];
    CUDA_OK(cudaIpcGetMemHandle(&h[0], p->part.p));
    CUDA_OK(cudaIpcGetMemHandle(&h[1], p->xfull.p));
    CUDA_OK(cudaIpcGetMemHandle(&h[2], p->flags.p));
    CUDA_OK(cudaIpcGetMemHandle(&h[3], p->recv.p));
    memcpy(handles, h, sizeof(h));
  });
}

int b200pdlp_p2p_import(b200pdlp_problem* p, const uint8_t* all_handles) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !all_handles || p->world < 2) throw Error(B200PDLP_ERR_ARG, "p2p_import needs a multi-GPU problem");
    if (p->world > kMaxPeers) throw Error(B200PDLP_ERR_ARG, "too many ranks for the P2P path");
    set_device(p);
    for (int g = 0; g < p->world; g++) {
      if (g == p->rank) {
        p->peers.part[g] = p->part.p; p->peers.xfull[g] = p->xfull.p; p->peers.flags[g] = p->flags.p;
        p->peers.recv[g] = p->recv.p;
        continue;
      }
      cudaIpcMemHandle_t h[4];
      memcpy(h, all_handles + (size_t)g * B200PDLP_IPC_BYTES, sizeof(h));
      void* q[4];
      for (int k = 0; k < 4; k++) {
        CUDA_OK(cudaIpcOpenMemHandle(&q[k], h[k], cudaIpcMemLazyEnablePeerAccess));
        p->ipc_opened.push_back(q[k]);
      }
      p->peers.part[g] = (double*)q[0]; p->peers.xfull[g] = (double*)q[1]; p->peers.flags[g] = (unsigned long long*)q[2];
      p->peers.recv[g] = (double*)q[3];
    }
    p->p2p = true;
    // graphs captured for the NCCL path are stale now
    drop_graphs(p);
  });
}

int b200pdlp_p2p_link_local(b200pdlp_problem** probs, int32_t count) {
  DeviceGuard dg;
  return guarded([&] {
    if (!probs || count < 2 || count > kMaxPeers) throw Error(B200PDLP_ERR_ARG, "p2p_link_local: bad arguments");
    std::vector<b200pdlp_problem*> by_rank(count, nullptr);
    for (int k = 0; k < count; k++) {
      b200pdlp_problem* p = probs[k];
      if (!p || p->world != count || p->rank < 0 || p->rank >= count || by_rank[p->rank])
        throw Error(B200PDLP_ERR_ARG, "p2p_link_local: need exactly one problem per rank of the same world");
      by_rank[p->rank] = p;
    }
    for (int k = 0; k < count; k++)
      if (by_rank[k]->device != by_rank[0]->device) {
        int ok = 0;
        CUDA_OK(cudaDeviceCanAccessPeer(&ok, by_rank[k]->device, by_rank[0]->device));
        if (!ok) throw Error(B200PDLP_ERR_ARG, "p2p_link_local: devices cannot access each other");
      }
    auto group = std::make_shared<LocalGroup>();
    group->world = count;
    for (int k = 0; k < count; k++) { set_device(by_rank[k]); preload_multi_gpu_kernels(); }
    for (int k = 0; k < count; k++) {
      b200pdlp_problem* p = by_rank[k];
      set_device(p);
      for (int g = 0; g < count; g++) {
        if (by_rank[g]->device != p->device) {
          const cudaError_t e = cudaDeviceEnablePeerAccess(by_rank[g]->device, 0);
          if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CUDA_OK(e);
          cudaGetLastError();
        }
        p->peers.part[g] = by_rank[g]->part.p; p->peers.xfull[g] = by_rank[g]->xfull.p;
        p->peers.flags[g] = by_rank[g]->flags.p; p->peers.recv[g] = by_rank[g]->recv.p;
      }
      p->p2p = true;
      p->local_link = true;
      p->group = group;
      drop_graphs(p);
    }
  });
}

int b200pdlp_p2p_release(b200pdlp_problem* p) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p) throw Error(B200PDLP_ERR_ARG, "null argument");
    set_device(p);
    CUDA_OK(cudaStreamSynchronize(p->stream));
    for (void* q : p->ipc_opened) cudaIpcCloseMemHandle(q);
    p->ipc_opened.clear();
    p->p2p = false;
    p->local_link = false;
    p->group.reset();
    drop_graphs(p);
  });
}

int b200pdlp_form_create(const b200pdlp_lp* lp, int32_t scaling, b200pdlp_form** out) {
  return guarded([&] {
    check_lp(lp);
    if (!out) throw Error(B200PDLP_ERR_ARG, "null argument");
    auto* f = new b200pdlp_form();
    formulate(*lp, f->f);
    scale(f->f, scaling != 0);
    *out = f;
  });
}
int b200pdlp_hipdlp_form_create(const b200pdlp_lp* lp, int32_t scaling_mode, int32_t ruiz_iterations, b200pdlp_form** out) {
  return guarded([&] {
    check_lp(lp);
    if (!out || ruiz_iterations < 0) throw Error(B200PDLP_ERR_ARG, "bad argument");
    auto* f = new b200pdlp_form();
    formulate_hipdlp(*lp, f->f);
    scale_hipdlp(f->f, scaling_mode, ruiz_iterations);
    *out = f;
  });
}
int b200pdlp_hipdlp_power_method(const b200pdlp_form* f, double* lambda) {
  if (!f || !lambda || !f->f.hipdlp) return B200PDLP_ERR_ARG;
  *lambda = power_method_hipdlp(f->f);
  return B200PDLP_OK;
}
void b200pdlp_form_destroy(b200pdlp_form* f) { delete f; }
int b200pdlp_form_dims(const b200pdlp_form* f, int32_t dims[5], double scalars[3]) {
  if (!f || !dims || !scalars) return B200PDLP_ERR_ARG;
  dims[0] = f->f.n; dims[1] = f->f.m; dims[2] = f->f.nnz; dims[3] = f->f.neq; dims[4] = f->f.n_orig;
  scalars[0] = f->f.norm_cost; scalars[1] = f->f.norm_rhs; scalars[2] = f->f.amax;
  return B200PDLP_OK;
}
static const std::vector<double>* form_vector(const StdForm& f, int which) {
  switch (which) {
    case 0: return &f.cost;
    case 1: return &f.lower;
    case 2: return &f.upper;
    case 3: return &f.rhs;
    case 4: return &f.col_scale;
    case 5: return &f.row_scale;
    case 6: return &f.row_upper;   // HiPDLP forms only (empty otherwise)
  }
  return nullptr;
}
int b200pdlp_form_get_vector(const b200pdlp_form* f, int32_t which, double* dst, int32_t cap) {
  if (!f || !dst) return B200PDLP_ERR_ARG;
  const std::vector<double>* v = form_vector(f->f, which);
  if (!v) return B200PDLP_ERR_ARG;
  const int k = std::min<int>(cap, (int)v->size());
  memcpy(dst, v->data(), (size_t)k * sizeof(double));
  return k;
}
int b200pdlp_form_get_csc(const b200pdlp_form* f, int32_t* start, int32_t* index, double* value) {
  if (!f || !start || !index || !value) return B200PDLP_ERR_ARG;
  memcpy(start, f->f.cbeg.data(), (size_t)(f->f.n + 1) * sizeof(int));
  memcpy(index, f->f.cidx.data(), (size_t)f->f.nnz * sizeof(int));
  memcpy(value, f->f.cval.data(), (size_t)f->f.nnz * sizeof(double));
  return B200PDLP_OK;
}
int b200pdlp_form_get_csr(b200pdlp_form* f, int32_t* rowptr, int32_t* col, double* val) {
  return guarded([&] {
    if (!f || !rowptr || !col || !val) throw Error(B200PDLP_ERR_ARG, "null argument");
    if (f->f.rptr.empty()) build_row_index(f->f);
    Csr a;
    build_row_major(f->f, 0, f->f.m, a);
    memcpy(rowptr, a.rowptr.data(), (size_t)(a.nrows + 1) * sizeof(int));
    memcpy(col, a.col.data(), (size_t)a.nnz * sizeof(int));
    memcpy(val, a.val.data(), (size_t)a.nnz * sizeof(double));
  });
}
int b200pdlp_form_get_row_map(const b200pdlp_form* f, int32_t* row_new_idx, int32_t* row_class) {
  if (!f || !row_new_idx || !row_class) return B200PDLP_ERR_ARG;
  memcpy(row_new_idx, f->f.row_new_idx.data(), (size_t)f->f.m * sizeof(int));
  memcpy(row_class, f->f.row_class.data(), (size_t)f->f.m * sizeof(int));
  return B200PDLP_OK;
}

int b200pdlp_form_layout_eval(b200pdlp_form* fh, int32_t rank, int32_t world, int32_t ordered_max, const double* x,
                              const double* y, double* ax, double* aty, double stats[12]) {
  return guarded([&] {
    if (!fh || !x || !y || !ax || !aty || !stats) throw Error(B200PDLP_ERR_ARG, "null argument");
    if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world) throw Error(B200PDLP_ERR_ARG, "bad rank/world");
    StdForm& f = fh->f;
    const bool timing = getenv("B200PDLP_TIMING") != nullptr;
    auto t0 = std::chrono::steady_clock::now();
    auto tl = t0;
    HostLayout L;
    build_layout(f, rank, world, ordered_max, L, [&](const char* what) {
      if (!timing) return;
      auto t1 = std::chrono::steady_clock::now();
      fprintf(stderr, "[b200pdlp layout] %-28s %8.1f ms\n", what, std::chrono::duration<double, std::milli>(t1 - tl).count());
      tl = t1;
    });
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (world == 1) {
      // the plan-only path (device-side fill) must produce the same orderings and descriptors
      HostLayout P;
      build_layout(f, rank, world, ordered_max, P, nullptr, /*plan_only=*/true);
      auto same_plan = [](const SellMatrix& a, const SellMatrix& b) {
        return a.nrows == b.nrows && a.padded == b.padded && a.lcount == b.lcount && a.n_partials == b.n_partials &&
               a.slices.size() == b.slices.size() && a.segs.size() == b.segs.size() && a.long_rows.size() == b.long_rows.size() &&
               (a.slices.empty() || !memcmp(a.slices.data(), b.slices.data(), a.slices.size() * sizeof(a.slices[0]))) &&
               (a.segs.empty() || !memcmp(a.segs.data(), b.segs.data(), a.segs.size() * sizeof(a.segs[0]))) &&
               (a.long_rows.empty() || !memcmp(a.long_rows.data(), b.long_rows.data(), a.long_rows.size() * sizeof(a.long_rows[0])));
      };
      if (P.rperm != L.rperm || P.cperm != L.cperm || !same_plan(P.A, L.A) || !same_plan(P.AT, L.AT))
        throw Error(B200PDLP_ERR_STATE, "plan-only layout differs from the full layout");
    }
    const int n = f.n, ml = L.ml;
    // x in the kernel-facing layout: device column order, segmented when world > 1
    std::vector<double> xin((size_t)L.world * L.seg_len + 8, 0.0), out_rows((size_t)std::max(ml, 1), 0.0);
    for (int j = 0; j < n; j++) xin[L.seg_pos(j)] = x[L.cperm[j]];
    sell_apply_host(L.A, xin.data(), out_rows.data());
    for (int i = 0; i < ml; i++) ax[L.r0 + L.rperm[i]] = out_rows[i];
    // y of the local rows in device row order
    std::vector<double> yin((size_t)std::max(ml, 1) + 8, 0.0), out_cols((size_t)std::max(n, 1), 0.0);
    for (int i = 0; i < ml; i++) yin[i] = y[L.r0 + L.rperm[i]];
    sell_apply_host(L.AT, yin.data(), out_cols.data());
    if (world == 1) {
      for (int j = 0; j < n; j++) aty[L.cperm[j]] = out_cols[j];
    } else {
      // the kernel writes body row r to part[at_outpos[r]]; undo the segmentation, then the column order
      std::vector<double> part((size_t)L.world * L.seg_len, 0.0);
      for (int r = 0; r < n; r++) part[L.at_outpos[r]] = out_cols[r];
      for (int j = 0; j < n; j++) aty[L.cperm[j]] = part[L.seg_pos(j)];
    }
    stats[0] = L.r0; stats[1] = L.r1; stats[2] = L.ordered ? 1 : 0;
    stats[3] = (double)L.A.padded; stats[4] = (double)L.A.long_rows.size(); stats[5] = (double)L.A.segs.size();
    stats[6] = (double)L.AT.padded; stats[7] = (double)L.AT.long_rows.size(); stats[8] = (double)L.AT.segs.size();
    stats[9] = L.shard_len; stats[10] = L.seg_len; stats[11] = ms;
  });
}

// the device prologue against its host twin, array by array, bit for bit (report[0..31], see include/b200pdlp.h); false if
// the sizes differ (nothing else is compared then)
static double cmp_dev_i(const int* dev, const int* host, size_t cnt) {
  std::vector<int> t(cnt);
  if (cnt) CUDA_OK(cudaMemcpy(t.data(), dev, cnt * sizeof(int), cudaMemcpyDeviceToHost));
  double bad = 0;
  for (size_t i = 0; i < cnt; i++) bad += t[i] != host[i];
  return bad;
}
static double cmp_dev_d(const double* dev, const double* host, size_t cnt) {
  std::vector<double> t(cnt);
  if (cnt) CUDA_OK(cudaMemcpy(t.data(), dev, cnt * sizeof(double), cudaMemcpyDeviceToHost));
  double bad = 0;
  for (size_t i = 0; i < cnt; i++) bad += memcmp(&t[i], &host[i], sizeof(double)) != 0;
  return bad;
}
// one sliced-ELL matrix of the device prologue against the host's: *r_slices = -1 if the sizes differ
static void cmp_sell(const DevSellOwned& D, const SellMatrix& H, double* r_slices, double* r_col, double* r_val, double* r_long) {
  if ((size_t)D.nslices != H.slices.size() || D.padded != H.padded || (size_t)D.nlong != H.long_rows.size() ||
      (size_t)D.nsegs != H.segs.size() || D.lcount != H.lcount) { *r_slices = -1; return; }
  *r_slices = cmp_dev_i(reinterpret_cast<const int*>(D.slices), reinterpret_cast<const int*>(H.slices.data()), 4 * H.slices.size());
  *r_col = cmp_dev_i(D.col, H.col.data(), (size_t)H.padded);
  *r_val = cmp_dev_d(D.val, H.val.data(), (size_t)H.padded);
  *r_long = cmp_dev_i(reinterpret_cast<const int*>(D.long_rows), reinterpret_cast<const int*>(H.long_rows.data()), 4 * H.long_rows.size()) +
            cmp_dev_i(reinterpret_cast<const int*>(D.segs), reinterpret_cast<const int*>(H.segs.data()), 4 * H.segs.size()) +
            cmp_dev_i(D.lcol, H.lcol.data(), H.lcol.size()) + cmp_dev_d(D.lval, H.lval.data(), H.lval.size());
}
static bool prep_compare_arrays(const DevicePrologue& P, const StdForm& f, const HostLayout& L, double* report) {
  const auto cmp_i = cmp_dev_i;
  const auto cmp_d = cmp_dev_d;
  const DevProblemArrays& a = P.arr;
  const int n = f.n, m = f.m, nnz = f.nnz;
  report[0] = a.n != n; report[1] = a.m != m; report[2] = a.nnz != nnz; report[3] = a.neq != f.neq;
  if (report[0] + report[1] + report[2] + report[3] > 0) return false;
  report[4] = cmp_i(P.form.cbeg, f.cbeg.data(), n + 1);
  report[5] = cmp_i(P.form.cidx, f.cidx.data(), nnz);
  report[6] = cmp_d(P.form.cval, f.cval.data(), nnz);
  report[7] = cmp_d(P.form.cost, f.cost.data(), n);
  report[8] = cmp_d(P.form.lower, f.lower.data(), n);
  report[9] = cmp_d(P.form.upper, f.upper.data(), n);
  report[10] = cmp_d(P.form.colscale, f.col_scale.data(), n);
  report[11] = cmp_d(P.form.rhs, f.rhs.data(), m);
  report[12] = cmp_d(P.form.rowscale, f.row_scale.data(), m);
  report[13] = cmp_i(P.form.rptr, f.rptr.data(), m + 1);
  report[14] = cmp_i(P.form.rpos, f.rpos.data(), nnz);
  report[15] = cmp_i(a.row_new_idx, f.row_new_idx.data(), m);
  report[16] = cmp_i(a.row_class, f.row_class.data(), m);
  report[17] = cmp_i(a.rperm, L.rperm.data(), m);
  report[18] = cmp_i(a.cperm, L.cperm.data(), n);
  cmp_sell(P.A, L.A, report + 19, report + 20, report + 21, report + 25);
  cmp_sell(P.AT, L.AT, report + 22, report + 23, report + 24, report + 26);
  report[27] = P.sc.amax != f.amax;
  report[28] = std::fabs(std::sqrt(P.sc.norm_cost_sq) - f.norm_cost) / (1.0 + f.norm_cost);
  report[29] = std::fabs(std::sqrt(P.sc.norm_rhs_sq) - f.norm_rhs) / (1.0 + f.norm_rhs);
  {
    std::vector<double> t(std::max(n, m));
    double bad = 0;
    auto cmp_perm = [&](const double* dev, const std::vector<double>& v, const std::vector<int>& perm, int len) {
      for (int i = 0; i < len; i++) t[i] = v[perm[i]];
      bad += cmp_d(dev, t.data(), len);
    };
    cmp_perm(a.cost, f.cost, L.cperm, n); cmp_perm(a.lower, f.lower, L.cperm, n); cmp_perm(a.upper, f.upper, L.cperm, n);
    cmp_perm(a.colscale, f.col_scale, L.cperm, n); cmp_perm(a.rhs, f.rhs, L.rperm, m); cmp_perm(a.rowscale, f.row_scale, L.rperm, m);
    report[30] = bad;
  }
  report[31] = P.sc.cols_sorted;
  return true;
}

// Test entry point: the device prologue (device_prep.cu) against its host twin (host_prep.cpp), array by array, bit for
// bit.  report[k] = number of mismatching entries of item k (0 everywhere = identical), see include/b200pdlp.h.
int b200pdlp_debug_prep_compare(const b200pdlp_lp* lp, int32_t scaling, double report[32]) {
  DeviceGuard dg;
  return guarded([&] {
    check_lp(lp);
    if (!report) throw Error(B200PDLP_ERR_ARG, "null argument");
    for (int k = 0; k < 32; k++) report[k] = 0.0;
    StdForm f;
    formulate(*lp, f);
    scale(f, scaling != 0);
    if (f.rptr.empty()) build_row_index(f);
    HostLayout L;
    build_layout(f, 0, 1, /*ordered_max=*/-1, L);
    TempPrologue T;
    T.P.keep_form = true;
    run_prologue(T.P, T.stream, *lp, scaling != 0);
    prep_compare_arrays(T.P, f, L, report);
  });
}

// The same for the HiPDLP mode's prologue (DevicePrologue::hipdlp against host_prep_hipdlp.cpp); report[32..39] adds the
// HiPDLP items, see include/b200pdlp.h.
int b200pdlp_debug_prep_compare_hipdlp(const b200pdlp_lp* lp, int32_t scaling_mode, int32_t ruiz_iterations, double report[40]) {
  DeviceGuard dg;
  return guarded([&] {
    check_lp(lp);
    if (!report) throw Error(B200PDLP_ERR_ARG, "null argument");
    for (int k = 0; k < 40; k++) report[k] = 0.0;
    StdForm f;
    formulate_hipdlp(*lp, f);
    scale_hipdlp(f, scaling_mode, ruiz_iterations);
    if (f.rptr.empty()) build_row_index(f);
    HostLayout L;
    build_layout(f, 0, 1, /*ordered_max=*/-1, L);
    TempPrologue T;
    DevicePrologue& P = T.P;
    P.keep_form = true;
    P.hipdlp = true;
    P.scaling_mode = scaling_mode;
    P.ruiz_iterations = ruiz_iterations;
    run_prologue(P, T.stream, *lp, true);
    if (!prep_compare_arrays(P, f, L, report)) return;
    const int m = f.m, n0 = lp->num_col, nnz0 = lp->a_start[n0];
    // the norms set omega and both step sizes: bitwise
    const double nc = std::sqrt(P.sc.norm_cost_sq), nr = std::sqrt(P.sc.norm_rhs_sq);
    report[28] = memcmp(&nc, &f.norm_cost, sizeof(double)) != 0;
    report[29] = memcmp(&nr, &f.norm_rhs, sizeof(double)) != 0;
    report[32] = cmp_dev_d(P.form.row_upper, f.row_upper.data(), m);
    {
      std::vector<double> t(m);
      for (int i = 0; i < m; i++) t[i] = f.row_upper[L.rperm[i]];
      report[33] = cmp_dev_d(P.arr.rup, t.data(), m);
    }
    {
      // row-major copy of the caller's matrix: counting sort of the positions by row (a row's entries in column order)
      std::vector<int> ptr(m + 1, 0), col(nnz0), fill;
      std::vector<double> val(nnz0);
      for (int q = 0; q < nnz0; q++) ptr[lp->a_index[q] + 1]++;
      for (int i = 0; i < m; i++) ptr[i + 1] += ptr[i];
      fill.assign(ptr.begin(), ptr.end() - 1);
      for (int j = 0; j < n0; j++)
        for (int q = lp->a_start[j]; q < lp->a_start[j + 1]; q++) { const int k = fill[lp->a_index[q]]++; col[k] = j; val[k] = lp->a_value[q]; }
      report[34] = cmp_dev_i(P.arr.orow_ptr, ptr.data(), m + 1);
      report[35] = cmp_dev_i(P.arr.orow_col, col.data(), nnz0) + cmp_dev_d(P.arr.orow_val, val.data(), nnz0);
    }
    report[36] = (P.sc.scaled != 0) != f.scaled;
  });
}

// The block-mode prologue of b200pdlp_solve_hipdlp_multi (run_hipdlp_shard_prologue, every rank on the current device)
// against formulate_hipdlp + scale_hipdlp + plan_hipdlp_shards (ordered_max = -1) + build_hipdlp_shard, bit for bit;
// report[8 + 9 world], see include/b200pdlp.h.
int b200pdlp_debug_hipdlp_shard_prep_compare(const b200pdlp_lp* lp, int32_t scaling_mode, int32_t ruiz_iterations, int32_t world,
                                             double* report) {
  DeviceGuard dg;
  return guarded([&] {
    check_lp(lp);
    if (!report || world < 2 || world > kMaxPeers || ruiz_iterations < 0) throw Error(B200PDLP_ERR_ARG, "bad argument");
    for (int k = 0; k < 8 + 9 * world; k++) report[k] = 0.0;
    StdForm f;
    formulate_hipdlp(*lp, f);
    scale_hipdlp(f, scaling_mode, ruiz_iterations);
    HipShards S;
    plan_hipdlp_shards(f, world, /*ordered_max=*/-1, S);
    std::vector<int> ranks(world);
    for (int g = 0; g < world; g++) ranks[g] = g;
    TempPrologue T;
    run_hipdlp_shard_prologue(*lp, scaling_mode, ruiz_iterations, world, ranks, T);
    const DevicePrologue& P = T.P;
    const DevProblemArrays& a = P.arr;
    const int n = f.n, m = f.m;
    report[0] = (a.n != n) + (a.m != m) + (a.nnz != f.nnz) + (a.neq != f.neq);
    if (report[0] > 0) return;
    {
      std::vector<double> t(std::max(n, m));
      auto cmp_perm = [&](const double* dev, const std::vector<double>& v, const std::vector<int>& perm, int len) {
        for (int i = 0; i < len; i++) t[i] = v[perm[i]];
        return cmp_dev_d(dev, t.data(), len);
      };
      report[1] = cmp_perm(a.cost, f.cost, S.cperm, n) + cmp_perm(a.lower, f.lower, S.cperm, n) + cmp_perm(a.upper, f.upper, S.cperm, n) +
                  cmp_perm(a.colscale, f.col_scale, S.cperm, n) + cmp_perm(a.rhs, f.rhs, S.rperm, m) +
                  cmp_perm(a.rowscale, f.row_scale, S.rperm, m);
      report[2] = cmp_perm(a.rup, f.row_upper, S.rperm, m);
    }
    const double nc = std::sqrt(P.sc.norm_cost_sq), nr = std::sqrt(P.sc.norm_rhs_sq);
    report[3] = memcmp(&nc, &f.norm_cost, sizeof(double)) != 0;
    report[4] = memcmp(&nr, &f.norm_rhs, sizeof(double)) != 0;
    report[5] = (P.sc.scaled != 0) != f.scaled;
    report[6] = cmp_dev_i(a.rperm, S.rperm.data(), m) + cmp_dev_i(a.cperm, S.cperm.data(), n);
    for (int g = 0; g < world; g++) {
      double* r = report + 8 + 9 * g;
      r[0] = (P.rb[g] != S.rb[g]) + (P.rb[g + 1] != S.rb[g + 1]) + (P.cb[g] != S.cb[g]) + (P.cb[g + 1] != S.cb[g + 1]);
      SellMatrix A, AT;
      build_hipdlp_shard(S, g, A, AT);
      cmp_sell(P.block_A[g], A, r + 1, r + 2, r + 3, r + 4);
      cmp_sell(P.block_AT[g], AT, r + 5, r + 6, r + 7, r + 8);
    }
  });
}

void b200pdlp_release_cache(void) { dev_cache_release(); }

// page-lock / unlock caller memory (cudaHostRegister): H2D / D2H copies of registered buffers run at PCIe speed and
// truly asynchronously; pageable buffers are staged by the driver at a fraction of that
int b200pdlp_host_register(void* ptr, size_t bytes) {
  return guarded([&] {
    if (!ptr || bytes == 0) throw Error(B200PDLP_ERR_ARG, "null argument");
    CUDA_OK(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
  });
}
int b200pdlp_host_unregister(void* ptr) {
  return guarded([&] {
    if (!ptr) throw Error(B200PDLP_ERR_ARG, "null argument");
    CUDA_OK(cudaHostUnregister(ptr));
  });
}

int b200pdlp_partition_rows(const b200pdlp_lp* lp, int32_t world, int32_t* bounds) {
  return guarded([&] {
    check_lp(lp);
    if (world < 1 || !bounds) throw Error(B200PDLP_ERR_ARG, "bad argument");
    StdForm f;
    formulate(*lp, f);
    std::vector<int> b = partition_rows(f, world);
    for (int g = 0; g <= world; g++) bounds[g] = b[g];
  });
}

}  // extern "C"
