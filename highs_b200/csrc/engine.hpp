// highs_b200/csrc/engine.hpp -- what the host-side engine files share (engine.cu, engine_hipdlp.cu, engine_batch.cu):
// the problem handle, the device buffers, the error and entry-point helpers, and the functions one file calls in another.
#pragma once

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

// the message b200pdlp_last_error() returns: one per thread, shared by every engine file (defined in engine.cu)
extern thread_local std::string g_last_error;

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
inline NcclApi& nccl() {
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
  DevBuf<unsigned> nz;           // zero-skip shape (DevSell::zskip_grid): nonzero bitmap of the input vector
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

constexpr int kSlotK1 = 0, kSlotK2 = 1, kSlotK3 = 2, kSlotChk = 3, kNumSlots = 4;
constexpr int kOutsCount = 64;

inline void set_device(const b200pdlp_problem* p) { CUDA_OK(cudaSetDevice(p->device)); }

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

struct CheckResult { Residuals it[2]; bool timed_out = false; };
struct RestartMemo { double pf_lr = 0, df_lr = 0, gap_lr = 0, pf_lc = 0, df_lc = 0, gap_lc = 0; int last_iter = 0; };

// ---- the entry points' helpers
template <class F>
int guarded(F&& fn) {
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
void run_per_rank(int count, const char* label, F&& fn, const int* ids = nullptr) {
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

inline void check_params(const b200pdlp_params& prm) {
  if (prm.device_scaling != 0 && prm.device_scaling != -1)
    throw Error(B200PDLP_ERR_ARG, "b200pdlp: params.device_scaling must be 0 (default) or -1 (host prologue)");
}

// what check_lp checks without reading an array: the sizes, and the arrays the sizes call for are present
inline bool lp_fields_ok(const b200pdlp_lp* lp) {
  return lp && lp->num_col >= 0 && lp->num_row >= 0 && lp->a_start && (lp->num_col == 0 || (lp->col_cost && lp->col_lower && lp->col_upper)) &&
         (lp->num_row == 0 || (lp->row_lower && lp->row_upper));
}

// deep: also the O(n) / O(nnz) validation of a_start and a_index (the device prologue does both in its first sweep)
inline void check_lp(const b200pdlp_lp* lp, bool deep = true) {
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

// fn(i) for i < count on up to one host thread per core; after all have run, the failure of the lowest index is rethrown
// with "member i: " before its message
template <class F>
void for_members(int count, F&& fn) {
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

// ---- defined in one engine file, called in another
// engine.cu: problem construction
int device_count_checked();
void open_problem(b200pdlp_problem* p, int device, int rank, int world);
void run_prologue(DevicePrologue& P, cudaStream_t s, const b200pdlp_lp& lp, bool do_scale);
void take_layout(b200pdlp_problem* p, HostLayout&& L);
void set_full_length_dims(b200pdlp_problem* p);
void take_prologue(const b200pdlp_lp& lp, DevicePrologue& P, b200pdlp_problem* p);
void upload_permuted(DevBuf<double>& d, const std::vector<double>& v, const int* perm, int offset, int len, int size,
                     double pad = 0.0);
void alloc_scratch(b200pdlp_problem* p, bool zero);
void alloc_peer_words(b200pdlp_problem* p);
void alloc_postsolve_staging(b200pdlp_problem* p);
int std_form_cols(const b200pdlp_lp& lp, double inf);
bool device_prep_fits(const b200pdlp_lp& lp, int ordered_max, double inf);
void adopt_matrix(DeviceMatrix& M, DevSellOwned& O);
void apply_spmv_grid(b200pdlp_problem* p);
void ensure_host_maps(b200pdlp_problem* p);

// engine.cu: the PDLP solve's host control, which the batch rounds share
void fill_pow_tables(PdhgState* h);
void arm_step(PdhgState* h);
void assemble_check_a(const StdForm& f, const double* o, CheckResult& cr, double dscale[2], double pscale[2]);
void assemble_check_b(const StdForm& f, const double* o, CheckResult& cr, const double dscale[2], const double pscale[2]);
int check_decision(const b200pdlp_params& prm, double tol_p, double tol_d, const PdhgState* h, const CheckResult& chk,
                   RestartMemo& memo, int* term_iterate, int* choice);
void restart_steps(PdhgState* h, int choice, const CheckResult& c, RestartMemo& mm, double dx2, double dy2);
int next_check_iter(int iter, int interval, int iter_limit);
void host_start_point(const StdForm& f, const b200pdlp_warm* warm, std::vector<double>& x0, std::vector<double>& y0);
double proj_zero(const StdForm& f, int j);
void host_postsolve(const StdForm& f, bool have_check, std::vector<double>& hx, std::vector<double>& hy,
                    std::vector<double>& hax, const std::vector<double>& haty, b200pdlp_result* out);
void fill_result(b200pdlp_result* out, const StdForm& f, const PdhgState* h, int term, int term_iterate, int restarts,
                 const CheckResult& chk);
void trace_row(b200pdlp_result* out, const PdhgState* h, const CheckResult& c, int restart);

// engine.cu: the kernel-level and test entry points' helpers
void require_mode(const b200pdlp_problem* p, bool hipdlp, const char* who);
void upload_perm(b200pdlp_problem* p, double* d, const double* v, const std::vector<int>& perm);
void download_perm(b200pdlp_problem* p, double* v, const double* d, const std::vector<int>& perm);
void cmp_sell(const DevSellOwned& D, const SellMatrix& H, double* r_slices, double* r_col, double* r_val, double* r_long);
bool prep_compare_arrays(const DevicePrologue& P, const StdForm& f, const HostLayout& L, double* report);

// elements of the device array dev[0..count) whose bytes differ from host[0..count)
template <class T>
double dev_mismatches(const T* dev, const T* host, size_t count) {
  std::vector<T> t(count);
  if (count) CUDA_OK(cudaMemcpy(t.data(), dev, count * sizeof(T), cudaMemcpyDeviceToHost));
  double bad = 0;
  for (size_t i = 0; i < count; i++) bad += memcmp(&t[i], host + i, sizeof(T)) != 0;
  return bad;
}

// engine_hipdlp.cu
void hip_host_postsolve(const b200pdlp_lp& lp, const StdForm& f, const int* cperm, const int* rperm, const double* x,
                        const double* y, const double* sp, const double* sn, b200pdlp_result* out);
void hip_trace_row(b200pdlp_result* out, const HipController& ctl, const double* sums, bool restart, bool converged);

}  // namespace b200
