// highs_b200/csrc/engine.cu -- host side of the B200 PDLP engine: problem construction, the PDLP solve, the multi-GPU
// plumbing and the C ABI (include/b200pdlp.h) of everything but the HiPDLP mode (engine_hipdlp.cu) and the batches
// (engine_batch.cu).
//
// The host owns what cuPDLP-C's PDHG_Solve owns (/root/reference/highs/pdlp/cupdlp/
// cupdlp_solver.c:899-1106): the outer loop, the check schedule (first 10
// iterations, then every 40), termination, infeasibility detection and the
// restart decisions (cupdlp_restart.c:3-99, cupdlp_proj.c:88-148).  Everything that
// touches an n- or m-vector runs in pdhg_kernels.cu.  Between two checks the host
// does not synchronise: it points state.stop_iter at the next check iteration and
// replays a CUDA graph of PDHG passes; the adaptive step rule runs on the device.
#include "engine.hpp"

namespace b200 {

thread_local std::string g_last_error;

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

// experiment (B200PDLP_SPMV_CTAS_PER_SM=k, one GPU, tree mode): the SpMV bodies run on a persistent grid of k CTAs per SM and
// walk their slices in a software pipeline (spmv_sell_kernel<Epi, true>) instead of one CTA per 8 slices
void apply_spmv_grid(b200pdlp_problem* p) {
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
  // Zero-skip shape of the PDLP pass SpMVs (spmv_sell_zskip_kernel: the nonzero bitmap of the input staged in shared memory,
  // only the entries that may be nonzero gathered; same sums as the shape chosen above) wherever the matrix is not tiled and
  // the bitmap of its input fits in a CTA's shared memory.  Measured on one H100 (DESIGN.md section 6).
  // B200PDLP_ZERO_SKIP=0 turns it off to compare the two shapes; it changes no result.
  if (!p->form.hipdlp && val("B200PDLP_ZERO_SKIP", 1) != 0) {
    auto zskip = [&](DeviceMatrix& M, int len) {
      if (M.dev.tiled || M.dev.nslices == 0) return;
      const int bytes = (int)(((size_t)len + 127) / 128 * 16);
      const int per_sm = zskip_ctas_per_sm(bytes);
      if (per_sm <= 0) return;
      M.nz.alloc((size_t)bytes / 4, false);
      M.dev.nzmap = M.nz.p; M.dev.nz_bytes = bytes; M.dev.zskip_grid = per_sm * sms;
    };
    zskip(p->A, p->n);
    zskip(p->AT, p->m);
  }
  if (getenv("B200PDLP_TIMING")) {
    fprintf(stderr, "[b200pdlp setup] SpMV shapes: A %s (%d CTAs, tiles staged %d/%d)  A' %s (%d CTAs, tiles staged %d/%d)\n",
            p->A.dev.tiled ? "tiled" : (p->A.dev.pipelined ? "persistent" : "one slice per warp"), p->A.dev.nblocks_body,
            p->A.tiles_staged, p->A.ntiles,
            p->AT.dev.tiled ? "tiled" : (p->AT.dev.pipelined ? "persistent" : "one slice per warp"), p->AT.dev.nblocks_body,
            p->AT.tiles_staged, p->AT.ntiles);
    fprintf(stderr, "[b200pdlp setup] zero-skip pass SpMVs: A %d CTAs  A' %d CTAs (0: off)\n", p->A.dev.zskip_grid,
            p->AT.dev.zskip_grid);
  }
}

// ---- problem construction.  Every creator below is a sequence of these steps plus what is its own.

// the number of CUDA devices; none is an error: the engine has no CPU fallback
int device_count_checked() {
  int ndev = 0;
  const cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    throw Error(B200PDLP_ERR_CUDA, std::string("no CUDA device: the engine has no CPU fallback (") + cudaGetErrorString(e) + ")");
  return ndev;
}

// rank `rank` of `world` on `device` (< 0: the caller's current device): selects the device and creates the problem's stream
void open_problem(b200pdlp_problem* p, int device, int rank, int world) {
  device_count_checked();
  if (device >= 0) p->device = device; else CUDA_OK(cudaGetDevice(&p->device));
  set_device(p);
  p->rank = rank; p->world = world;
  CUDA_OK(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
}

// the only caller of DevicePrologue::run: bad input -> ERR_ARG, CUDA errors -> ERR_CUDA; a host std::bad_alloc passes
// through (guarded: ERR_ALLOC)
void run_prologue(DevicePrologue& P, cudaStream_t s, const b200pdlp_lp& lp, bool do_scale) {
  try {
    P.run(s, lp, do_scale, /*long_threshold=*/512);
  } catch (const std::invalid_argument& ex) {
    throw Error(B200PDLP_ERR_ARG, ex.what());
  } catch (const std::runtime_error& ex) {
    throw Error(B200PDLP_ERR_CUDA, ex.what());
  }
}

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
void take_layout(b200pdlp_problem* p, HostLayout&& L) {
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
void set_full_length_dims(b200pdlp_problem* p) {
  const StdForm& f = p->form;
  const int n = f.n, m = f.m;
  p->n = n; p->m = m; p->ml = m; p->r0 = 0; p->r1 = m; p->neq_local = f.neq;
  p->row_bounds = {0, m};
  p->nl = p->nl_real = n; p->c0 = 0; p->shard_len = n; p->seg_len = n;
  p->csr_local.nrows = m; p->csr_local.ncols = n; p->csr_local.nnz = f.nnz;   // dimensions only (built on demand)
}

// what a problem that holds every row takes from a device prologue: the form's scalars, the dimensions and the device-order
// vectors, adopted on one GPU; in block mode every rank takes its own copy (the matrices are the caller's: A / A' or a block)
void take_prologue(const b200pdlp_lp& lp, DevicePrologue& P, b200pdlp_problem* p) {
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
void upload_permuted(DevBuf<double>& d, const std::vector<double>& v, const int* perm, int offset, int len, int size,
                     double pad) {
  std::vector<double> t((size_t)std::max(size, 1), pad);
  for (int i = 0; i < len; i++) t[i] = v[offset + perm[i]];
  d.alloc(size, false);
  d.upload(t.data(), size);
}

// reduction scratch (sized for the larger launch shape, so after apply_spmv_grid), the check's device scalars and their pinned
// mirror.  The term scratch has p->ordered_cap entries per accumulator: set by pdlp in ordered mode, 0 for HiPDLP, whose check
// reduces without it.  zero: every buffer zeroed at allocation; the counters are zero before the first launch either way.
void alloc_scratch(b200pdlp_problem* p, bool zero) {
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
void alloc_peer_words(b200pdlp_problem* p) {
  p->flags.alloc(kMaxPeers);
  p->epochs.alloc(1);
  p->fault.alloc(1);
}

// staging of the hot start and of the solution in original order (device postsolve)
void alloc_postsolve_staging(b200pdlp_problem* p) {
  p->io_col.alloc((size_t)2 * std::max(p->form.n_orig, 1), false);
  p->io_row.alloc((size_t)2 * std::max(p->m, 1), false);
}

// The size rule of both device prologues.  Ordered mode keeps the host prologue; it is decided on the STANDARD FORM's size,
// n = num_col + one slack column per ranged or free row (CupdlpWrapper.cpp:328-345; `inf` is the mode's infinite row bound),
// so count them when the answer depends on it.  An empty matrix keeps it too.
int std_form_cols(const b200pdlp_lp& lp, double inf) {
  int nslack = 0;
  for (int i = 0; i < lp.num_row; i++) {
    const bool lo = lp.row_lower[i] > -inf, up = lp.row_upper[i] < inf;
    nslack += (lo && up && lp.row_lower[i] != lp.row_upper[i]) || (!lo && !up);
  }
  return lp.num_col + nslack;
}
bool device_prep_fits(const b200pdlp_lp& lp, int ordered_max, double inf) {
  const int omax = ordered_max == 0 ? 4096 : ordered_max;
  if (omax > 0 && lp.num_col <= omax && lp.num_row <= omax && std_form_cols(lp, inf) <= omax) return false;
  return lp.num_col > 0 && lp.num_row > 0 && lp.a_start[lp.num_col] > 0;
}

// ---- LPs whose arrays are device memory (the device-array batches and single solves)
// check_lp's message for a BatchPrepErr of a sizing kernel
const char* prep_error_text(int err) {
  switch (err) {
    case kPrepStart0: return "b200pdlp: a_start[0] must be 0 and a_start[num_col] >= 0";
    case kPrepDecreasing: return "b200pdlp: a_start must be non-decreasing";
    case kPrepIndex: return "b200pdlp: a_index entry outside [0, num_row)";
    default: return "b200pdlp: malformed b200pdlp_lp";
  }
}

// ptr (NULL: not given) must be device or managed memory of `device`; i >= 0: the array belongs to member i of a batch
void check_device_array(const void* ptr, int device, int i, const char* field, const char* who) {
  if (!ptr) return;
  cudaPointerAttributes a{};
  const cudaError_t e = cudaPointerGetAttributes(&a, ptr);
  if (e != cudaSuccess) cudaGetLastError();
  if (e != cudaSuccess || !((a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device))
    throw Error(B200PDLP_ERR_ARG, std::string(who) + (i >= 0 ? ": member " + std::to_string(i) : std::string()) + ": " +
                                      field + " is not device memory of device " + std::to_string(device));
}

// the arrays of an LP, in this order
void check_device_lp(const b200pdlp_lp& lp, int device, int i, const char* who) {
  check_device_array(lp.a_start, device, i, "a_start", who);
  check_device_array(lp.a_index, device, i, "a_index", who);
  check_device_array(lp.a_value, device, i, "a_value", who);
  check_device_array(lp.col_cost, device, i, "col_cost", who);
  check_device_array(lp.col_lower, device, i, "col_lower", who);
  check_device_array(lp.col_upper, device, i, "col_upper", who);
  check_device_array(lp.row_lower, device, i, "row_lower", who);
  check_device_array(lp.row_upper, device, i, "row_upper", who);
}

// the four vectors of a result, in this order
void check_device_result(const b200pdlp_result& out, int device, int i, const char* who) {
  check_device_array(out.col_value, device, i, "result col_value", who);
  check_device_array(out.col_dual, device, i, "result col_dual", who);
  check_device_array(out.row_value, device, i, "result row_value", who);
  check_device_array(out.row_dual, device, i, "result row_dual", who);
}

// The route of a single solve on device arrays, from the grid-wide sizing kernel's two passes on stream s (batch_prep.cu
// lp_size_kernel: check_lp(deep) and the slack rows under the mode's classification) and one read-back of its record: Ordered when the
// standard form is within ordered_max (device_prep_fits' rule), else Tree when it has rows, columns and nonzeros, else
// Degenerate.  A malformed LP is ERR_ARG with check_lp's message, in check_lp's order.  *nnz = a_start[num_col].
enum class DeviceRoute { Ordered, Tree, Degenerate };
static DeviceRoute device_lp_route(cudaStream_t s, const b200pdlp_lp& lp, bool hipdlp, int ordered_max, const char* who, int* nnz) {
  BatchPrep P{};
  P.n0 = lp.num_col; P.m = lp.num_row; P.sense = lp.sense;
  P.a_start = lp.a_start; P.a_index = lp.a_index; P.a_value = lp.a_value;
  P.col_cost = lp.col_cost; P.col_lower = lp.col_lower; P.col_upper = lp.col_upper;
  P.row_lower = lp.row_lower; P.row_upper = lp.row_upper;
  DevBuf<LpSize> d;
  d.alloc(1, false);
  PinnedArray<LpSize> z(1);
  CUDA_OK(cudaMemsetAsync(d.p, 0, sizeof(LpSize), s));
  launch_lp_size(s, P, hipdlp, d.p);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(z.p, d.p, sizeof(LpSize), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  for (int e : {kPrepNull, kPrepStart0, kPrepDecreasing, kPrepIndex})
    if (z.p->err_bits & (1u << e)) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": " + prep_error_text(e));
  *nnz = z.p->nnz;
  const int omax = ordered_max == 0 ? 4096 : ordered_max;
  if (omax > 0 && std::max<long long>((long long)lp.num_col + z.p->nslack, lp.num_row) <= omax) return DeviceRoute::Ordered;
  return lp.num_col > 0 && lp.num_row > 0 && z.p->nnz > 0 ? DeviceRoute::Tree : DeviceRoute::Degenerate;
}

// A degenerate LP of a single device-array solve (no rows, no columns or no nonzeros: well-formed, it has no matrix) takes
// the host prologue, as in the host-array solve: its vectors (and hot start) come down, solve() runs on host copies, and the
// four result vectors go back up into the caller's device vectors (those given) on stream s.
static void solve_degenerate(cudaStream_t s, const b200pdlp_lp& lp, const b200pdlp_warm* warm, b200pdlp_result* out,
                             const std::function<void(const b200pdlp_lp&, const b200pdlp_warm*, b200pdlp_result*)>& solve) {
  const int n0 = lp.num_col, m = lp.num_row;
  std::vector<int> start((size_t)n0 + 1);
  std::vector<std::vector<double>> h(12);
  auto down = [&](int k, const double* d, int len) {
    h[k].assign((size_t)std::max(len, 1), 0.0);
    if (d && len > 0) CUDA_OK(cudaMemcpyAsync(h[k].data(), d, (size_t)len * sizeof(double), cudaMemcpyDeviceToHost, s));
    return h[k].data();
  };
  CUDA_OK(cudaMemcpyAsync(start.data(), lp.a_start, start.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
  b200pdlp_lp hl = lp;
  hl.a_start = start.data(); hl.a_index = nullptr; hl.a_value = nullptr;
  hl.col_cost = down(0, lp.col_cost, n0); hl.col_lower = down(1, lp.col_lower, n0); hl.col_upper = down(2, lp.col_upper, n0);
  hl.row_lower = down(3, lp.row_lower, m); hl.row_upper = down(4, lp.row_upper, m);
  b200pdlp_warm hw{};
  const bool hot = warm && warm->col_value && warm->row_value && warm->row_dual;
  if (hot) { hw.col_value = down(5, warm->col_value, n0); hw.row_value = down(6, warm->row_value, m); hw.row_dual = down(7, warm->row_dual, m); }
  CUDA_OK(cudaStreamSynchronize(s));
  b200pdlp_result r = *out;
  r.col_value = down(8, nullptr, n0); r.col_dual = down(9, nullptr, n0); r.row_value = down(10, nullptr, m); r.row_dual = down(11, nullptr, m);
  solve(hl, hot ? &hw : nullptr, &r);
  auto up = [&](double* d, const double* v, int len) {
    if (d && len > 0) CUDA_OK(cudaMemcpyAsync(d, v, (size_t)len * sizeof(double), cudaMemcpyHostToDevice, s));
  };
  up(out->col_value, r.col_value, n0); up(out->col_dual, r.col_dual, n0); up(out->row_value, r.row_value, m); up(out->row_dual, r.row_dual, m);
  CUDA_OK(cudaStreamSynchronize(s));
  r.col_value = out->col_value; r.col_dual = out->col_dual; r.row_value = out->row_value; r.row_dual = out->row_dual;
  *out = r;
}

void solve_lp_device(const b200pdlp_lp& lp, bool hipdlp, int& device, int ordered_max, const b200pdlp_warm* warm,
                     b200pdlp_result* out, const char* who, const std::function<void()>& batch, const CreateProblem& create_host,
                     const CreateProblem& create_device, const SolveProblem& solve) {
  if (!lp_fields_ok(&lp)) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": b200pdlp: malformed b200pdlp_lp");
  if (lp.sense != 1.0 && lp.sense != -1.0) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": b200pdlp: sense must be +1 or -1");
  device = select_device(device);
  check_device_lp(lp, device, -1, who);
  if (warm) {
    check_device_array(warm->col_value, device, -1, "warm col_value", who);
    check_device_array(warm->row_value, device, -1, "warm row_value", who);
    check_device_array(warm->row_dual, device, -1, "warm row_dual", who);
  }
  check_device_result(*out, device, -1, who);
  const auto t0 = std::chrono::steady_clock::now();
  ProblemPtr p(new b200pdlp_problem());   // its stream serves the sizing and, in tree mode, the solve
  open_problem(p.get(), device, 0, 1);
  int nnz = 0;
  const DeviceRoute route = device_lp_route(p->stream, lp, hipdlp, ordered_max, who, &nnz);
  auto setup_seconds = [&] { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); };
  if (route == DeviceRoute::Ordered) {
    batch();
  } else if (route == DeviceRoute::Degenerate) {
    solve_degenerate(p->stream, lp, warm, out, [&](const b200pdlp_lp& hl, const b200pdlp_warm* hw, b200pdlp_result* r) {
      ProblemPtr q(new b200pdlp_problem());
      create_host(hl, q.get());
      r->setup_seconds = setup_seconds();
      solve(q.get(), hl, hw, r);
    });
  } else {
    p->device_io = true;
    p->prep.inputs_on_device = true;
    p->prep.device_nnz = nnz;
    create_device(lp, p.get());
    out->setup_seconds = setup_seconds();
    solve(p.get(), lp, warm, out);
  }
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
void adopt_matrix(DeviceMatrix& M, DevSellOwned& O) {
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

// p: opened on its device (open_problem)
static void create_problem_device(const b200pdlp_lp& lp, const b200pdlp_params& prm, b200pdlp_problem* p) {
  NvtxRange nvtx("b200pdlp: prologue (device)");
  Laps lap;
  ensure_side_stream(p);
  p->dev_form = true;
  if (getenv("B200PDLP_KEEP_FORM")) p->prep.keep_form = true;
  DevicePrologue& P = p->prep;
  run_prologue(P, p->stream, lp, prm.scaling != 0);
  lap("setup", "device prologue");
  if (lap.on) {
    fprintf(stderr, "[b200pdlp setup] sectors per gathered lane (sampled): A %.3f  A' %.3f\n",
            P.sc.a_lanes ? (double)P.sc.a_sectors / P.sc.a_lanes : 0.0, P.sc.at_lanes ? (double)P.sc.at_sectors / P.sc.at_lanes : 0.0);
    fprintf(stderr, "[b200pdlp setup] LP arrays copied to the device: %zu bytes\n", P.h2d_bytes);
  }
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
  if (!p->device_io) alloc_postsolve_staging(p);
  alloc_scratch(p, false);
  p->state.alloc(1, false);
  p->redbuf.alloc(16, false);
  alloc_host_mirrors(p);
  lap("setup", "vectors + scratch");
}

// host copies of what the device prologue keeps in HBM, fetched when a test accessor needs them
void ensure_host_maps(b200pdlp_problem* p) {
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
                     p->upper.p, p->xsum.p, r1, p->A.dev.nzmap);
  launch_spmv_dual(s, p->A.dev, st, p->x[0].p, p->x[1].p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p,
                   p->rhs.p, p->ysum.p, p->neq_local, 0, r2, p->axsum.p, p->AT.dev.nzmap);
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
  return capture_graph(p->stream, [&] { for (int i = 0; i < passes; i++) enqueue_pass(p); });
}

void fill_pow_tables(PdhgState* h) {
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
static const char kPeerLate[] = "P2P barrier timed out (a peer rank did not arrive)";
// P2P: reads the barriers' fault word behind the work on the stream (and synchronises the stream).  A barrier that gave up
// waiting for a peer leaves inconsistent data behind: stop with `msg` instead of going on with it.
static void throw_if_peer_fault(b200pdlp_problem* p, const char* msg) {
  if (!p->p2p) return;
  int* hfault = reinterpret_cast<int*>(p->hflag + 2);
  CUDA_OK(cudaMemcpyAsync(hfault, p->fault.p, sizeof(int), cudaMemcpyDeviceToHost, p->stream));
  CUDA_OK(cudaStreamSynchronize(p->stream));
  if (*hfault) throw Error(B200PDLP_ERR_STATE, msg);
}
static void pull_state(b200pdlp_problem* p) {
  CUDA_OK(cudaMemcpyAsync(p->hstate, p->state.p, sizeof(PdhgState), cudaMemcpyDeviceToHost, p->stream));
  if (p->p2p) throw_if_peer_fault(p, kPeerLate);
  else CUDA_OK(cudaStreamSynchronize(p->stream));
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
void assemble_check_a(const StdForm& f, const double* o, CheckResult& cr, double dscale[2], double pscale[2]) {
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
void assemble_check_b(const StdForm& f, const double* o, CheckResult& cr, const double dscale[2], const double pscale[2]) {
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
void restart_steps(PdhgState* h, int choice, const CheckResult& c, RestartMemo& mm, double dx2, double dy2) {
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
void arm_step(PdhgState* h) {
  h->eta = std::sqrt(h->tau * h->sigma);
  if (h->adaptive) {
    h->tau_try = h->eta / std::sqrt(h->beta);
    h->sigma_try = h->eta * std::sqrt(h->beta);
  } else {
    h->tau_try = h->tau;
    h->sigma_try = h->sigma;
  }
}

double time_limit_or_none(double time_limit) { return (time_limit >= 0 && std::isfinite(time_limit)) ? time_limit : -1.0; }

double step_beta(double cost_sq, double rhs_sq) { return std::fmin(cost_sq, rhs_sq) > 1e-6 ? cost_sq / rhs_sq : 1.0; }
void adaptive_step_sizes(PdhgState* h, double amax) {
  h->tau = (1.0 / amax) / std::sqrt(h->beta);
  h->sigma = h->tau * h->beta;
}
void fixed_step_sizes(PdhgState* h, double lambda) {
  h->tau = 0.8 / std::sqrt(lambda);
  h->sigma = h->tau;
  h->tau /= std::sqrt(h->beta);
  h->sigma *= std::sqrt(h->beta);
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
int check_decision(const b200pdlp_params& prm, double tol_p, double tol_d, const PdhgState* h, const CheckResult& chk,
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
int next_check_iter(int iter, int interval, int iter_limit) {
  int next = iter + 1;
  while (!(next < 10 || next % interval == 0 || next == iter_limit - 1)) next++;
  return next;
}

// PDHG_PreSolve's hot start (cupdlp_solver.c:1217-1279) + PDHG_Project_Bounds in standard-form order: x0[n], y0[m] (zero
// without a complete hot start)
void host_start_point(const StdForm& f, const b200pdlp_warm* warm, std::vector<double>& x0, std::vector<double>& y0) {
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
double proj_zero(const StdForm& f, int j) {
  double v = 0.0;
  v = v < f.upper[j] ? v : f.upper[j];
  v = v > f.lower[j] ? v : f.lower[j];
  return v;
}

// PDHG_PostSolve (cupdlp_solver.c:1281-1435) on the host: x, y, A x, A'y of the returned iterate in standard-form order ->
// the four HighsSolution vectors in `out` (scaled in place)
void host_postsolve(const StdForm& f, bool have_check, std::vector<double>& hx, std::vector<double>& hy,
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
void fill_result(b200pdlp_result* out, const StdForm& f, const PdhgState* h, int term, int term_iterate, int restarts,
                        const CheckResult& chk) {
  out->value_valid = 1; out->dual_valid = 1;
  out->term_code = term; out->term_iterate = term_iterate;
  out->iters = h->iter; out->passes = h->passes; out->restarts = restarts;
  const Residuals& R = chk.it[(term == B200PDLP_OPTIMAL && term_iterate == 1) ? 1 : 0];
  out->primal_obj = R.pobj; out->dual_obj = R.dobj; out->primal_feas = R.pfeas; out->dual_feas = R.dfeas;
  out->gap = R.gap; out->rel_gap = R.relgap;
  out->form_cols = f.n; out->form_rows = f.m; out->form_nnz = f.nnz; out->form_neq = f.neq;
}

void trace_row(b200pdlp_result* out, const PdhgState* h, const CheckResult& c, int restart) {
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
  return capture_graph(p->stream, [&] { *launches = enqueue_check_device(p, light); });
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
  const int kp = p->kernels_per_pass();
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

// ---- the phases of the single solve, in the order solve_on_device runs them
// the check control block: pinned host copy, mapped time-limit word, device copy (filled by a copy on p->stream)
static void ensure_ctl(b200pdlp_problem* p) {
  if (p->hctl) return;
  p->hctl = static_cast<SolveCtl*>(pinned_cache_alloc(sizeof(SolveCtl), false));
  p->htime = static_cast<int*>(pinned_cache_alloc(64, true));
  p->ctl.alloc(1, false);
}
static int* mapped_time_flag(b200pdlp_problem* p) {
  int* d = nullptr;
  CUDA_OK(cudaHostGetDevicePointer(&d, p->htime, 0));
  return d;
}
// the control block zeroed, with the fields every check reads (the caller adds the time flag, the trace and the memo)
static SolveCtl* reset_ctl(b200pdlp_problem* p, double tol_p, double tol_d, double tol_gap, int iter_limit, int interval,
                           bool restart_on) {
  ensure_ctl(p);
  SolveCtl* c = p->hctl;
  memset(c, 0, sizeof(SolveCtl));
  c->tol_p = tol_p; c->tol_d = tol_d; c->tol_gap = tol_gap;
  c->sense = p->form.sense; c->offset = p->form.offset;
  c->iter_limit = iter_limit; c->interval = interval; c->restart_on = restart_on; c->world = p->world;
  c->term = -1;
  return c;
}

// Graphs: one check interval of passes, and a short one for top-ups after rejected steps.  A few spare passes per replay:
// a rejected line-search step then still reaches the next check iteration inside the same replay (spare passes are no-ops
// once state.iter == state.stop_iter) instead of costing a host round trip.  The device-driven loop captures its graphs
// when it first needs them, unless `eager` (logical shards): everything that allocates or instantiates happens before ANY
// rank launches a kernel that waits for its peers (see LocalGroup), so every graph is captured and uploaded here.
static void prepare_graphs(b200pdlp_problem* p, const b200pdlp_params& prm, int interval, bool dev_checks, bool eager) {
  cudaStream_t s = p->stream;
  const int want = std::min(prm.graph_passes > 0 ? prm.graph_passes : interval + 4, kPowTab - 16);   // the step-rule tables cover one replay
  if (p->graph_main && p->graph_main_passes != want) { cudaGraphExecDestroy(p->graph_main); p->graph_main = nullptr; }
  p->graph_main_passes = want;
  p->no_graph = getenv("B200PDLP_NO_GRAPH") != nullptr;
  if (p->no_graph || (dev_checks && !eager)) return;
  if (!p->graph_main) p->graph_main = capture_passes(p, want);
  if (!p->graph_small) { p->graph_small_passes = 4; p->graph_small = capture_passes(p, 4); }
  if (!eager) return;
  for (cudaGraphExec_t g : {p->graph_main, p->graph_small}) CUDA_OK(cudaGraphUpload(g, s));
  if (!dev_checks) return;
  ensure_ctl(p);
  for (int k = 2; k <= 5; k++) if (!p->graph_pow2[k]) { p->graph_pow2[k] = capture_passes(p, 1 << k); CUDA_OK(cudaGraphUpload(p->graph_pow2[k], s)); }
  if (!p->graph_check) { p->graph_check = capture_check(p, false, &p->check_launches[0]); CUDA_OK(cudaGraphUpload(p->graph_check, s)); }
  if (!p->graph_check_light) { p->graph_check_light = capture_check(p, true, &p->check_launches[1]); CUDA_OK(cudaGraphUpload(p->graph_check_light, s)); }
}

// initial point: PDHG_PreSolve (hot start, cupdlp_solver.c:1217-1279) + PDHG_Init_Variables (:531-591) before the steps
static void start_point(b200pdlp_problem* p, const b200pdlp_warm* warm) {
  const StdForm& f = p->form;
  cudaStream_t s = p->stream;
  const int m = p->m, ml = p->ml, nl = p->nl;   // nl: column entries held by this rank (== n on one GPU)
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
  if (p->dev_form) {
    // maps and scales live in HBM: the hot start goes up in original order and is permuted / scaled / projected there
    const double *wc = nullptr, *wv = nullptr, *wd = nullptr;
    if (warm && warm->col_value && warm->row_value && warm->row_dual && p->device_io) {
      wc = warm->col_value; wv = warm->row_value; wd = warm->row_dual;
    } else if (warm && warm->col_value && warm->row_value && warm->row_dual) {
      CUDA_OK(cudaMemcpyAsync(p->io_col.p, warm->col_value, (size_t)f.n_orig * sizeof(double), cudaMemcpyHostToDevice, s));
      CUDA_OK(cudaMemcpyAsync(p->io_row.p, warm->row_value, (size_t)m * sizeof(double), cudaMemcpyHostToDevice, s));
      CUDA_OK(cudaMemcpyAsync(p->io_row.p + m, warm->row_dual, (size_t)m * sizeof(double), cudaMemcpyHostToDevice, s));
      wc = p->io_col.p; wv = p->io_row.p; wd = p->io_row.p + m;
    }
    launch_init_point(s, p->prep.arr, f.sense, wc, wv, wd, p->colscale.p, p->lower.p, p->upper.p, p->rowscale.p, p->x[0].p,
                      p->xsum.p, p->y[0].p);
    p->launches += 2;
  } else {
    std::vector<double> x0, y0;
    host_start_point(f, warm, x0, y0);
    std::vector<double> xp(std::max(nl, 1), 0.0), yp(std::max(ml, 1));
    for (int i = 0; i < p->nl_real; i++) xp[i] = x0[p->cperm[p->c0 + i]];
    for (int i = 0; i < ml; i++) yp[i] = y0[p->r0 + p->rperm[i]];
    CUDA_OK(cudaMemcpyAsync(p->x[0].p, xp.data(), (size_t)nl * sizeof(double), cudaMemcpyHostToDevice, s));
    if (ml) CUDA_OK(cudaMemcpyAsync(p->y[0].p, yp.data(), (size_t)ml * sizeof(double), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));
  }
}

// PDHG_Init_Step_Sizes (cupdlp_step.c:312-375)
static void init_step_sizes(b200pdlp_problem* p, PdhgState* h) {
  const StdForm& f = p->form;
  double a = 0.0, b = 0.0;   // cupdlp_twoNormSquared = dot(x,x), sequential on the reference's CPU path
  if (p->dev_form) { a = p->beta_cost_sq; b = p->beta_rhs_sq; }   // tree sums from the device prologue
  else {
    for (int j = 0; j < f.n; j++) a += f.cost[j] * f.cost[j];
    for (int i = 0; i < f.m; i++) b += f.rhs[i] * f.rhs[i];
  }
  h->beta = step_beta(a, b);
  if (h->adaptive) adaptive_step_sizes(h, f.amax);
  else fixed_step_sizes(h, power_method(p));
}

// sums start at proj(0) like PDHG_Init_Variables :577-583; the average is recomputed at every check
static void start_products_and_sums(b200pdlp_problem* p) {
  const StdForm& f = p->form;
  cudaStream_t s = p->stream;
  const int nl = p->nl, ml = p->ml;
  full_ax(p, p->x[0].p, p->ax[0].p);
  full_aty(p, p->y[0].p, p->aty[0].p);
  if (!p->dev_form) {
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
}

struct LoopLimits {   // the time limit counts from t_loop
  int interval;
  double tol_p, tol_d, t_lim;   // t_lim < 0: none
  std::chrono::steady_clock::time_point t_loop;
  double elapsed() const { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t_loop).count(); }
  bool over() const { return t_lim >= 0 && elapsed() > t_lim; }
};
struct LoopOutcome {
  int term = B200PDLP_TIMELIMIT_OR_ITERLIMIT, term_iterate = 0, restarts = 0;
  bool have_check = false;
  CheckResult chk;
  double iter_ms = 0.0;   // device time of the passes
};

// device-driven loop: the checks decide on the device (termination, restarts, next check iteration); the host
// enqueues [check, passes to the next check] rounds ahead from the deterministic check schedule and reads the control
// block once per batch.  A rejected line-search step makes a round fall short; the following rounds make up for it
// (kernels are no-ops outside their turn) and the next read-back re-synchronises the prediction.
static LoopOutcome device_loop(b200pdlp_problem* p, const b200pdlp_params& prm, const b200pdlp_warm* warm,
                               const LoopLimits& lim, b200pdlp_result* out) {
  cudaStream_t s = p->stream;
  PdhgState* h = p->hstate;
  const int nl = p->nl, ml = p->ml;
  SolveCtl* c = reset_ctl(p, lim.tol_p, lim.tol_d, prm.tol_gap, prm.iter_limit, lim.interval, prm.restart != 0);
  *p->htime = lim.over() ? 1 : 0;
  c->time_flag = lim.t_lim >= 0 ? mapped_time_flag(p) : nullptr;   // (no limit: spare the device the read over PCIe)
  // dense-check phase (iterations 0 .. kDenseChecks-1 are all check iterations): the passes carry A xSum and A'ySum, the
  // checks are two vector sweeps.  B200PDLP_LIGHT_CHECK=0: every check multiplies the average iterate by A and A'.
  const bool hot = warm && warm->col_value && warm->row_value && warm->row_dual;
  bool h_light = p->axsum.p && p->atysum.p && (p->world == 1 || !hot);   // (several GPUs: A_g xSum of a hot start would need the gathered xSum)
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
  LoopOutcome o;
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
      if (pred_iter >= prm.iter_limit - 1) break;
      const int next = next_check_iter(pred_iter, lim.interval, prm.iter_limit);
      CUDA_OK(cudaEventRecord(ev(), s));
      enqueue_passes_device(p, next - pred_iter);
      CUDA_OK(cudaEventRecord(ev(), s));
      passes += next - pred_iter;
      pred_iter = next;
    }
    CUDA_OK(cudaMemcpyAsync(c, p->ctl.p, sizeof(SolveCtl), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaMemcpyAsync(h, p->state.p, sizeof(PdhgState), cudaMemcpyDeviceToHost, s));
    const size_t npairs = nev / 2;   // events so far come in (before, after) pairs around the passes
    cudaEvent_t fin = ev();
    CUDA_OK(cudaEventRecord(fin, s));
    if (lim.t_lim >= 0) {
      // poll, so that the time-limit word can be raised while the batch runs
      while (cudaEventQuery(fin) == cudaErrorNotReady) {
        if (lim.elapsed() > lim.t_lim) *p->htime = 1;
        std::this_thread::yield();
      }
    }
    CUDA_OK(cudaEventSynchronize(fin));
    throw_if_peer_fault(p, kPeerLate);
    for (size_t k = 0; k < npairs; k++) {
      float ms = 0.f;
      CUDA_OK(cudaEventElapsedTime(&ms, *evs[2 * k], *evs[2 * k + 1]));
      o.iter_ms += ms;
    }
    if (c->term >= 0) break;
    // not finished: continue from where the device really is
    h_light = h_light && h->light_on != 0;
    pred_iter = h->iter;
    carry = std::max(0, h->stop_iter - h->iter);
  }
  o.term = c->term; o.term_iterate = c->term_iterate; o.restarts = c->restarts;
  o.have_check = c->checks > 0;
  for (int t = 0; t < 2; t++) {
    const DevResiduals& d = c->res[t];
    Residuals& R = o.chk.it[t];
    R.pobj = d.pobj; R.dobj = d.dobj; R.pfeas = d.pfeas; R.dfeas = d.dfeas; R.gap = d.gap; R.relgap = d.relgap;
    R.pinf_obj = d.pinf_obj; R.pinf_res = d.pinf_res; R.dinf_obj = d.dinf_obj; R.dinf_res = d.dinf_res;
  }
  if (c->trace) {
    out->trace_len = std::min(c->trace_len, out->trace_cap);
    if (out->trace_len > 0)
      CUDA_OK(cudaMemcpyAsync(out->trace, p->trace_dev.p, (size_t)out->trace_len * B200PDLP_TRACE_COLS * sizeof(double),
                              cudaMemcpyDeviceToHost, s));
  }
  return o;
}

// host-driven loop (cupdlp_solver.c:939-1106)
static LoopOutcome host_loop(b200pdlp_problem* p, const b200pdlp_params& prm, const LoopLimits& lim, b200pdlp_result* out) {
  cudaStream_t s = p->stream;
  PdhgState* h = p->hstate;
  LoopOutcome o;
  RestartMemo memo;
  bool have_spec = false, spec_flag = false;   // a speculative check already produced the next check's scalars
  const bool speculate = can_speculate_check(p);
  CudaEvent ev0, ev1;
  while (h->iter < prm.iter_limit) {
    const bool timed_out_local = lim.over();
    if (have_spec) { o.chk = parse_fused_check(p, spec_flag); have_spec = false; }
    else o.chk = run_check(p, timed_out_local);
    o.have_check = true;
    const Residuals &L = o.chk.it[0], &A = o.chk.it[1];
    if (prm.log_level >= 2)
      printf("[b200pdlp] it %8d  pobj %+.8e dobj %+.8e  pfeas %.2e dfeas %.2e | avg pobj %+.8e dobj %+.8e pfeas %.2e dfeas %.2e  tau %.3e sigma %.3e\n",
             h->iter, L.pobj, L.dobj, L.pfeas, L.dfeas, A.pobj, A.dobj, A.pfeas, A.dfeas, h->tau, h->sigma);
    int choice = 0;
    const int t_code = check_decision(prm, lim.tol_p, lim.tol_d, h, o.chk, memo, &o.term_iterate, &choice);
    if (t_code >= 0) { o.term = t_code; trace_row(out, h, o.chk, 0); break; }
    if (choice) { do_restart(p, choice, o.chk, memo); o.restarts++; arm_step(h); }
    trace_row(out, h, o.chk, choice);
    const int next = next_check_iter(h->iter, lim.interval, prm.iter_limit);
    h->stop_iter = next;
    fill_pow_tables(h);
    push_state(p);
    CUDA_OK(cudaEventRecord(ev0, s));
    bool have_ev1 = false;
    while (true) {
      const int need = next - h->iter;
      if (p->no_graph) {
        for (int q = 0; q < std::min(need + 4, p->graph_main_passes); q++) { enqueue_pass(p); p->launches += p->kernels_per_pass(); }
      } else if (need >= p->graph_main_passes / 2 || need > p->graph_small_passes) {
        CUDA_OK(cudaGraphLaunch(p->graph_main, s));
        p->launches += (long long)p->graph_main_passes * p->kernels_per_pass();
      } else if (need > 1) {
        CUDA_OK(cudaGraphLaunch(p->graph_small, s));
        p->launches += (long long)p->graph_small_passes * p->kernels_per_pass();
      } else {
        enqueue_pass(p);
        p->launches += p->kernels_per_pass();
      }
      if (speculate) {
        if (!have_ev1) { CUDA_OK(cudaEventRecord(ev1, s)); have_ev1 = true; }
        spec_flag = lim.over();
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
    o.iter_ms += ms;
  }
  return o;
}

// B200PDLP_DEBUG_MG: per-rank barrier / exchange counts and checksums of what the postsolve is about to assemble
static void debug_mg_dump(b200pdlp_problem* p, const LoopOutcome& o) {
  const PdhgState* h = p->hstate;
  const int ml = p->ml;
  unsigned long long ep[16] = {0};
  if (p->epochs.p) CUDA_OK(cudaMemcpy(ep, p->epochs.p, sizeof(ep), cudaMemcpyDeviceToHost));
  auto csum = [&](const double* d, int len) {
    std::vector<double> t(std::max(len, 1));
    if (len > 0) CUDA_OK(cudaMemcpy(t.data(), d, (size_t)len * sizeof(double), cudaMemcpyDeviceToHost));
    double a = 0.0; for (int i = 0; i < len; i++) a += t[i] * (1.0 + (i % 7)); return a;
  };
  fprintf(stderr, "[b200pdlp mg-debug] rank %d iter %d cur %d term %d term_iterate %d light_on %d | barrier0 %llu barrier1 %llu exchange %llu | "
          "x[cur] %.17g xavg %.17g y[cur] %.17g yavg %.17g ax[cur] %.17g axavg %.17g aty0 %.17g atyavg %.17g\n",
          p->rank, h->iter, h->cur, o.term, o.term_iterate, h->light_on, ep[0], ep[1], ep[10],
          csum(p->x[h->cur].p, p->nl), csum(p->xavg.p, p->nl), csum(p->y[h->cur].p, ml), csum(p->yavg.p, ml),
          csum(p->ax[h->cur].p, ml), csum(p->axavg.p, ml), csum(p->aty[0].p, p->nl), csum(p->atyavg.p, p->nl));
}

// device order -> standard-form order, whole vectors on every rank.
// Logical shards share ONE CUDA context: a context-synchronising driver call on one rank's host thread (a pageable copy
// that needs staging memory, a lazy module load, an allocation) waits for every running kernel, including a peer's
// barrier kernel that is spinning for THIS rank's next launch -- a deadlock that only the barrier's timeout breaks
// (and the assembly would then run on with stale segments).  So with local links every host-blocking copy
// of the assembly sits between two host-side rendezvous, when no barrier kernel is in flight.  Separate processes
// (CUDA IPC) have separate contexts and do not need this.
struct Assembly {
  b200pdlp_problem* p;
  std::vector<double> t = std::vector<double>(std::max<size_t>(std::max(p->n, std::max(p->ml, 1)), p->xfull.n));   // staging
  const bool dbg = p->world > 1 && getenv("B200PDLP_DEBUG_MG") != nullptr, rendezvous = p->local_link && p->group;
  int dbg_stage = 0;
  void dbg_segments(const char* what) {
    if (!dbg) return;
    char line[1024]; int k = snprintf(line, sizeof line, "[b200pdlp mg-debug] rank %d stage %d %s segments:", p->rank, dbg_stage++, what);
    for (int g = 0; g < p->world && k < 900; g++) {
      double a = 0.0;
      for (int i = 0; i < p->seg_len; i++) a += t[(size_t)g * p->seg_len + i] * (1.0 + (i % 7));
      k += snprintf(line + k, sizeof line - k, " %.15g", a);
    }
    fprintf(stderr, "%s\n", line);
  }
  // barrier of the assembly; with local links the ranks also meet on the host before AND after it (see above): nobody
  // launches a kernel that spins for its peers while a peer's host may still sit in a blocking copy, and nobody starts a
  // blocking copy while a peer's barrier kernel is still in flight
  void xchg() {
    cudaStream_t s = p->stream;
    if (rendezvous) { CUDA_OK(cudaStreamSynchronize(s)); p->group->arrive_and_wait(); }
    launch_p2p_exchange(s, p->outs.p + 60, 0, p->peers, p->world, p->rank, p->epochs.p, p->fault.p);
    p->launches++;
    if (rendezvous) { CUDA_OK(cudaStreamSynchronize(s)); p->group->arrive_and_wait(); }
  }
  // this rank's column shard d -> h, the whole column vector
  void download_cols(const double* d, std::vector<double>& h) {
    cudaStream_t s = p->stream;
    const bool peers = p->world > 1 && p->p2p && !p->comm;
    if (peers) {
      // no NCCL communicator (logical shards of one process, or B200PDLP_NO_NCCL): all-gather through the peers' xfull,
      // with a barrier before anyone reads and one before anyone overwrites
      launch_push_shard(s, d, p->nl, p->peers, p->world, p->rank, p->seg_len);
      p->launches++;
      xchg();
      CUDA_OK(cudaMemcpyAsync(t.data(), p->xfull.p, p->xfull.n * sizeof(double), cudaMemcpyDeviceToHost, s));
      xchg();
    } else if (p->world > 1) {   // all-gather the column shards
      CUDA_OK(cudaMemcpyAsync(p->send.p, d, (size_t)p->nl * sizeof(double), cudaMemcpyDeviceToDevice, s));
      gather_shards(p);
      CUDA_OK(cudaMemcpyAsync(t.data(), p->xfull.p, p->xfull.n * sizeof(double), cudaMemcpyDeviceToHost, s));
    } else {
      CUDA_OK(cudaMemcpyAsync(t.data(), d, (size_t)p->n * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    CUDA_OK(cudaStreamSynchronize(s));
    if (peers) dbg_segments("columns");
    for (int j = 0; j < p->n; j++) h[p->cperm[j]] = t[seg_pos(p, j)];   // (several GPUs: a segmented vector)
  }
  // this rank's rows d -> h, the whole row vector
  void download_rows(const double* d, std::vector<double>& h) {
    cudaStream_t s = p->stream;
    const int m = p->m, ml = p->ml;
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
  }
};

// PDHG_PostSolve (cupdlp_solver.c:1281-1435), on the device (device_prep.cu post_*_kernel) or on the host
static void write_solution(b200pdlp_problem* p, const LoopOutcome& o, b200pdlp_result* out, Laps& lap) {
  const StdForm& f = p->form;
  cudaStream_t s = p->stream;
  const PdhgState* h = p->hstate;
  const int cur = h->cur, nl = p->nl, m = p->m;
  const bool use_avg = (o.term == B200PDLP_OPTIMAL && o.term_iterate == 1);
  const double* dx = use_avg ? p->xavg.p : p->x[cur].p;
  const double* dy = use_avg ? p->yavg.p : p->y[cur].p;
  const double* dax = use_avg ? p->axavg.p : p->ax[cur].p;
  if (p->world > 1 && h->accepted_last && !use_avg) {   // (only when the loop never ran a check, e.g. iter_limit <= 0)
    if (p->p2p) launch_reduce_part_p2p(s, nl, p->aty[0].p, p->peers, p->world, p->rank, p->seg_len, 1);
    else CUDA_OK(cudaMemcpyAsync(p->aty[0].p, p->red.p, (size_t)nl * sizeof(double), cudaMemcpyDeviceToDevice, s));
  }
  throw_if_peer_fault(p, kPeerLate);
  const double* daty = use_avg ? p->atyavg.p : p->aty[p->world == 1 ? cur : 0].p;
  if (p->dev_form) {
    // un-permute, un-scale, sign conventions, slacks of BOUND rows; four original-order vectors come back
    if (out->col_value && out->col_dual && out->row_value && out->row_dual) {
      const int n0 = f.n_orig;
      const bool direct = p->device_io;
      launch_postsolve(s, p->prep.arr, f.sense, o.have_check ? 1 : 0, dx, daty, dy, dax, p->cost.p, p->lower.p, p->upper.p,
                       p->colscale.p, p->rowscale.p, direct ? out->col_value : p->io_col.p, direct ? out->col_dual : p->io_col.p + n0,
                       direct ? out->row_value : p->io_row.p, direct ? out->row_dual : p->io_row.p + m);
      p->launches += 2;
      if (!direct) {
        CUDA_OK(cudaMemcpyAsync(out->col_value, p->io_col.p, (size_t)n0 * sizeof(double), cudaMemcpyDeviceToHost, s));
        CUDA_OK(cudaMemcpyAsync(out->col_dual, p->io_col.p + n0, (size_t)n0 * sizeof(double), cudaMemcpyDeviceToHost, s));
        CUDA_OK(cudaMemcpyAsync(out->row_value, p->io_row.p, (size_t)m * sizeof(double), cudaMemcpyDeviceToHost, s));
        CUDA_OK(cudaMemcpyAsync(out->row_dual, p->io_row.p + m, (size_t)m * sizeof(double), cudaMemcpyDeviceToHost, s));
      }
    }
    CUDA_OK(cudaStreamSynchronize(s));
    lap("solve", "postsolve (device) + download");
    return;
  }
  std::vector<double> hx(p->n), hy(m, 0.0), hax(m, 0.0), haty(p->n);
  {
    Assembly a{p};
    a.download_cols(dx, hx); a.download_cols(daty, haty); a.download_rows(dy, hy); a.download_rows(dax, hax);
  }
  // a barrier of the assembly that timed out leaves stale segments behind: an error, not a result
  throw_if_peer_fault(p, "P2P barrier timed out while the solution was being assembled (a peer rank did not arrive)");
  lap("solve", "solution download");
  host_postsolve(f, o.have_check, hx, hy, hax, haty, out);
}

static void solve_on_device(b200pdlp_problem* p, const b200pdlp_params& prm, const b200pdlp_warm* warm, b200pdlp_result* out) {
  NvtxRange nvtx("b200pdlp: solve");
  nvtxRangePushA("b200pdlp: initial point + graphs");
  using clk = std::chrono::steady_clock;
  set_device(p);
  const auto t_begin = clk::now();
  const StdForm& f = p->form;
  const int interval = prm.check_interval > 0 ? prm.check_interval : 40;
  const bool dev_checks = use_device_checks(p, prm);
  const bool logical_shards = p->local_link && p->group;
  const long long launches0 = p->launches;
  PdhgState* h = p->hstate;
  memset(h, 0, sizeof(PdhgState));
  h->adaptive = prm.adaptive_step != 0;
  out->trace_len = 0;
  Laps lap;
  lap.rank = p->world > 1 ? p->rank : -1;
  if (logical_shards) {
    prepare_graphs(p, prm, interval, dev_checks, /*eager=*/true);
    CUDA_OK(cudaStreamSynchronize(p->stream));
    lap("solve", "graphs ready (logical shards)");
    p->group->arrive_and_wait();
  }
  start_point(p, warm);
  init_step_sizes(p, h);
  start_products_and_sums(p);
  arm_step(h);
  fill_pow_tables(h);
  push_state(p);
  CUDA_OK(cudaStreamSynchronize(p->stream));
  lap("solve", "initial point + state");
  if (!logical_shards) prepare_graphs(p, prm, interval, dev_checks, /*eager=*/false);
  lap("solve", "graph capture");
  nvtxRangePop();

  nvtxRangePushA("b200pdlp: PDHG loop");
  CudaEvent evl0, evl1;
  CUDA_OK(cudaEventRecord(evl0, p->stream));
  const LoopLimits lim{interval, prm.tol_primal * (1.0 + f.norm_rhs), prm.tol_dual * (1.0 + f.norm_cost),
                       time_limit_or_none(prm.time_limit), clk::now()};
  const LoopOutcome o = dev_checks ? device_loop(p, prm, warm, lim, out) : host_loop(p, prm, lim, out);
  CUDA_OK(cudaEventRecord(evl1, p->stream));
  CUDA_OK(cudaEventSynchronize(evl1));
  float loop_ms = 0.f;
  CUDA_OK(cudaEventElapsedTime(&loop_ms, evl0, evl1));
  const double solve_seconds = lim.elapsed();
  out->loop_device_ms = loop_ms;
  lap("solve", "iterations");
  nvtxRangePop();

  NvtxRange nvtx_post("b200pdlp: postsolve + download");
  if (p->world > 1 && getenv("B200PDLP_DEBUG_MG")) debug_mg_dump(p, o);
  write_solution(p, o, out, lap);
  fill_result(out, f, h, o.term, o.term_iterate, o.restarts, o.chk);
  out->kernel_launches = (int)std::min<long long>(p->launches - launches0, 2147483647LL);
  out->solve_seconds = solve_seconds;
  out->iter_device_ms = o.iter_ms;
  out->setup_seconds += std::chrono::duration<double>(lim.t_loop - t_begin).count();
  lap("solve", "postsolve (host)");
}

// A problem of b200pdlp_hipdlp_problem_create holds the HiPDLP iterate set only (hipdlp_buffers), and one of
// b200pdlp_problem_create the pdlp one only: each family of entry points rejects the other's problems.
static bool is_hipdlp_problem(const b200pdlp_problem* p) { return p->hip.state.p != nullptr; }
void require_mode(const b200pdlp_problem* p, bool hipdlp, const char* who) {
  if (is_hipdlp_problem(p) == hipdlp) return;
  throw Error(B200PDLP_ERR_ARG, std::string(who) + (hipdlp ? ": not a HiPDLP problem (create it with b200pdlp_hipdlp_problem_create)"
                                                           : ": a HiPDLP problem (use the b200pdlp_hipdlp_* entry points)"));
}

// the kernel-level entry points' copies of host vectors in standard-form order: d[i] = v[perm[i]] (upload_perm) and back
// (download_perm), each synchronised with the problem's stream
void upload_perm(b200pdlp_problem* p, double* d, const double* v, const std::vector<int>& perm) {
  const int len = (int)perm.size();
  if (len == 0) return;
  std::vector<double> t(len);
  for (int i = 0; i < len; i++) t[i] = v[perm[i]];
  CUDA_OK(cudaMemcpyAsync(d, t.data(), (size_t)len * sizeof(double), cudaMemcpyHostToDevice, p->stream));
  CUDA_OK(cudaStreamSynchronize(p->stream));
}
void download_perm(b200pdlp_problem* p, double* v, const double* d, const std::vector<int>& perm) {
  const int len = (int)perm.size();
  if (len == 0) return;
  std::vector<double> t(len);
  CUDA_OK(cudaMemcpyAsync(t.data(), d, (size_t)len * sizeof(double), cudaMemcpyDeviceToHost, p->stream));
  CUDA_OK(cudaStreamSynchronize(p->stream));
  for (int i = 0; i < len; i++) v[perm[i]] = t[i];
}

// ---- the device prologue against its host twin, array by array, bit for bit (report[0..31], see include/b200pdlp.h)
// one sliced-ELL matrix of the device prologue against the host's: *r_slices = -1 if the sizes differ
void cmp_sell(const DevSellOwned& D, const SellMatrix& H, double* r_slices, double* r_col, double* r_val, double* r_long) {
  if ((size_t)D.nslices != H.slices.size() || D.padded != H.padded || (size_t)D.nlong != H.long_rows.size() ||
      (size_t)D.nsegs != H.segs.size() || D.lcount != H.lcount) { *r_slices = -1; return; }
  *r_slices = dev_mismatches(reinterpret_cast<const int*>(D.slices), reinterpret_cast<const int*>(H.slices.data()), 4 * H.slices.size());
  *r_col = dev_mismatches(D.col, H.col.data(), (size_t)H.padded);
  *r_val = dev_mismatches(D.val, H.val.data(), (size_t)H.padded);
  *r_long = dev_mismatches(reinterpret_cast<const int*>(D.long_rows), reinterpret_cast<const int*>(H.long_rows.data()), 4 * H.long_rows.size()) +
            dev_mismatches(reinterpret_cast<const int*>(D.segs), reinterpret_cast<const int*>(H.segs.data()), 4 * H.segs.size()) +
            dev_mismatches(D.lcol, H.lcol.data(), H.lcol.size()) + dev_mismatches(D.lval, H.lval.data(), H.lval.size());
}
// the arrays of a one-problem prologue; false if the sizes differ (nothing else is compared then)
bool prep_compare_arrays(const DevicePrologue& P, const StdForm& f, const HostLayout& L, double* report) {
  const DevProblemArrays& a = P.arr;
  const int n = f.n, m = f.m, nnz = f.nnz;
  report[0] = a.n != n; report[1] = a.m != m; report[2] = a.nnz != nnz; report[3] = a.neq != f.neq;
  if (report[0] + report[1] + report[2] + report[3] > 0) return false;
  report[4] = dev_mismatches(P.form.cbeg, f.cbeg.data(), n + 1);
  report[5] = dev_mismatches(P.form.cidx, f.cidx.data(), nnz);
  report[6] = dev_mismatches(P.form.cval, f.cval.data(), nnz);
  report[7] = dev_mismatches(P.form.cost, f.cost.data(), n);
  report[8] = dev_mismatches(P.form.lower, f.lower.data(), n);
  report[9] = dev_mismatches(P.form.upper, f.upper.data(), n);
  report[10] = dev_mismatches(P.form.colscale, f.col_scale.data(), n);
  report[11] = dev_mismatches(P.form.rhs, f.rhs.data(), m);
  report[12] = dev_mismatches(P.form.rowscale, f.row_scale.data(), m);
  report[13] = dev_mismatches(P.form.rptr, f.rptr.data(), m + 1);
  report[14] = dev_mismatches(P.form.rpos, f.rpos.data(), nnz);
  report[15] = dev_mismatches(a.row_new_idx, f.row_new_idx.data(), m);
  report[16] = dev_mismatches(a.row_class, f.row_class.data(), m);
  report[17] = dev_mismatches(a.rperm, L.rperm.data(), m);
  report[18] = dev_mismatches(a.cperm, L.cperm.data(), n);
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
      bad += dev_mismatches(dev, t.data(), len);
    };
    cmp_perm(a.cost, f.cost, L.cperm, n); cmp_perm(a.lower, f.lower, L.cperm, n); cmp_perm(a.upper, f.upper, L.cperm, n);
    cmp_perm(a.colscale, f.col_scale, L.cperm, n); cmp_perm(a.rhs, f.rhs, L.rperm, m); cmp_perm(a.rowscale, f.row_scale, L.rperm, m);
    report[30] = bad;
  }
  report[31] = P.sc.cols_sorted;
  return true;
}

}  // namespace b200

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
      if (use_device_prep(*lp, *params, world)) { open_problem(p, params->device, 0, 1); create_problem_device(*lp, *params, p); }
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
    require_mode(p, false, "b200pdlp_spmv_ax");
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
    require_mode(p, false, "b200pdlp_spmv_aty");
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
    require_mode(p, false, "b200pdlp_primal_step");
    if (p->world != 1) throw Error(B200PDLP_ERR_ARG, "kernel-level entry points are single-GPU");
    set_device(p);
    ensure_host_maps(p);
    const int n = p->n;
    upload_perm(p, p->x[0].p, x, p->cperm);
    upload_perm(p, p->aty[0].p, aty, p->cperm);
    kernel_api_state(p, tau, tau);
    const ReduceScratch r1 = p->rs(kSlotK1, n);
    launch_primal_step(p->stream, n, p->state.p, p->x[0].p, p->x[1].p, p->aty[0].p, p->aty[1].p, p->cost.p, p->lower.p,
                       p->upper.p, p->xsum.p, r1, p->A.dev.nzmap);
    p->launches++;
    download_perm(p, x_new, p->x[1].p, p->cperm);
    if (dx2) *dx2 = sum_partials(p, r1, primal_step_grid(n));
    CUDA_OK(cudaGetLastError());
  });
}

int b200pdlp_dual_step(b200pdlp_problem* p, const double* x_new, const double* y, const double* ax, double sigma,
                       double* y_new, double* ax_new, double* dy2) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !x_new || !y || !ax || !y_new || !ax_new) throw Error(B200PDLP_ERR_ARG, "null argument");
    require_mode(p, false, "b200pdlp_dual_step");
    if (p->world != 1) throw Error(B200PDLP_ERR_ARG, "kernel-level entry points are single-GPU");
    set_device(p);
    ensure_host_maps(p);
    const int m = p->m;
    cudaStream_t s = p->stream;
    upload_perm(p, p->x[1].p, x_new, p->cperm);
    upload_perm(p, p->y[0].p, y, p->rperm);
    upload_perm(p, p->ax[0].p, ax, p->rperm);
    kernel_api_state(p, sigma, sigma);
    const ReduceScratch r2 = p->rs(kSlotK2, m);
    if (p->A.dev.nzmap) launch_nz_bitmap(s, p->n, p->x[1].p, p->A.dev.nzmap);   // x' came from the caller, not from K1
    launch_spmv_dual(s, p->A.dev, p->state.p, p->x[0].p, p->x[1].p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p, p->rhs.p,
                     p->ysum.p, p->neq_local, 0, r2, nullptr, p->AT.dev.nzmap);
    p->launches++;
    download_perm(p, y_new, p->y[1].p, p->rperm);
    download_perm(p, ax_new, p->ax[1].p, p->rperm);
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
    require_mode(p, false, "b200pdlp_residuals");
    if (p->world != 1) throw Error(B200PDLP_ERR_ARG, "kernel-level entry points are single-GPU");
    set_device(p);
    ensure_host_maps(p);
    const int n = p->n, m = p->m;
    cudaStream_t s = p->stream;
    upload_perm(p, p->x[0].p, x, p->cperm);
    upload_perm(p, p->y[0].p, y, p->rperm);
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

// the restart sums |x - xlr|^2, |y - ylr|^2 from the restart sweep's block partials, added in check_finish_kernel's order:
// thread t adds partials t, t + 128, ... from 0, a shuffle tree inside each warp, then the four warps in order
static void finish_order_sums(const std::vector<double>& prst, int nbs, double d2[2]) {
  constexpr int kT = 128;
  for (int a = 0; a < 2; a++) {
    double w[kT / 32];
    for (int g = 0; g < kT / 32; g++) {
      double v[32];
      for (int l = 0; l < 32; l++) {
        double s = 0.0;
        for (int i = g * 32 + l; i < nbs; i += kT) s += prst[(size_t)a * nbs + i];
        v[l] = s;
      }
      for (int o = 16; o > 0; o >>= 1)
        for (int l = 0; l + o < 32; l++) v[l] = v[l] + v[l + o];   // (ascending l reads v[l + o] before it changes)
      w[g] = v[0];
    }
    double s = 0.0;
    for (int g = 0; g < kT / 32; g++) s += w[g];
    d2[a] = s;
  }
}

int b200pdlp_check_device(b200pdlp_problem* p, const b200pdlp_check_in* in, double* x, double* y, double* ax, double* aty,
                          double* xsum, double* ysum, double* xlr, double* ylr, double* axsum, double* atysum, double* xavg,
                          double* yavg, double* axavg, double* atyavg, b200pdlp_check_out* out) {
  DeviceGuard dg;
  return guarded([&] {
    const char* who = "b200pdlp_check_device";
    if (!p || !in || !x || !y || !ax || !aty || !xsum || !ysum || !xlr || !ylr || !xavg || !yavg || !axavg || !atyavg || !out ||
        (in->light && (!axsum || !atysum)))
      throw Error(B200PDLP_ERR_ARG, std::string(who) + ": null argument");
    require_mode(p, false, who);
    if (p->world != 1) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": kernel-level entry points are single-GPU");
    if (p->ordered) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": an ordered-mode problem (its checks run on the host)");
    if (in->interval < 1 || in->iter < 0 || in->step_iter < 0)
      throw Error(B200PDLP_ERR_ARG, std::string(who) + ": interval must be >= 1, iter and step_iter >= 0");
    if (in->light && (!p->axsum.p || !p->atysum.p || in->iter >= kDenseChecks))
      throw Error(B200PDLP_ERR_ARG, std::string(who) + ": the light check needs iter < 10 and a problem that carries A xSum");
    set_device(p);
    ensure_host_maps(p);
    const int n = p->n;
    cudaStream_t s = p->stream;
    const bool light = in->light != 0;
    upload_perm(p, p->x[0].p, x, p->cperm); upload_perm(p, p->aty[0].p, aty, p->cperm);
    upload_perm(p, p->xsum.p, xsum, p->cperm); upload_perm(p, p->xlr.p, xlr, p->cperm);
    upload_perm(p, p->y[0].p, y, p->rperm); upload_perm(p, p->ax[0].p, ax, p->rperm);
    upload_perm(p, p->ysum.p, ysum, p->rperm); upload_perm(p, p->ylr.p, ylr, p->rperm);
    if (light) { upload_perm(p, p->atysum.p, atysum, p->cperm); upload_perm(p, p->axsum.p, axsum, p->rperm); }
    // the state and control blocks of a solve at its check iteration
    const double nan = std::numeric_limits<double>::quiet_NaN();
    PdhgState* h = p->hstate;
    memset(h, 0, sizeof(PdhgState));
    h->iter = in->iter; h->step_iter = in->step_iter; h->adaptive = in->adaptive; h->pending = in->pending;
    h->beta = in->beta; h->tau = in->tau; h->sigma = in->sigma; h->sum_step = in->sum_step; h->w_pending = in->w_pending;
    h->eta = h->tau_try = h->sigma_try = nan;
    for (int t = 0; t < kPowTab; t++) h->pow_red[t] = h->pow_grow[t] = nan;
    h->pow_base = -1;
    h->stop_iter = in->iter; h->cur = 0; h->light_on = light ? 1 : 0; h->done = 0;
    push_state(p);
    if (p->trace_dev.n < (size_t)B200PDLP_TRACE_COLS) p->trace_dev.alloc(B200PDLP_TRACE_COLS, false);
    CUDA_OK(cudaMemsetAsync(p->trace_dev.p, 0, B200PDLP_TRACE_COLS * sizeof(double), s));
    SolveCtl* c = reset_ctl(p, in->tol_p, in->tol_d, in->tol_gap, in->iter_limit, in->interval, in->restart_on != 0);
    *p->htime = in->time_flag;
    c->time_flag = mapped_time_flag(p);
    c->pf_lr = in->pf_lr; c->df_lr = in->df_lr; c->gap_lr = in->gap_lr;
    c->pf_lc = in->pf_lc; c->df_lc = in->df_lc; c->gap_lc = in->gap_lc;
    c->last_restart_iter = in->last_restart_iter;
    c->trace = p->trace_dev.p; c->trace_cap = 1;
    CUDA_OK(cudaMemcpyAsync(p->ctl.p, c, sizeof(SolveCtl), cudaMemcpyHostToDevice, s));
    p->launches += enqueue_check_device(p, light);
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaMemcpyAsync(c, p->ctl.p, sizeof(SolveCtl), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaMemcpyAsync(h, p->state.p, sizeof(PdhgState), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaMemcpyAsync(out->trace, p->trace_dev.p, B200PDLP_TRACE_COLS * sizeof(double), cudaMemcpyDeviceToHost, s));
    const int nbs = restart_sweep_grid(n, p->ml);
    std::vector<double> prst((size_t)2 * nbs);
    CUDA_OK(cudaMemcpyAsync(prst.data(), p->rs(kSlotK1, n).partials, prst.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CUDA_OK(cudaStreamSynchronize(s));
    for (int a = 0; a < 28; a++) out->sums[a] = c->sums[a];
    for (int t = 0; t < 2; t++) {
      const DevResiduals& R = c->res[t];
      const double v[10] = {R.pobj, R.dobj, R.pfeas, R.dfeas, R.gap, R.relgap, R.pinf_obj, R.pinf_res, R.dinf_obj, R.dinf_res};
      for (int k = 0; k < 10; k++) out->res[t][k] = v[k];
    }
    out->term = c->term; out->term_iterate = c->term_iterate;
    out->restart_choice = c->trace_len > 0 ? (int)out->trace[12] : 0;
    out->restarts = c->restarts; out->checks = c->checks; out->trace_len = c->trace_len; out->done = h->done;
    out->stop_iter = h->stop_iter; out->pending = h->pending; out->pow_base = h->pow_base;
    out->pf_lr = c->pf_lr; out->df_lr = c->df_lr; out->gap_lr = c->gap_lr;
    out->pf_lc = c->pf_lc; out->df_lc = c->df_lc; out->gap_lc = c->gap_lc;
    out->last_restart_iter = c->last_restart_iter; out->reserved = 0;
    out->beta = h->beta; out->tau = h->tau; out->sigma = h->sigma; out->eta = h->eta;
    out->tau_try = h->tau_try; out->sigma_try = h->sigma_try; out->sum_step = h->sum_step;
    out->restart_sq[0] = out->restart_sq[1] = 0.0;
    if (out->restart_choice) finish_order_sums(prst, nbs, out->restart_sq);
    for (int t = 0; t < kPowTab; t++) { out->pow_red[t] = h->pow_red[t]; out->pow_grow[t] = h->pow_grow[t]; }
    download_perm(p, x, p->x[0].p, p->cperm); download_perm(p, aty, p->aty[0].p, p->cperm);
    download_perm(p, xsum, p->xsum.p, p->cperm); download_perm(p, xlr, p->xlr.p, p->cperm);
    download_perm(p, xavg, p->xavg.p, p->cperm); download_perm(p, atyavg, p->atyavg.p, p->cperm);
    download_perm(p, y, p->y[0].p, p->rperm); download_perm(p, ax, p->ax[0].p, p->rperm);
    download_perm(p, ysum, p->ysum.p, p->rperm); download_perm(p, ylr, p->ylr.p, p->rperm);
    download_perm(p, yavg, p->yavg.p, p->rperm); download_perm(p, axavg, p->axavg.p, p->rperm);
    if (light) { download_perm(p, atysum, p->atysum.p, p->cperm); download_perm(p, axsum, p->axsum.p, p->rperm); }
  });
}

// one record per long row of M: {standard-form row, first slot, segments}; perm maps M's device rows to standard-form order
static int long_row_records(const DeviceMatrix& M, const std::vector<int>& perm, int32_t* out) {
  std::vector<int4> lr(M.long_rows.n);
  if (!lr.empty()) CUDA_OK(cudaMemcpy(lr.data(), M.long_rows.p, lr.size() * sizeof(int4), cudaMemcpyDeviceToHost));
  for (size_t k = 0; k < lr.size(); k++) {
    out[3 * k] = perm[lr[k].x];
    out[3 * k + 1] = M.dev.nblocks_body + lr[k].y;
    out[3 * k + 2] = lr[k].z;
  }
  return (int)lr.size();
}

int b200pdlp_pass_partials(b200pdlp_problem* p, const double* x, const double* y, const double* ax, const double* aty,
                           double tau, double sigma, double* x_new, double* y_new, double* ax_new, double* aty_new,
                           double* slots, int32_t cap, int32_t* long_rows, int32_t long_cap, b200pdlp_pass_out* out) {
  DeviceGuard dg;
  return guarded([&] {
    const char* who = "b200pdlp_pass_partials";
    if (!p || !x || !y || !ax || !aty || !x_new || !y_new || !ax_new || !aty_new || !slots || !long_rows || !out)
      throw Error(B200PDLP_ERR_ARG, std::string(who) + ": null argument");
    require_mode(p, false, who);
    if (p->world != 1) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": kernel-level entry points are single-GPU");
    if (p->ordered) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": an ordered-mode problem (its sums add terms, not slots)");
    const int n = p->n;
    const int nb[3] = {primal_step_grid(n), p->A.grid(), p->AT.grid()};
    const int nlong = (int)(p->A.long_rows.n + p->AT.long_rows.n);
    if (cap < std::max(nb[0], std::max(nb[1], nb[2])) || long_cap < nlong)
      throw Error(B200PDLP_ERR_ARG, std::string(who) + ": cap must be >= " + std::to_string(std::max(nb[0], std::max(nb[1], nb[2]))) +
                                        " and long_cap >= " + std::to_string(nlong));
    set_device(p);
    ensure_host_maps(p);
    upload_perm(p, p->x[0].p, x, p->cperm); upload_perm(p, p->aty[0].p, aty, p->cperm);
    upload_perm(p, p->y[0].p, y, p->rperm); upload_perm(p, p->ax[0].p, ax, p->rperm);
    kernel_api_state(p, tau, sigma);
    enqueue_pass(p);
    p->launches += p->kernels_per_pass();
    CUDA_OK(cudaGetLastError());
    const int slot_ids[3] = {kSlotK1, kSlotK2, kSlotK3};
    for (int k = 0; k < 3; k++)
      CUDA_OK(cudaMemcpyAsync(slots + (size_t)k * cap, p->rs(slot_ids[k], 0).partials, (size_t)nb[k] * sizeof(double),
                              cudaMemcpyDeviceToHost, p->stream));
    pull_state(p);
    out->dx2 = p->hstate->dx2; out->dy2 = p->hstate->dy2; out->inter = p->hstate->inter;
    for (int k = 0; k < 3; k++) out->slots[k] = nb[k];
    out->long_a = long_row_records(p->A, p->rperm, long_rows);
    out->long_at = long_row_records(p->AT, p->cperm, long_rows + 3 * (size_t)out->long_a);
    download_perm(p, x_new, p->x[1].p, p->cperm); download_perm(p, aty_new, p->aty[1].p, p->cperm);
    download_perm(p, y_new, p->y[1].p, p->rperm); download_perm(p, ax_new, p->ax[1].p, p->rperm);
  });
}

int b200pdlp_bench_spmv(b200pdlp_problem* p, int32_t which, int32_t reps, float* ms_total) {
  DeviceGuard dg;
  return guarded([&] {
    if (!p || !ms_total || reps < 1) throw Error(B200PDLP_ERR_ARG, "bad argument");
    require_mode(p, false, "b200pdlp_bench_spmv");
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
    require_mode(p, false, "b200pdlp_bench_pass");
    set_device(p);
    cudaStream_t s = p->stream;
    PdhgState* st = p->state.p;
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
                           p->upper.p, p->xsum.p, r1, p->A.dev.nzmap);
        CUDA_OK(cudaEventRecord(ev[1], s));
        launch_spmv_dual(s, p->A.dev, st, p->x[0].p, p->x[1].p, p->y[0].p, p->y[1].p, p->ax[0].p, p->ax[1].p,
                         p->rhs.p, p->ysum.p, p->neq_local, 0, r2, nullptr, p->AT.dev.nzmap);
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
          p->launches += p->kernels_per_pass();
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
      p->launches += p->kernels_per_pass();
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
    require_mode(p, false, "b200pdlp_problem_solve");
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
    if (use_device_prep(*lp, *params, 1)) { open_problem(p.get(), params->device, 0, 1); create_problem_device(*lp, *params, p.get()); }
    else create_problem(*lp, *params, 0, 1, p.get());
    out->setup_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    solve_on_device(p.get(), *params, warm, out);
    CUDA_OK(cudaGetLastError());
    Laps lap;
    p.reset();
    lap("solve", "teardown");
  });
}

int b200pdlp_solve_device(const b200pdlp_lp* lp, const b200pdlp_params* params, const b200pdlp_warm* warm, b200pdlp_result* out) {
  DeviceGuard dg;
  const char* who = "b200pdlp_solve_device";
  return guarded([&] {
    if (!lp || !params || !out) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": null argument");
    check_params(*params);
    b200pdlp_params prm = *params;
    solve_lp_device(*lp, false, prm.device, prm.ordered_max, warm, out, who, [&] { solve_batch_device(1, lp, prm, warm, out); },
                    [&](const b200pdlp_lp& l, b200pdlp_problem* q) { create_problem(l, prm, 0, 1, q); },
                    [&](const b200pdlp_lp& l, b200pdlp_problem* q) { create_problem_device(l, prm, q); },
                    [&](b200pdlp_problem* q, const b200pdlp_lp&, const b200pdlp_warm* w, b200pdlp_result* r) { solve_on_device(q, prm, w, r); });
    CUDA_OK(cudaGetLastError());
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