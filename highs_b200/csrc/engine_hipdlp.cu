// highs_b200/csrc/engine_hipdlp.cu -- host side of the HiPDLP mode (reflected Halpern PDHG) on one GPU and on several,
// and its entry points of the C ABI (include/b200pdlp.h).
#include "engine.hpp"

namespace b200 {

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

// the host form's cost, bounds, scaling factors, rhs (= row lower) and row upper in the device orders (cperm, rperm)
static void upload_hipdlp_vectors(b200pdlp_problem* p, const StdForm& f, const int* cperm, const int* rperm) {
  const int n = f.n, m = f.m;
  upload_permuted(p->cost, f.cost, cperm, 0, n, n); upload_permuted(p->lower, f.lower, cperm, 0, n, n);
  upload_permuted(p->upper, f.upper, cperm, 0, n, n); upload_permuted(p->colscale, f.col_scale, cperm, 0, n, n);
  upload_permuted(p->rhs, f.rhs, rperm, 0, m, m); upload_permuted(p->hip.rup, f.row_upper, rperm, 0, m, m);
  upload_permuted(p->rowscale, f.row_scale, rperm, 0, m, m);
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
  upload_hipdlp_vectors(p, f, p->cperm.data(), p->rperm.data());
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
  upload_hipdlp_vectors(p, f, S.cperm.data(), S.rperm.data());
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
void hip_host_postsolve(const b200pdlp_lp& lp, const StdForm& f, const int* cperm, const int* rperm, const double* x,
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

// PDLPSolver::powerMethod (pdhg.cc:1529-1671) on the device: 20 iterations of q <- A A'q / |A A'q| from the ones vector,
// lambda = |A'q|^2; no host round trip inside (the norm stays on the device), one read-back at the end.  Several GPUs:
// every rank holds q and z whole, forms its columns of w and its rows of z, and gathers them; the norms are then the
// one-GPU sums over full vectors.  Uses dy, axp, atdy (and atyp on several GPUs) as scratch.
static double hip_power_method(b200pdlp_problem* p) {
  auto& h = p->hip;
  cudaStream_t s = p->stream;
  const int n = p->n, m = p->m;
  const bool shard = hip_sharded(p);
  const int r0 = p->hip_r0, c0 = p->hip_c0;
  if (n == 0 || m == 0) return 1.0;
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
  return p->houts[16];
}

// one row of b200pdlp_result::trace per block (B200PDLP_HIP_TRACE_COLS, include/b200pdlp.h) from the block-end check's sums
// and the controller's decisions: host values the loop already holds, no device work
void hip_trace_row(b200pdlp_result* out, const HipController& ctl, const double* sums, bool restart, bool converged) {
  if (!out->trace || out->trace_len >= out->trace_cap) return;
  double* t = out->trace + (size_t)out->trace_len * B200PDLP_HIP_TRACE_COLS;
  t[0] = ctl.iters;
  for (int q = 0; q < 9; q++) t[1 + q] = sums[q];
  t[10] = restart ? 1.0 : 0.0;
  t[11] = restart ? ctl.primal_weight : 0.0;
  t[12] = restart ? ctl.primal_step : 0.0;
  t[13] = restart ? ctl.dual_step : 0.0;
  t[14] = ctl.fpe;
  t[15] = converged ? 1.0 : 0.0;
  out->trace_len++;
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
  const int c0 = p->hip_c0;
  out->trace_len = 0;
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
  const double op_norm_sq = hip_power_method(p);
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
      const bool block_converged =
          ctl.pfeas < ctl.tol * (1.0 + f.norm_rhs) && ctl.dfeas < ctl.tol * (1.0 + f.norm_cost) && ctl.relgap < ctl.tol;
      hip_trace_row(out, ctl, p->houts, restart, block_converged);
      if (block_converged) { converged = true; sol_x = h.xn.p; sol_y = h.yn.p; break; }
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

// ---- HiPDLP kernel-level entry points (tests): one Halpern step (hip_step), one check (hip_check) and the power method
// (hip_power_method) of the solve, on host vectors in standard-form order, single GPU.  Like the pdlp ones they use the
// problem's iterate buffers as scratch.
static void hip_kernel_api(b200pdlp_problem* p, const char* who) {
  if (!p) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": null problem");
  require_mode(p, true, who);
  if (p->world != 1 || hip_sharded(p)) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": kernel-level entry points are single-GPU");
  set_device(p);
  ensure_host_maps(p);
  if ((int)p->cperm.size() != p->n || (int)p->rperm.size() != p->m)
    throw Error(B200PDLP_ERR_STATE, std::string(who) + ": the problem has no host copy of its orderings");
}
}  // namespace b200

extern "C" {

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

int b200pdlp_hipdlp_problem_create(const b200pdlp_lp* lp, const b200pdlp_hipdlp_params* params, b200pdlp_problem** out) {
  DeviceGuard dg;
  return guarded([&] {
    if (!params || !out) throw Error(B200PDLP_ERR_ARG, "b200pdlp_hipdlp_problem_create: null argument");
    check_lp(lp);
    ProblemPtr p(new b200pdlp_problem());
    create_problem_hipdlp(*lp, *params, p.get());
    *out = p.release();
  });
}

int b200pdlp_hipdlp_step(b200pdlp_problem* p, double primal_step, double dual_step, int32_t halpern_iteration, int32_t k_offset,
                         int32_t is_major, double* x, const double* xa, double* aty, double* y, const double* ya, double* rx,
                         double* xn, double* hslack, double* yn, double* ry) {
  DeviceGuard dg;
  return guarded([&] {
    if (!x || !xa || !aty || !y || !ya || !rx || !xn || !hslack || !yn || !ry)
      throw Error(B200PDLP_ERR_ARG, "b200pdlp_hipdlp_step: null argument");
    hip_kernel_api(p, "b200pdlp_hipdlp_step");
    auto& h = p->hip;
    const std::vector<int>&cp = p->cperm, &rp = p->rperm;
    upload_perm(p, h.x.p, x, cp); upload_perm(p, h.xa.p, xa, cp); upload_perm(p, h.aty.p, aty, cp);
    upload_perm(p, h.xn.p, xn, cp); upload_perm(p, h.hslack.p, hslack, cp);
    upload_perm(p, h.y.p, y, rp); upload_perm(p, h.ya.p, ya, rp); upload_perm(p, h.yn.p, yn, rp); upload_perm(p, h.ry.p, ry, rp);
    h.hstate->primal_step = primal_step; h.hstate->dual_step = dual_step; h.hstate->halpern_iteration = halpern_iteration;
    CUDA_OK(cudaMemcpyAsync(h.state.p, h.hstate, sizeof(HipState), cudaMemcpyHostToDevice, p->stream));
    hip_step(p, k_offset, is_major ? 1 : 0);
    CUDA_OK(cudaGetLastError());
    download_perm(p, x, h.x.p, cp); download_perm(p, rx, h.rx.p, cp); download_perm(p, aty, h.aty.p, cp);
    download_perm(p, xn, h.xn.p, cp); download_perm(p, hslack, h.hslack.p, cp);
    download_perm(p, y, h.y.p, rp); download_perm(p, yn, h.yn.p, rp); download_perm(p, ry, h.ry.p, rp);
  });
}

int b200pdlp_hipdlp_check(b200pdlp_problem* p, int32_t major, const double* x, const double* y, const double* xa,
                          const double* ya, const double* rx, const double* ry, const double* hslack, double out[9],
                          double* sp, double* sn, double* ax, double* aty, double* atdy) {
  DeviceGuard dg;
  return guarded([&] {
    if (!x || !y || !xa || !ya || !out || !sp || !sn || !ax || !aty || !atdy || (major && (!rx || !ry || !hslack)))
      throw Error(B200PDLP_ERR_ARG, "b200pdlp_hipdlp_check: null argument");
    hip_kernel_api(p, "b200pdlp_hipdlp_check");
    auto& h = p->hip;
    const std::vector<int>&cp = p->cperm, &rp = p->rperm;
    upload_perm(p, major ? h.xn.p : h.x.p, x, cp); upload_perm(p, h.xa.p, xa, cp);
    upload_perm(p, major ? h.yn.p : h.y.p, y, rp); upload_perm(p, h.ya.p, ya, rp);
    if (major) { upload_perm(p, h.rx.p, rx, cp); upload_perm(p, h.hslack.p, hslack, cp); upload_perm(p, h.ry.p, ry, rp); }
    hip_check(p, major ? 1 : 0);
    CUDA_OK(cudaGetLastError());
    for (int q = 0; q < 9; q++) out[q] = p->houts[q];
    download_perm(p, sp, h.sp.p, cp); download_perm(p, sn, h.sn.p, cp);
    download_perm(p, ax, h.axp.p, rp); download_perm(p, aty, h.atyp.p, cp);
    if (major) download_perm(p, atdy, h.atdy.p, cp);
    else std::fill(atdy, atdy + p->n, 0.0);
  });
}

int b200pdlp_hipdlp_problem_power_method(b200pdlp_problem* p, double* lambda) {
  DeviceGuard dg;
  return guarded([&] {
    if (!lambda) throw Error(B200PDLP_ERR_ARG, "b200pdlp_hipdlp_problem_power_method: null argument");
    hip_kernel_api(p, "b200pdlp_hipdlp_problem_power_method");
    *lambda = hip_power_method(p);
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
    report[32] = dev_mismatches(P.form.row_upper, f.row_upper.data(), m);
    {
      std::vector<double> t(m);
      for (int i = 0; i < m; i++) t[i] = f.row_upper[L.rperm[i]];
      report[33] = dev_mismatches(P.arr.rup, t.data(), m);
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
      report[34] = dev_mismatches(P.arr.orow_ptr, ptr.data(), m + 1);
      report[35] = dev_mismatches(P.arr.orow_col, col.data(), nnz0) + dev_mismatches(P.arr.orow_val, val.data(), nnz0);
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
        return dev_mismatches(dev, t.data(), len);
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
    report[6] = dev_mismatches(a.rperm, S.rperm.data(), m) + dev_mismatches(a.cperm, S.cperm.data(), n);
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

}  // extern "C"
