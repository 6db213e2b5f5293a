// highs_b200/csrc/engine_batch.cu -- host side of the batches of small LPs (PDLP and HiPDLP mode, host or device arrays),
// their prologue / postsolve comparators and the KKT batch, with their entry points of the C ABI (include/b200pdlp.h).
#include "engine.hpp"

namespace b200 {

// b200pdlp_solve_batch: every member is an ordered-mode problem, solved by one CTA of batch_round_kernel (batch_kernels.cu).
// The host runs each member's prologue (formulate, scale, build_layout with identity orderings) on its threads, packs every
// member into a few pooled buffers, then drives ROUNDS: one launch, one read-back of the control blocks and states, the
// decisions of every member that checked (the same functions solve_on_device calls), one upload.  Each member returns the
// bits b200pdlp_solve returns for it alone.

// every batch runs on `device` (< 0: the current device); returns its number
int select_device(int device) {
  device_count_checked();
  if (device >= 0) CUDA_OK(cudaSetDevice(device));
  int current = 0;
  CUDA_OK(cudaGetDevice(&current));
  return current;
}

// a member of a host-array batch must be an ordered-mode problem (max(n, m) <= ordered_max) under the row classification of
// its mode (std_form_cols with row_inf: formulate's 1e20, or HiPDLP's infinity as in use_device_prep_hipdlp): checked before
// any device work
static void check_ordered_member(const b200pdlp_lp* lp, int ordered_max, double row_inf, int i, const char* who) {
  const int rc = guarded([&] {
    check_lp(lp);
    const int omax = ordered_max == 0 ? 4096 : ordered_max;
    if (omax < 0) throw Error(B200PDLP_ERR_ARG, "ordered_max < 0: a batch solves ordered-mode problems only");
    const int n = std_form_cols(*lp, row_inf);
    if (std::max(n, lp->num_row) > omax)
      throw Error(B200PDLP_ERR_ARG, "standard form " + std::to_string(lp->num_row) + " x " + std::to_string(n) +
                                        " exceeds ordered_max = " + std::to_string(omax));
  });
  if (rc != B200PDLP_OK) throw Error(rc, std::string(who) + ": member " + std::to_string(i) + ": " + g_last_error);
}

// a member of b200pdlp_solve_hipdlp_batch_mixed: true for a tree member (HiPDLP's classification puts its standard form past
// ordered_max, or ordered_max < 0), which must fit the cluster kernel (batch_kernels.cu: every check sum and dot product one
// element per thread of hip_tree_blocks' grid); checked before any device work
constexpr int kTreeMemberMax = 262144;
static bool check_mixed_member(const b200pdlp_lp* lp, int ordered_max, int i, const char* who) {
  bool tree = false;
  const int rc = guarded([&] {
    check_lp(lp);
    const int omax = ordered_max == 0 ? 4096 : ordered_max;
    const int n = std_form_cols(*lp, std::numeric_limits<double>::infinity());
    const int big = std::max(n, lp->num_row);
    tree = omax < 0 || big > omax;
    if (tree && big > kTreeMemberMax)
      throw Error(B200PDLP_ERR_ARG, "standard form " + std::to_string(lp->num_row) + " x " + std::to_string(n) +
                                        " exceeds max(n, m) = " + std::to_string(kTreeMemberMax) +
                                        " of a tree member: solve it with b200pdlp_solve_hipdlp");
  });
  if (rc != B200PDLP_OK) throw Error(rc, std::string(who) + ": member " + std::to_string(i) + ": " + g_last_error);
  return tree;
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

// a member of a host-array batch: its layouts from the host prologue and its offsets in the batch's pools
struct PooledMember {
  HostLayout L;
  size_t vec = 0, sl_a = 0, sl_at = 0, e_a = 0, e_at = 0;
  // tree-mode layouts only (b200pdlp_solve_hipdlp_batch_mixed): the long rows' descriptors, entries and the scratch
  size_t sg_a = 0, lr_a = 0, sg_at = 0, lr_at = 0, le_a = 0, le_at = 0, scr = 0;
};

// the scratch doubles of a tree-mode member (HipTreeMember): the check's block partials and the segment partials of A and,
// twice, of A'; none for an ordered layout
static size_t tree_scratch_len(const PooledMember& b) {
  if (b.L.ordered) return 0;
  return 9 * (size_t)hip_tree_blocks(std::max(b.L.A.ncols, b.L.A.nrows)) + (size_t)b.L.A.n_partials + 2 * (size_t)b.L.AT.n_partials;
}

struct BatchHost : BatchRun, PooledMember {   // one member of b200pdlp_solve_batch on the host
  std::vector<double> x0, y0;
};

// the vectors of a member's block `v` (BatchVec) as BatchMember pointers
static void batch_member_vectors(BatchMember& M, double* v, int n, int m) {
  using V = BatchVec;
  auto c = [&](int k) { return V::col(v, n, k); };
  auto r = [&](int k) { return V::row(v, n, m, k); };
  M.n = n; M.m = m;
  M.cost = c(V::kCost); M.lower = c(V::kLower); M.upper = c(V::kUpper); M.colscale = c(V::kColscale);
  M.x0 = c(V::kX0); M.x1 = c(V::kX1); M.aty0 = c(V::kAty0); M.aty1 = c(V::kAty1);
  M.xsum = c(V::kXsum); M.xavg = c(V::kXavg); M.atyavg = c(V::kAtyavg); M.xlr = c(V::kXlr);
  M.rhs = r(V::kRhs); M.rowscale = r(V::kRowscale);
  M.y0 = r(V::kY0); M.y1 = r(V::kY1); M.ax0 = r(V::kAx0); M.ax1 = r(V::kAx1);
  M.ysum = r(V::kYsum); M.yavg = r(V::kYavg); M.axavg = r(V::kAxavg); M.ylr = r(V::kYlr);
}

// the layouts of a member descriptor (BatchMember, HipBatchMember)
template <class D>
static void set_layouts(D& M, const int4* a_slices, const int* a_col, const double* a_val, const int4* at_slices,
                        const int* at_col, const double* at_val) {
  M.a_slices = a_slices; M.a_col = a_col; M.a_val = a_val;
  M.at_slices = at_slices; M.at_col = at_col; M.at_val = at_val;
}
static void set_layouts(HipTreeMember& M, const int4* a_slices, const int* a_col, const double* a_val, const int4* at_slices,
                        const int* at_col, const double* at_val) {
  set_layouts(M.b, a_slices, a_col, a_val, at_slices, at_col, at_val);
}

// The pooled device buffers of a host-array batch: every member's vector block, and the slice descriptors, column ids and
// values of its A and A'
struct BatchPools {
  std::vector<double> hvec;   // the host copy of the vector blocks (the host postsolve downloads them into it)
  DevBuf<double> vec, val;
  DevBuf<int> col;
  DevBuf<int4> sl;
  DevBuf<int4> lsg;           // tree-mode layouts: segs and long_rows of A and A'
  DevBuf<int> lcol;
  DevBuf<double> lval, scr;
};

// Lays the members out in the pools (block_len(n, m): the doubles of a vector block), packs their layouts, lets fill(i, v)
// write member i's vector block v (zeroed) on the host threads, and uploads the pools and the members' descriptors
// (D, whose vectors describe(M, i, v) sets for device block v) on s; returns with s idle.
template <class D, class Member, class Fill, class Describe>
static void upload_pools(cudaStream_t s, std::vector<Member>& B, size_t (*block_len)(int, int), Fill&& fill,
                         Describe&& describe, BatchPools& P, DevBuf<D>& dmem) {
  const int count = (int)B.size();
  size_t nvec = 0, nsl = 0, nent = 0, nlsg = 0, nle = 0, nscr = 0;
  for (Member& b : B) {
    b.vec = nvec; nvec += block_len(b.f.n, b.f.m);
    b.sl_a = nsl; nsl += b.L.A.slices.size();
    b.sl_at = nsl; nsl += b.L.AT.slices.size();
    b.e_a = nent; nent += b.L.A.col.size();
    b.e_at = nent; nent += b.L.AT.col.size();
    b.sg_a = nlsg; nlsg += b.L.A.segs.size();
    b.lr_a = nlsg; nlsg += b.L.A.long_rows.size();
    b.sg_at = nlsg; nlsg += b.L.AT.segs.size();
    b.lr_at = nlsg; nlsg += b.L.AT.long_rows.size();
    b.le_a = nle; nle += b.L.A.segs.empty() ? 0 : b.L.A.lcol.size();
    b.le_at = nle; nle += b.L.AT.segs.empty() ? 0 : b.L.AT.lcol.size();
    b.scr = nscr; nscr += tree_scratch_len(b);
  }
  P.hvec.assign(std::max<size_t>(nvec, 1), 0.0);
  std::vector<double> hval(std::max<size_t>(nent, 1), 0.0);
  std::vector<int> hcol(std::max<size_t>(nent, 1), 0);
  std::vector<int4> hsl(std::max<size_t>(nsl, 1)), hlsg(std::max<size_t>(nlsg, 1));
  std::vector<int> hlcol(std::max<size_t>(nle, 1), 0);
  std::vector<double> hlval(std::max<size_t>(nle, 1), 0.0);
  for_members(count, [&](int i) {
    const Member& b = B[i];
    fill(i, P.hvec.data() + b.vec);
    static_assert(sizeof(SellMatrix::Slice) == sizeof(int4), "descriptor layout");
    memcpy(hsl.data() + b.sl_a, b.L.A.slices.data(), b.L.A.slices.size() * sizeof(int4));
    memcpy(hsl.data() + b.sl_at, b.L.AT.slices.data(), b.L.AT.slices.size() * sizeof(int4));
    std::copy(b.L.A.col.begin(), b.L.A.col.end(), hcol.begin() + b.e_a);
    std::copy(b.L.AT.col.begin(), b.L.AT.col.end(), hcol.begin() + b.e_at);
    std::copy(b.L.A.val.begin(), b.L.A.val.end(), hval.begin() + b.e_a);
    std::copy(b.L.AT.val.begin(), b.L.AT.val.end(), hval.begin() + b.e_at);
    static_assert(sizeof(SellMatrix::Seg) == sizeof(int4) && sizeof(SellMatrix::LongRow) == sizeof(int4), "descriptor layout");
    auto longs = [&](const SellMatrix& S, size_t sg, size_t lr, size_t le) {
      if (S.segs.empty()) return;
      memcpy(hlsg.data() + sg, S.segs.data(), S.segs.size() * sizeof(int4));
      memcpy(hlsg.data() + lr, S.long_rows.data(), S.long_rows.size() * sizeof(int4));
      std::copy(S.lcol.begin(), S.lcol.end(), hlcol.begin() + le);
      std::copy(S.lval.begin(), S.lval.end(), hlval.begin() + le);
    };
    longs(b.L.A, b.sg_a, b.lr_a, b.le_a);
    longs(b.L.AT, b.sg_at, b.lr_at, b.le_at);
  });
  P.vec.alloc(P.hvec.size(), false); P.val.alloc(hval.size(), false); P.col.alloc(hcol.size(), false); P.sl.alloc(hsl.size(), false);
  if (nlsg > 0) { P.lsg.alloc(hlsg.size(), false); P.lcol.alloc(hlcol.size(), false); P.lval.alloc(hlval.size(), false); }
  if (nscr > 0) P.scr.alloc(nscr, false);
  dmem.alloc(count, false);
  std::vector<D> hmem((size_t)count);
  for (int i = 0; i < count; i++) {
    const Member& b = B[i];
    describe(hmem[i], i, P.vec.p + b.vec);
    set_layouts(hmem[i], P.sl.p + b.sl_a, P.col.p + b.e_a, P.val.p + b.e_a, P.sl.p + b.sl_at, P.col.p + b.e_at, P.val.p + b.e_at);
  }
  CUDA_OK(cudaMemcpyAsync(P.vec.p, P.hvec.data(), P.hvec.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(P.val.p, hval.data(), hval.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(P.col.p, hcol.data(), hcol.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(P.sl.p, hsl.data(), hsl.size() * sizeof(int4), cudaMemcpyHostToDevice, s));
  if (nlsg > 0) {
    CUDA_OK(cudaMemcpyAsync(P.lsg.p, hlsg.data(), hlsg.size() * sizeof(int4), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaMemcpyAsync(P.lcol.p, hlcol.data(), hlcol.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaMemcpyAsync(P.lval.p, hlval.data(), hlval.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  }
  CUDA_OK(cudaMemcpyAsync(dmem.p, hmem.data(), (size_t)count * sizeof(D), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaStreamSynchronize(s));
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
    h->beta = step_beta(r.cost_sq, r.rhs_sq);
    if (h->adaptive) adaptive_step_sizes(h, r.f.amax);
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
  const double t_lim = time_limit_or_none(prm.time_limit);
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
        fixed_step_sizes(h, c.outs[kBatchLambda]);
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
  select_device(prm.device);
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

  // ---- the pools, one descriptor per member; identity orderings (ordered mode): standard-form order is device order
  using V = BatchVec;
  BatchPools pools;
  DevBuf<BatchMember> dmem;
  upload_pools(s, B, V::len, [&](int i, double* v) {
    const BatchHost& b = B[i];
    const StdForm& f = b.f;
    const int n = f.n, m = f.m;
    std::copy(f.cost.begin(), f.cost.end(), V::col(v, n, V::kCost));
    std::copy(f.lower.begin(), f.lower.end(), V::col(v, n, V::kLower));
    std::copy(f.upper.begin(), f.upper.end(), V::col(v, n, V::kUpper));
    std::copy(f.col_scale.begin(), f.col_scale.end(), V::col(v, n, V::kColscale));
    std::copy(b.x0.begin(), b.x0.end(), V::col(v, n, V::kX0));
    double* xsum = V::col(v, n, V::kXsum);
    for (int j = 0; j < n; j++) xsum[j] = proj_zero(f, j);
    std::copy(f.rhs.begin(), f.rhs.end(), V::row(v, n, m, V::kRhs));
    std::copy(f.row_scale.begin(), f.row_scale.end(), V::row(v, n, m, V::kRowscale));
    std::copy(b.y0.begin(), b.y0.end(), V::row(v, n, m, V::kY0));
  }, [&](BatchMember& M, int i, double* v) {
    batch_member_vectors(M, v, B[i].f.n, B[i].f.m);
    M.neq = B[i].L.neq_local;
  }, pools, dmem);
  lap("batch", "pools + upload");

  std::vector<BatchRun*> R((size_t)count);
  for (int i = 0; i < count; i++) R[i] = &B[i];
  PinnedArray<PdhgState> hst((size_t)count);
  const BatchLoop loop = batch_rounds(s, count, prm, dmem.p, R, hst.p, outs);
  lap("batch", "rounds");

  // ---- PDHG_PostSolve of every member, on the host
  NvtxRange nvtx_post("b200pdlp: batch postsolve + download");
  CUDA_OK(cudaMemcpyAsync(pools.hvec.data(), pools.vec.p, pools.hvec.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  const double setup_seconds = std::chrono::duration<double>(loop.t_loop - t_begin).count();
  for_members(count, [&](int i) {
    BatchHost& b = B[i];
    const StdForm& f = b.f;
    const PdhgState* h = hst.p + i;
    const int n = f.n, m = f.m, cur = h->cur;
    const bool use_avg = b.term == B200PDLP_OPTIMAL && b.term_iterate == 1;
    const double* v = pools.hvec.data() + b.vec;
    const double* dx = V::col(v, n, use_avg ? V::kXavg : V::kX0 + cur);
    const double* daty = V::col(v, n, use_avg ? V::kAtyavg : V::kAty0 + cur);
    const double* dy = V::row(v, n, m, use_avg ? V::kYavg : V::kY0 + cur);
    const double* dax = V::row(v, n, m, use_avg ? V::kAxavg : V::kAx0 + cur);
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

// every array pointer of the batch (warms: NULL for none) must be device memory of `device`: the lowest failing member, field
static void check_device_arrays(int count, const b200pdlp_lp* lps, const b200pdlp_warm* warms, const b200pdlp_result* outs,
                                int device, const char* who) {
  for (int i = 0; i < count; i++) {
    check_device_lp(lps[i], device, i, who);
    if (warms) {
      check_device_array(warms[i].col_value, device, i, "warm col_value", who);
      check_device_array(warms[i].row_value, device, i, "warm row_value", who);
      check_device_array(warms[i].row_dual, device, i, "warm row_dual", who);
    }
    check_device_result(outs[i], device, i, who);
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
  DevBuf<double> dbls, vec, val;   // the form's values and the scaling factors: nnz + 2 n + m; the vector blocks; the layouts' values
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

// The members' descriptors and the sizing kernel (the array checks, the row classes and orders, the form's dimensions):
// one read-back of `count` records into D.size, on stream s of the current device.  lps[i] / warms[i]: host structs whose
// arrays are device memory.
static void device_batch_size(cudaStream_t s, int count, const b200pdlp_lp* lps, const b200pdlp_warm* warms,
                              const PrepMode& mode, DeviceBatch& D) {
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
  D.prep.alloc(count, false); D.dsize.alloc(count, false);
  CUDA_OK(cudaMemcpyAsync(D.prep.p, D.hp.data(), (size_t)count * sizeof(BatchPrep), cudaMemcpyHostToDevice, s));
  if (mode.hip) launch_hip_batch_size(s, count, D.prep.p, D.dsize.p);
  else launch_batch_size(s, count, D.prep.p, D.dsize.p);
  CUDA_OK(cudaGetLastError());
  D.size.resize((size_t)count);
  CUDA_OK(cudaMemcpyAsync(D.size.data(), D.dsize.p, (size_t)count * sizeof(BatchSize), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
}

// The pools and the prologue kernel of ordered members whose sizing D holds (D.hp, D.size; D.prep is allocated anew when it
// does not hold `count` descriptors), then one read-back of the scalar records, on stream s.
static void device_batch_prep(cudaStream_t s, int count, const b200pdlp_lp* lps, const PrepMode& mode, DeviceBatch& D) {
  if (D.prep.n != (size_t)count) D.prep.alloc(count, false);
  D.drec.alloc((size_t)count * kPrepRec, false);
  // ---- the pools: each member's slices of them
  size_t ni = 0, nd = 0, nv = 0, nsl = 0, ne = 0;
  for (int i = 0; i < count; i++) {
    const BatchSize& z = D.size[i];
    const size_t n = z.n, m = lps[i].num_row, nnz = z.nnz;
    ni += 3 * nnz + n + m + 1;
    if (mode.hip) ni += m + 1 + (nnz - n) + 2 * (size_t)lps[i].num_col;   // optr, opos (nnz0), sortcols
    nd += nnz + 2 * n + m;
    nv += mode.hip ? HipBatchVec::len(z.n, lps[i].num_row) : BatchVec::len(z.n, lps[i].num_row);
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
    nv += mode.hip ? HipBatchVec::len(n, m) : BatchVec::len(n, m);
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
    // rec[kRecCostSq], rec[kRecRhsSq] of every member: |c|^2 and |b|^2 of the unscaled form
    CUDA_OK(cudaMemcpy2DAsync(D.rec.data(), kPrepRec * sizeof(double), D.drec.p, kPrepRec * sizeof(double), 2 * sizeof(double),
                              count, cudaMemcpyDeviceToHost, s));
  } else {
    launch_batch_prep(s, count, D.prep.p, mode.scaling != 0);
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaMemcpyAsync(D.rec.data(), D.drec.p, D.rec.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  }
  CUDA_OK(cudaStreamSynchronize(s));
}

// Validation and sizing (one read-back of `count` records), the pools, then the prologue (one read-back of the scalar
// records), on stream s of the current device.  lps[i] / warms[i]: host structs whose arrays are device memory.
static void device_batch_prologue(cudaStream_t s, int count, const b200pdlp_lp* lps, const b200pdlp_warm* warms,
                                  const PrepMode& mode, int ordered_max, const char* who, DeviceBatch& D, Laps& lap) {
  const int omax = ordered_max == 0 ? 4096 : ordered_max;
  device_batch_size(s, count, lps, warms, mode, D);
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
  device_batch_prep(s, count, lps, mode, D);
  lap("batch device", "prologue (device)");
}

void solve_batch_device(int count, const b200pdlp_lp* lps, const b200pdlp_params& prm, const b200pdlp_warm* warms,
                               b200pdlp_result* outs) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  Laps lap;
  const int device = select_device(prm.device);
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
    f.norm_cost = std::sqrt(r[kRecCostSq]); f.norm_rhs = std::sqrt(r[kRecRhsSq]); f.amax = r[kRecAmax];
    b.cost_sq = r[kRecScaledCostSq]; b.rhs_sq = r[kRecScaledRhsSq];
    b.tol_p = prm.tol_primal * (1.0 + f.norm_rhs);
    b.tol_d = prm.tol_dual * (1.0 + f.norm_cost);
    R[i] = &b;
    BatchMember& M = hmem[i];
    batch_member_vectors(M, P.vec, P.n, P.m);
    M.neq = P.neq;
    set_layouts(M, P.a_slices, P.a_col, P.a_val, P.at_slices, P.at_col, P.at_val);
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

// ---- b200pdlp_debug_batch_prep_compare / _hipdlp_batch_prep_compare: the device prologues and postsolves against their
// host twins
static const int kBatchPrepItems = 27;
static const int kHipBatchPrepItems = 24;

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
  RawLps(int count, const b200pdlp_lp* lps) {
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
};

// a member's ordered sliced-ELL layout from the device prologue (slices, column ids, values) against the host's: r[0..2]
// (r[1], r[2] = -1 when the slices differ)
static void sell_mismatches(const SellMatrix& H, const int4* sl, const int* col, const double* val, double* r) {
  const size_t ns = H.slices.size(), ne = H.col.size();
  r[0] = dev_mismatches(sl, reinterpret_cast<const int4*>(H.slices.data()), ns);
  if (r[0] != 0.0) { r[1] = r[2] = -1.0; return; }
  r[1] = dev_mismatches(col, H.col.data(), ne);
  r[2] = dev_mismatches(val, H.val.data(), ne);
}

// fresh device vectors, in `out`, for the postsolve of every member's probe: post[i]'s col_value and col_dual (n0 each),
// row_value and row_dual (m each); its other fields zero
template <class Post>
static void probe_outputs(const DeviceBatch& D, DevBuf<double>& out, std::vector<Post>& post) {
  size_t len = 0;
  for (const BatchPrep& P : D.hp) len += 2 * (size_t)P.n0 + 2 * (size_t)P.m;
  out.alloc(len, false);
  post.assign(D.hp.size(), Post{});
  len = 0;
  for (size_t i = 0; i < D.hp.size(); i++) {
    const int n0 = D.hp[i].n0, m = D.hp[i].m;
    double* o = out.p + len;
    post[i].col_value = o; post[i].col_dual = o + n0; post[i].row_value = o + 2 * n0; post[i].row_dual = o + 2 * n0 + m;
    len += 2 * (size_t)n0 + 2 * (size_t)m;
  }
}

static void batch_prep_compare(int count, const b200pdlp_lp* lps, int scaling, double* report) {
  using V = BatchVec;
  device_count_checked();
  RawLps raw(count, lps);
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
    const double* v = P.vec;
    rep[1] = dev_mismatches(V::col(v, n, V::kCost), f.cost.data(), n);
    rep[2] = dev_mismatches(V::col(v, n, V::kLower), f.lower.data(), n);
    rep[3] = dev_mismatches(V::col(v, n, V::kUpper), f.upper.data(), n);
    rep[4] = dev_mismatches(V::row(v, n, m, V::kRhs), f.rhs.data(), m);
    rep[5] = dev_mismatches(V::col(v, n, V::kColscale), f.col_scale.data(), n);
    rep[6] = dev_mismatches(V::row(v, n, m, V::kRowscale), f.row_scale.data(), m);
    rep[7] = dev_mismatches(P.row_new_idx, f.row_new_idx.data(), m);
    static_assert(sizeof(RowClass) == sizeof(int), "row classes are ints");
    rep[8] = dev_mismatches(P.row_class, reinterpret_cast<const int*>(f.row_class.data()), m);
    sell_mismatches(L.A, P.a_slices, P.a_col, P.a_val, rep + 9);
    sell_mismatches(L.AT, P.at_slices, P.at_col, P.at_val, rep + 12);
    rep[15] = dev_mismatches(V::col(v, n, V::kX0), x0.data(), n);
    rep[16] = dev_mismatches(V::row(v, n, m, V::kY0), y0.data(), m);
    std::vector<double> xsum(n);
    for (int j = 0; j < n; j++) xsum[j] = proj_zero(f, j);
    rep[17] = dev_mismatches(V::col(v, n, V::kXsum), xsum.data(), n);
    const double* r = D.rec.data() + (size_t)kPrepRec * i;
    double cost_sq = 0.0, rhs_sq = 0.0;
    for (int j = 0; j < n; j++) cost_sq += f.cost[j] * f.cost[j];
    for (int q = 0; q < m; q++) rhs_sq += f.rhs[q] * f.rhs[q];
    const double got[5] = {std::sqrt(r[kRecCostSq]), std::sqrt(r[kRecRhsSq]), r[kRecAmax], r[kRecScaledCostSq], r[kRecScaledRhsSq]};
    const double want[5] = {f.norm_cost, f.norm_rhs, f.amax, cost_sq, rhs_sq};
    for (int k = 0; k < 5; k++) rep[18 + k] = memcmp(got + k, want + k, sizeof(double)) != 0;
  }
  // the postsolve of a probe iterate (x, A'y, y, A x in half 0 of every block, a check assumed) into fresh device vectors
  std::vector<BatchPost> hpost;
  DevBuf<double> dout;
  probe_outputs(D, dout, hpost);
  std::vector<std::vector<double>> probes((size_t)count);
  for (int i = 0; i < count; i++) {
    const BatchPrep& P = D.hp[i];
    const int n = P.n, m = P.m;
    std::vector<double>& pr = probes[i];   // x, A'y (n each), y, A x (m each)
    pr.resize(2 * (size_t)n + 2 * (size_t)m);
    for (size_t k = 0; k < pr.size(); k++) pr[k] = batch_probe(i, (int)k);
    double* v = P.vec;
    CUDA_OK(cudaMemcpy(V::col(v, n, V::kX0), pr.data(), n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(V::col(v, n, V::kAty0), pr.data() + n, n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(V::row(v, n, m, V::kY0), pr.data() + 2 * n, m * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(V::row(v, n, m, V::kAx0), pr.data() + 2 * n + m, m * sizeof(double), cudaMemcpyHostToDevice));
    hpost[i].have_check = 1;
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
    rep[23] = dev_mismatches(q.col_value, cv.data(), n0);
    rep[24] = dev_mismatches(q.col_dual, cd.data(), n0);
    rep[25] = dev_mismatches(q.row_value, rv.data(), m);
    rep[26] = dev_mismatches(q.row_dual, rdual.data(), m);
  }
}

// ----------------------------------------------------------------------------------- batch of small LPs, HiPDLP mode
// b200pdlp_solve_hipdlp_batch: every member is an ordered-mode HiPDLP problem, solved by one CTA of hip_batch_round_kernel
// (batch_kernels.cu).  The host prologue (formulate_hipdlp, scale_hipdlp, build_layout) runs on host threads; the members are
// packed into pooled buffers, one descriptor each.  A round is one block of 40 Halpern steps for every unfinished member
// (round 0: the power method, the initial point and the iteration-0 check): one upload of the control blocks and states, one
// launch, one read-back, then each member's HipController decisions in the order solve_hipdlp_on_device takes them.  The
// PID weight's log / exp / log10 stay on the host.  Each member returns the bits b200pdlp_solve_hipdlp returns for it alone.

struct HipBatchRun {   // one member's host control over the rounds
  StdForm f;           // b200pdlp_solve_hipdlp_batch_device fills the scalars only: dimensions, sense, offset, norms, scaled
  HipController ctl;
  bool converged = false, timed_out = false;
  int sol = 0;   // converged: 0 at the iteration-0 check (x, y), 1 after a block (xn, yn)
  b200pdlp_result* trace = nullptr;   // b200pdlp_solve_hipdlp_batch_mixed: the result whose trace rows the blocks write
};

struct HipBatchHost : HipBatchRun, PooledMember {};   // one member of b200pdlp_solve_hipdlp_batch on the host

// the vectors of a HiPDLP member's block `v` (HipBatchVec) and its scalars as HipBatchMember fields
static void hip_batch_member(HipBatchMember& M, const StdForm& f, int neq, double* v) {
  using V = HipBatchVec;
  const int n = f.n, m = f.m;
  auto c = [&](int k) { return V::col(v, n, k); };
  auto r = [&](int k) { return V::row(v, n, m, k); };
  M.n = n; M.m = m; M.neq = neq; M.scaled = f.scaled ? 1 : 0; M.offset = f.offset;
  M.cost = c(V::kCost); M.lower = c(V::kLower); M.upper = c(V::kUpper); M.colscale = c(V::kColscale);
  M.x = c(V::kX); M.xa = c(V::kXa); M.xn = c(V::kXn); M.rx = c(V::kRx); M.aty = c(V::kAty); M.hslack = c(V::kHslack);
  M.atyp = c(V::kAtyp); M.atdy = c(V::kAtdy); M.sp = c(V::kSp); M.sn = c(V::kSn);
  M.rlo = r(V::kRlo); M.rup = r(V::kRup); M.rowscale = r(V::kRowscale);
  M.y = r(V::kY); M.ya = r(V::kYa); M.yn = r(V::kYn); M.ry = r(V::kRy); M.axp = r(V::kAxp); M.dy = r(V::kDy);
}

// The rounds of a HiPDLP batch, for every entry point: one upload of the control blocks and states, one launch per group,
// one read-back, then each member's HipController decisions in the order solve_hipdlp_on_device takes them, until no member
// is active or the time limit has passed.  Members [0, count - ntree) are ordered members (dmem, one CTA each), the rest
// tree members (dtree, one cluster of `cluster` CTAs each).
static BatchLoop hip_batch_rounds(cudaStream_t s, int count, const b200pdlp_hipdlp_params& prm, const HipBatchMember* dmem,
                                  const std::vector<HipBatchRun*>& B, const HipTreeMember* dtree = nullptr, int ntree = 0,
                                  int cluster = 1) {
  const int nord = count - ntree;
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
  const double t_lim = time_limit_or_none(prm.time_limit);
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
    launch_hip_batch_round(s, nord, dmem, dst.p, dctl.p);
    CUDA_OK(launch_hip_tree_round(s, ntree, cluster, dtree, dst.p + nord, dctl.p + nord));
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
        const bool block_converged = ctl.block_converged();
        if (b.trace) hip_trace_row(b.trace, ctl, c.outs, restart, block_converged);
        if (block_converged) {
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
  hip_fill_result(out, b.f, b.ctl, b.converged, b.timed_out);
  out->kernel_launches = (int)std::min<long long>(L.rounds, 2147483647LL);
  out->setup_seconds = setup_seconds;
  out->solve_seconds = L.solve_seconds;
  out->loop_device_ms = L.loop_ms;
  out->iter_device_ms = L.iter_ms;
}

// b200pdlp_solve_hipdlp_batch_mixed: the same rounds for members of any size up to kTreeMemberMax.  The tree-mode members
// (past ordered_max) take their tree layouts from the same host prologue and run on hip_tree_round_kernel (batch_kernels.cu),
// one thread-block cluster each, beside the ordered members' CTAs; each returns the bits b200pdlp_solve_hipdlp returns for it.
// STATUS: runs on hardware; tests/test_gpu_hipdlp_batch_mixed.py, tools/hipdlp_batch_mixed_bench.py (DESIGN.md section 6).

// B200PDLP_BATCH_CLUSTER=1|2|4|8 (tests, benchmarks), otherwise the largest C in {8, 4, 2} with which every one of the
// `ntree` clusters of the round kernel is resident at once, otherwise 1.  C changes no result (see batch_kernels.cu).
static int tree_cluster(int ntree) {
  if (const char* e = getenv("B200PDLP_BATCH_CLUSTER")) {
    const int c = atoi(e);
    if (c != 1 && c != 2 && c != 4 && c != 8) throw Error(B200PDLP_ERR_ARG, "B200PDLP_BATCH_CLUSTER must be 1, 2, 4 or 8");
    return c;
  }
  for (int c : {8, 4, 2}) {
    int fit = 0;
    if (hip_tree_max_clusters(ntree, c, &fit) != cudaSuccess) { cudaGetLastError(); continue; }
    if (fit >= ntree) return c;
  }
  return 1;
}

// b200pdlp_solve_hipdlp_batch and _batch_mixed (`mixed`: the results take the blocks' trace rows): device member k is the
// caller's member src[k]; members [0, count - ntree) are ordered members, the others tree members
static void solve_hipdlp_batch(int count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params& prm, b200pdlp_result* outs,
                               const std::vector<int>& src, int ntree, bool mixed) {
  using clk = std::chrono::steady_clock;
  const auto t_begin = clk::now();
  Laps lap;
  select_device(prm.device);
  StreamHolder sh;
  cudaStream_t s = sh.s;
  const int nord = count - ntree;
  std::vector<HipBatchHost> B((size_t)count);
  {
    NvtxRange nvtx("b200pdlp: HiPDLP batch prologue (host threads)");
    for_members(count, [&](int k) {
      HipBatchHost& b = B[k];
      formulate_hipdlp(lps[src[k]], b.f);
      scale_hipdlp(b.f, prm.scaling_mode, prm.ruiz_iterations);
      build_layout(b.f, 0, 1, prm.ordered_max, b.L);
      if (k < nord && (!b.L.ordered || !b.L.A.segs.empty() || !b.L.AT.segs.empty()))
        throw Error(B200PDLP_ERR_STATE, "the layout is not an ordered-mode layout");
      if (k >= nord && b.L.ordered) throw Error(B200PDLP_ERR_STATE, "the layout is not a tree-mode layout");
    });
  }
  lap("batch", "HiPDLP prologue (host threads)");

  // ---- the pools, one descriptor per member; the vectors in device order, as create_problem_hipdlp uploads them
  using V = HipBatchVec;
  BatchPools pools;
  DevBuf<HipTreeMember> dtree;
  upload_pools(s, B, V::len, [&](int k, double* v) {
    const HipBatchHost& b = B[k];
    const StdForm& f = b.f;
    const int n = f.n, m = f.m;
    const int* cperm = b.L.cperm.data();
    const int* rperm = b.L.rperm.data();
    double *cost = V::col(v, n, V::kCost), *lower = V::col(v, n, V::kLower), *upper = V::col(v, n, V::kUpper);
    double* colscale = V::col(v, n, V::kColscale);
    for (int j = 0; j < n; j++) {
      cost[j] = f.cost[cperm[j]]; lower[j] = f.lower[cperm[j]]; upper[j] = f.upper[cperm[j]]; colscale[j] = f.col_scale[cperm[j]];
    }
    double *rlo = V::row(v, n, m, V::kRlo), *rup = V::row(v, n, m, V::kRup), *rowscale = V::row(v, n, m, V::kRowscale);
    for (int r = 0; r < m; r++) { rlo[r] = f.rhs[rperm[r]]; rup[r] = f.row_upper[rperm[r]]; rowscale[r] = f.row_scale[rperm[r]]; }
  }, [&](HipTreeMember& M, int k, double* v) {
    const HipBatchHost& b = B[k];
    hip_batch_member(M.b, b.f, b.L.neq_local, v);
    auto longs = [&](HipTreeLong& T, const SellMatrix& S, size_t sg, size_t lr, size_t le) {
      T.nsegs = (int)S.segs.size(); T.nlong = (int)S.long_rows.size();
      T.segs = pools.lsg.p + sg; T.long_rows = pools.lsg.p + lr; T.lcol = pools.lcol.p + le; T.lval = pools.lval.p + le;
    };
    longs(M.la, b.L.A, b.sg_a, b.lr_a, b.le_a);
    longs(M.lat, b.L.AT, b.sg_at, b.lr_at, b.le_at);
    M.nb = hip_tree_blocks(std::max(b.f.n, b.f.m));
    if (b.L.ordered) return;
    M.partials = pools.scr.p + b.scr;
    M.a_part = M.partials + 9 * (size_t)M.nb;
    M.at_part[0] = M.a_part + b.L.A.n_partials;
    M.at_part[1] = M.at_part[0] + b.L.AT.n_partials;
  }, pools, dtree);
  // the ordered members' descriptors: the HipBatchMember that leads each of their HipTreeMember descriptors
  DevBuf<HipBatchMember> dmem;
  dmem.alloc(nord, false);
  if (nord > 0)
    CUDA_OK(cudaMemcpy2DAsync(dmem.p, sizeof(HipBatchMember), dtree.p, sizeof(HipTreeMember), sizeof(HipBatchMember), nord,
                              cudaMemcpyDeviceToDevice, s));
  const int cluster = ntree > 0 ? tree_cluster(ntree) : 1;
  lap("batch", "pools + upload");
  if (lap.on && ntree > 0) fprintf(stderr, "[b200pdlp batch] tree members %d, cluster of C = %d CTAs each\n", ntree, cluster);

  std::vector<HipBatchRun*> R((size_t)count);
  for (int k = 0; k < count; k++) {
    R[k] = &B[k];
    if (mixed) { B[k].trace = outs + src[k]; B[k].trace->trace_len = 0; }
  }
  const BatchLoop loop = hip_batch_rounds(s, count, prm, dmem.p, R, dtree.p + nord, ntree, cluster);
  lap("batch", "rounds");

  // ---- the host postsolve of every member (hip_host_postsolve, as the single solve's host prologue path), one download
  NvtxRange nvtx_post("b200pdlp: HiPDLP batch postsolve + download");
  CUDA_OK(cudaMemcpyAsync(pools.hvec.data(), pools.vec.p, pools.hvec.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  const double setup_seconds = std::chrono::duration<double>(loop.t_loop - t_begin).count();
  for_members(count, [&](int k) {
    const HipBatchHost& b = B[k];
    const StdForm& f = b.f;
    const int n = f.n, m = f.m;
    const double* v = pools.hvec.data() + b.vec;
    const double* x = b.converged ? V::col(v, n, b.sol ? V::kXn : V::kX) : nullptr;
    const double* y = b.converged ? V::row(v, n, m, b.sol ? V::kYn : V::kY) : nullptr;
    b200pdlp_result* out = outs + src[k];
    hip_host_postsolve(lps[src[k]], f, b.L.cperm.data(), b.L.rperm.data(), x, y, V::col(v, n, V::kSp), V::col(v, n, V::kSn), out);
    hip_batch_result(out, b, loop, setup_seconds);
  });
  lap("batch", "postsolve (host threads)");
}

// ---- b200pdlp_debug_hipdlp_batch_prep_compare: the ordered members' device prologue and postsolve (batch_prep.cu
// hip_batch_*_kernel) against formulate_hipdlp + scale_hipdlp + build_layout and hip_host_postsolve
static void hipdlp_batch_prep_compare(int count, const b200pdlp_lp* lps, int scaling_mode, int ruiz_iterations, double* report) {
  using V = HipBatchVec;
  device_count_checked();
  RawLps raw(count, lps);
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
    const double* v = P.vec;
    rep[1] = dev_mismatches(V::col(v, n, V::kCost), f.cost.data(), n);
    rep[2] = dev_mismatches(V::col(v, n, V::kLower), f.lower.data(), n);
    rep[3] = dev_mismatches(V::col(v, n, V::kUpper), f.upper.data(), n);
    rep[4] = dev_mismatches(V::row(v, n, m, V::kRlo), f.rhs.data(), m);
    rep[5] = dev_mismatches(V::row(v, n, m, V::kRup), f.row_upper.data(), m);
    rep[6] = dev_mismatches(V::col(v, n, V::kColscale), f.col_scale.data(), n);
    rep[7] = dev_mismatches(V::row(v, n, m, V::kRowscale), f.row_scale.data(), m);
    rep[8] = dev_mismatches(P.row_new_idx, f.row_new_idx.data(), m);
    rep[9] = dev_mismatches(P.row_class, reinterpret_cast<const int*>(f.row_class.data()), m);
    sell_mismatches(L.A, P.a_slices, P.a_col, P.a_val, rep + 10);
    sell_mismatches(L.AT, P.at_slices, P.at_col, P.at_val, rep + 13);
    const double* r = D.rec.data() + (size_t)kPrepRec * i;
    const double got[2] = {std::sqrt(r[kRecCostSq]), std::sqrt(r[kRecRhsSq])};
    const double want[2] = {f.norm_cost, f.norm_rhs};
    for (int k = 0; k < 2; k++) rep[16 + k] = memcmp(got + k, want + k, sizeof(double)) != 0;
    rep[18] = scaled != f.scaled;
    for (int j = 0; j < n; j++) rep[19] += L.cperm[j] != j;   // the batch assumes identity orderings
    for (int q = 0; q < m; q++) rep[19] += L.rperm[q] != q;
  }
  // the postsolve of a probe iterate (x, y, sp, sn; a converged member at the iteration-0 check) into fresh device vectors
  std::vector<HipBatchPost> hpost;
  DevBuf<double> dout;
  probe_outputs(D, dout, hpost);
  std::vector<std::vector<double>> probes((size_t)count);
  for (int i = 0; i < count; i++) {
    const BatchPrep& P = D.hp[i];
    const int n = P.n, m = P.m;
    std::vector<double>& pr = probes[i];   // x, sp, sn (n each), y (m)
    pr.resize(3 * (size_t)n + m);
    for (size_t k = 0; k < pr.size(); k++) pr[k] = batch_probe(i, (int)k);
    double* v = P.vec;
    CUDA_OK(cudaMemcpy(V::col(v, n, V::kX), pr.data(), n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(V::col(v, n, V::kSp), pr.data() + n, n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(V::col(v, n, V::kSn), pr.data() + 2 * n, n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(V::row(v, n, m, V::kY), pr.data() + 3 * n, m * sizeof(double), cudaMemcpyHostToDevice));
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
    rep[20] = dev_mismatches(q.col_value, cv.data(), n0);
    rep[21] = dev_mismatches(q.col_dual, cd.data(), n0);
    rep[22] = dev_mismatches(q.row_value, rv.data(), m);
    rep[23] = dev_mismatches(q.row_dual, rdual.data(), m);
  }
}

// ----------------------------------------------------------------------- HiPDLP batch of LPs already on the GPU
// b200pdlp_solve_hipdlp_batch_device and _mixed_device: solve_hipdlp_batch for LPs whose arrays are device memory.  Every
// member's prologue and postsolve run on the device, one CTA per member: the ordered members' in batch_prep.cu, the tree
// members' (_mixed_device only) in batch_tree_prep.cu.  The rounds are hip_batch_rounds with the tree members on
// hip_tree_round_kernel.  The host reads fixed-size records per member, never an array.
// STATUS: runs on hardware; tests/test_gpu_hipdlp_batch_device.py, tests/test_gpu_hipdlp_batch_mixed_device.py,
// tools/batch_device_bench.py, tools/hipdlp_batch_mixed_device_bench.py (DESIGN.md section 6).

// The tree members' device prologue: the members' BatchPrep (from the sizing), HipBatchPrep, HipTreePrep and plans, and the
// pools behind them
struct TreeBatch {
  std::vector<BatchPrep> hp;
  std::vector<HipBatchPrep> hx;
  std::vector<HipTreePrep> ht;
  std::vector<HipTreePlan> plan;
  std::vector<double> rec;   // [count][kPrepRec]: rec[kRecCostSq], rec[kRecRhsSq]
  std::vector<size_t> scr;   // each member's offset in `scratch` (HipTreeMember::partials)
  DevBuf<BatchPrep> prep;
  DevBuf<HipBatchPrep> dhx;
  DevBuf<HipTreePrep> dht;
  DevBuf<HipTreePlan> dplan;
  DevBuf<double> drec;
  DevBuf<int> perms, ints, col, lcol;
  DevBuf<int4> desc, slices;
  DevBuf<double> dbls, vec, val, lval, scratch;
  DevBuf<HipSortRec> srt;
};

// the descriptor arrays of one matrix hold at most this many long rows and segments (a long row has > kTreeLongRow entries,
// a segment up to kNnzPerBlock)
static int tree_desc_cap(int nnz) { return nnz / kTreeLongRow + nnz / kNnzPerBlock + 1; }

// Orderings and plans of the tree members (hp: their descriptors from the sizing, lps their LPs; ids[k] names member k in
// messages): one read-back of a HipTreePlan per member
static void tree_batch_plan(cudaStream_t s, const std::vector<BatchPrep>& hp, const std::vector<BatchSize>& size,
                            const std::vector<int>& ids, const char* who, TreeBatch& T) {
  const int count = (int)hp.size();
  T.hp = hp;
  T.ht.assign((size_t)count, HipTreePrep{});
  size_t np = 0, nd = 0, ns = 0;
  for (int k = 0; k < count; k++) {
    const size_t n = size[k].n, m = hp[k].m;
    np += 2 * (n + m);
    nd += 4 * (size_t)tree_desc_cap(size[k].nnz);
    ns += (m + 31) / 32 + (n + 31) / 32;
  }
  T.perms.alloc(np, false); T.desc.alloc(nd, false); T.slices.alloc(ns, false);
  np = nd = ns = 0;
  for (int k = 0; k < count; k++) {
    const BatchSize& z = size[k];
    BatchPrep& P = T.hp[k];
    HipTreePrep& H = T.ht[k];
    const int n = z.n, m = P.m, cap = tree_desc_cap(z.nnz);
    P.n = n; P.nnz = z.nnz; P.neq = z.neq;
    H.rperm = T.perms.p + np; H.rinv = H.rperm + m; H.cperm = H.rinv + m; H.cinv = H.cperm + n;
    np += 2 * ((size_t)n + m);
    H.cap = cap;
    H.a_segs = T.desc.p + nd; H.a_long = H.a_segs + cap; H.at_segs = H.a_long + cap; H.at_long = H.at_segs + cap;
    nd += 4 * (size_t)cap;
    P.a_slices = T.slices.p + ns; ns += (m + 31) / 32;
    P.at_slices = T.slices.p + ns; ns += (n + 31) / 32;
  }
  T.prep.alloc(count, false); T.dht.alloc(count, false); T.dplan.alloc(count, false);
  CUDA_OK(cudaMemcpyAsync(T.prep.p, T.hp.data(), (size_t)count * sizeof(BatchPrep), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(T.dht.p, T.ht.data(), (size_t)count * sizeof(HipTreePrep), cudaMemcpyHostToDevice, s));
  launch_hip_tree_plan(s, count, T.prep.p, T.dht.p, T.dplan.p);
  CUDA_OK(cudaGetLastError());
  T.plan.resize((size_t)count);
  CUDA_OK(cudaMemcpyAsync(T.plan.data(), T.dplan.p, (size_t)count * sizeof(HipTreePlan), cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
  for (int k = 0; k < count; k++)
    if (T.plan[k].err)
      throw Error(B200PDLP_ERR_ARG, std::string(who) + ": member " + std::to_string(ids[k]) +
                                        ": b200pdlp: matrix too large for 32-bit slice offsets");
}

// The pools of the tree members after their plans, then their prologue (formulate_hipdlp, scale_hipdlp, the device-order
// vectors, the tree layouts) and one read-back of |c|^2, |b|^2 per member
static void tree_batch_prep(cudaStream_t s, int scaling_mode, int ruiz_iterations, TreeBatch& T) {
  const int count = (int)T.hp.size();
  size_t ni = 0, nd = 0, nv = 0, ne = 0, nl = 0, nsrt = 0, nscr = 0;
  T.scr.resize((size_t)count);
  for (int k = 0; k < count; k++) {
    const BatchPrep& P = T.hp[k];
    const HipTreePlan& Z = T.plan[k];
    const size_t n = P.n, m = P.m, nnz = P.nnz, n0 = P.n0;
    ni += 3 * nnz + n + m + 1 + (m + 1) + (nnz - n + n0) + n0;
    nd += nnz + 2 * n + m;
    nv += HipBatchVec::len(P.n, P.m);
    ne += (size_t)Z.pad_a + 32 + (size_t)Z.pad_at + 32;
    nl += (size_t)Z.lcount_a + (size_t)Z.lcount_at;
    nsrt += Z.maxcol > kTreeSortTile ? 2 * (size_t)Z.maxcol : 0;   // (each member sorts in its own scratch)
    T.scr[k] = nscr;
    nscr += 9 * (size_t)hip_tree_blocks(std::max(P.n, P.m)) + (size_t)Z.nseg_a + 2 * (size_t)Z.nseg_at;
  }
  T.ints.alloc(ni, false); T.dbls.alloc(nd, false); T.vec.alloc(nv, false);
  T.col.alloc(ne, false); T.val.alloc(ne, false); T.lcol.alloc(nl, false); T.lval.alloc(nl, false);
  T.scratch.alloc(nscr, false); T.srt.alloc(nsrt, false);
  CUDA_OK(cudaMemsetAsync(T.vec.p, 0, std::max<size_t>(nv, 1) * sizeof(double), s));   // the iterates and sums start at 0
  CUDA_OK(cudaMemsetAsync(T.lcol.p, 0, std::max<size_t>(nl, 1) * sizeof(int), s));       // fill_sell_host's zeroed lcol / lval
  CUDA_OK(cudaMemsetAsync(T.lval.p, 0, std::max<size_t>(nl, 1) * sizeof(double), s));
  T.hx.assign((size_t)count, HipBatchPrep{});
  ni = nd = nv = ne = nl = nsrt = 0;
  T.drec.alloc((size_t)count * kPrepRec, false);
  for (int k = 0; k < count; k++) {
    BatchPrep& P = T.hp[k];
    HipBatchPrep& X = T.hx[k];
    HipTreePrep& H = T.ht[k];
    const HipTreePlan& Z = T.plan[k];
    const int n = P.n, m = P.m, nnz = P.nnz, n0 = P.n0;
    int* q = T.ints.p + ni;
    P.cbeg = q; P.cidx = q + n + 1; P.pcol = P.cidx + nnz; P.rpos = P.pcol + nnz; P.rwork = P.rpos + nnz;
    ni += 3 * (size_t)nnz + n + m + 1;
    X.optr = T.ints.p + ni; X.opos = X.optr + m + 1; X.sortcols = X.opos + (nnz - n + n0);
    ni += (size_t)m + 1 + (nnz - n + n0) + n0;
    double* d = T.dbls.p + nd;
    P.cval = d; P.cs = d + nnz; P.cs_next = P.cs + n; P.rs = P.cs_next + n;
    nd += (size_t)nnz + 2 * (size_t)n + m;
    P.vec = T.vec.p + nv; nv += HipBatchVec::len(n, m);
    P.a_col = T.col.p + ne; P.a_val = T.val.p + ne; ne += (size_t)Z.pad_a + 32;
    P.at_col = T.col.p + ne; P.at_val = T.val.p + ne; ne += (size_t)Z.pad_at + 32;
    H.a_lcol = T.lcol.p + nl; H.a_lval = T.lval.p + nl; nl += (size_t)Z.lcount_a;
    H.at_lcol = T.lcol.p + nl; H.at_lval = T.lval.p + nl; nl += (size_t)Z.lcount_at;
    H.srt = T.srt.p + nsrt; nsrt += Z.maxcol > kTreeSortTile ? 2 * (size_t)Z.maxcol : 0;
    P.rec = T.drec.p + (size_t)kPrepRec * k;
  }
  T.dhx.alloc(count, false);
  CUDA_OK(cudaMemcpyAsync(T.prep.p, T.hp.data(), (size_t)count * sizeof(BatchPrep), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(T.dhx.p, T.hx.data(), (size_t)count * sizeof(HipBatchPrep), cudaMemcpyHostToDevice, s));
  CUDA_OK(cudaMemcpyAsync(T.dht.p, T.ht.data(), (size_t)count * sizeof(HipTreePrep), cudaMemcpyHostToDevice, s));
  launch_hip_tree_prep(s, count, T.prep.p, T.dhx.p, T.dht.p, T.dplan.p, scaling_mode, ruiz_iterations);
  CUDA_OK(cudaGetLastError());
  T.rec.assign((size_t)count * kPrepRec, 0.0);
  CUDA_OK(cudaMemcpy2DAsync(T.rec.data(), kPrepRec * sizeof(double), T.drec.p, kPrepRec * sizeof(double), 2 * sizeof(double),
                            count, cudaMemcpyDeviceToHost, s));
  CUDA_OK(cudaStreamSynchronize(s));
}

// member k's HipTreeMember (its vectors, layouts, long rows and scratch), for the rounds
static HipTreeMember tree_member(const TreeBatch& T, int k, const StdForm& f) {
  const BatchPrep& P = T.hp[k];
  const HipTreePrep& H = T.ht[k];
  const HipTreePlan& Z = T.plan[k];
  HipTreeMember M{};
  hip_batch_member(M.b, f, P.neq, P.vec);
  set_layouts(M.b, P.a_slices, P.a_col, P.a_val, P.at_slices, P.at_col, P.at_val);
  M.la.nsegs = Z.nseg_a; M.la.nlong = Z.nlong_a; M.la.segs = H.a_segs; M.la.long_rows = H.a_long;
  M.la.lcol = H.a_lcol; M.la.lval = H.a_lval;
  M.lat.nsegs = Z.nseg_at; M.lat.nlong = Z.nlong_at; M.lat.segs = H.at_segs; M.lat.long_rows = H.at_long;
  M.lat.lcol = H.at_lcol; M.lat.lval = H.at_lval;
  M.nb = hip_tree_blocks(std::max(P.n, P.m));
  M.partials = T.scratch.p + T.scr[k];
  M.a_part = M.partials + 9 * (size_t)M.nb;
  M.at_part[0] = M.a_part + Z.nseg_a;
  M.at_part[1] = M.at_part[0] + Z.nseg_at;
  return M;
}

// the scalars of a member's form after a device prologue (P: its descriptor, r: its record)
static void device_form(StdForm& f, const BatchPrep& P, const b200pdlp_lp& lp, const double* r, bool scaled) {
  f.hipdlp = true;
  f.n = P.n; f.m = P.m; f.nnz = P.nnz; f.neq = P.neq; f.n_orig = P.n0;
  f.sense = lp.sense; f.offset = lp.offset;
  f.norm_cost = std::sqrt(r[kRecCostSq]); f.norm_rhs = std::sqrt(r[kRecRhsSq]);
  f.scaled = scaled;
}

// `mixed`: a member past ordered_max is a tree member and the results take the blocks' trace rows; otherwise such a member
// is an error
void solve_hipdlp_batch_device(int count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params& prm,
                                      b200pdlp_result* outs, bool mixed) {
  using clk = std::chrono::steady_clock;
  const char* who = mixed ? "b200pdlp_solve_hipdlp_batch_mixed_device" : "b200pdlp_solve_hipdlp_batch_device";
  const std::string nvtx_name = mixed ? "b200pdlp: HiPDLP mixed batch " : "b200pdlp: HiPDLP batch ";
  const auto t_begin = clk::now();
  Laps lap;
  const int device = select_device(prm.device);
  check_device_arrays(count, lps, nullptr, outs, device, who);
  StreamHolder sh;
  cudaStream_t s = sh.s;
  PrepMode mode;
  mode.hip = true; mode.scaling = prm.scaling_mode; mode.ruiz_iterations = prm.ruiz_iterations;
  DeviceBatch D;   // every member's sizing
  std::vector<int> src;   // device member k is the caller's member src[k]: the ordered members, then the tree members
  int ntree = 0;
  {
    NvtxRange nvtx((nvtx_name + "validation + sizing (device)").c_str());
    device_batch_size(s, count, lps, nullptr, mode, D);
    const int omax = prm.ordered_max == 0 ? 4096 : prm.ordered_max;
    std::vector<int> tree;
    for (int i = 0; i < count; i++) {   // the lowest failing member
      const BatchSize& z = D.size[i];
      const std::string at = std::string(who) + ": member " + std::to_string(i) + ": ";
      if (z.err != kPrepOk) throw Error(B200PDLP_ERR_ARG, at + prep_error_text(z.err));
      const int m = lps[i].num_row, big = std::max(z.n, m);
      if (omax < 0 || big > omax) {   // (a tree member's pad_a / pad_at, the ordered layout's padding, mean nothing)
        if (!mixed)
          throw Error(B200PDLP_ERR_ARG, at + "standard form " + std::to_string(m) + " x " + std::to_string(z.n) +
                                            " exceeds ordered_max = " + std::to_string(omax));
        if (big > kTreeMemberMax)
          throw Error(B200PDLP_ERR_ARG, at + "standard form " + std::to_string(m) + " x " + std::to_string(z.n) +
                                            " exceeds max(n, m) = " + std::to_string(kTreeMemberMax) +
                                            " of a tree member: solve it with b200pdlp_solve_hipdlp");
        tree.push_back(i);
      } else {
        if (z.pad_a >= 2000000000 || z.pad_at >= 2000000000)
          throw Error(B200PDLP_ERR_ARG, at + "b200pdlp: matrix too large for 32-bit slice offsets");
        src.push_back(i);
      }
    }
    ntree = (int)tree.size();
    src.insert(src.end(), tree.begin(), tree.end());
  }
  const int nord = count - ntree;
  lap("batch device", "validation + sizing");
  auto group = [&](int k0, int k1, std::vector<BatchPrep>& hp, std::vector<BatchSize>& sz, std::vector<b200pdlp_lp>& gl,
                   std::vector<int>& ids) {
    for (int k = k0; k < k1; k++) {
      hp.push_back(D.hp[src[k]]); sz.push_back(D.size[src[k]]); gl.push_back(lps[src[k]]); ids.push_back(src[k]);
    }
  };
  DeviceBatch O;   // the ordered members' prologue (their row maps stay in D's pools)
  std::vector<b200pdlp_lp> olps, tlps;
  std::vector<int> oids, tids;
  group(0, nord, O.hp, O.size, olps, oids);
  TreeBatch T;
  if (mixed) {
    NvtxRange nvtx("b200pdlp: HiPDLP mixed batch orderings + plans (device)");
    std::vector<BatchPrep> thp;
    std::vector<BatchSize> tsz;
    group(nord, count, thp, tsz, tlps, tids);
    if (ntree > 0) tree_batch_plan(s, thp, tsz, tids, who, T);
    lap("batch device", "orderings + plans");
  }
  {
    NvtxRange nvtx((nvtx_name + "prologue (device)").c_str());
    if (nord > 0) device_batch_prep(s, nord, olps.data(), mode, O);
    if (ntree > 0) tree_batch_prep(s, prm.scaling_mode, prm.ruiz_iterations, T);
  }
  lap("batch device", "prologue (device)");

  const bool scaled = (prm.scaling_mode & 7) != 0;   // scale_hipdlp: any of its passes is switched on
  std::vector<HipBatchRun> runs((size_t)count);
  std::vector<HipBatchRun*> R((size_t)count);
  std::vector<HipBatchMember> hmem((size_t)nord);
  std::vector<HipTreeMember> htree((size_t)ntree);
  for (int k = 0; k < count; k++) {
    HipBatchRun& b = runs[k];
    R[k] = &b;
    if (mixed) { b.trace = outs + src[k]; b.trace->trace_len = 0; }
    if (k < nord) {
      const BatchPrep& P = O.hp[k];
      device_form(b.f, P, lps[src[k]], O.rec.data() + (size_t)kPrepRec * k, scaled);
      hip_batch_member(hmem[k], b.f, P.neq, P.vec);
      set_layouts(hmem[k], P.a_slices, P.a_col, P.a_val, P.at_slices, P.at_col, P.at_val);
    } else {
      const int t = k - nord;
      device_form(b.f, T.hp[t], lps[src[k]], T.rec.data() + (size_t)kPrepRec * t, scaled);
      htree[t] = tree_member(T, t, b.f);
    }
  }
  DevBuf<HipBatchMember> dmem;
  DevBuf<HipTreeMember> dtree;
  dmem.alloc(nord, false); dtree.alloc(ntree, false);
  if (nord > 0) CUDA_OK(cudaMemcpyAsync(dmem.p, hmem.data(), (size_t)nord * sizeof(HipBatchMember), cudaMemcpyHostToDevice, s));
  if (ntree > 0) CUDA_OK(cudaMemcpyAsync(dtree.p, htree.data(), (size_t)ntree * sizeof(HipTreeMember), cudaMemcpyHostToDevice, s));
  const int cluster = ntree > 0 ? tree_cluster(ntree) : 1;
  if (lap.on && ntree > 0) fprintf(stderr, "[b200pdlp batch] tree members %d, cluster of C = %d CTAs each\n", ntree, cluster);
  const BatchLoop loop = hip_batch_rounds(s, count, prm, dmem.p, R, dtree.p, ntree, cluster);
  lap("batch device", "rounds");

  // ---- the postsolve of every member on the device, into the caller's vectors
  NvtxRange nvtx_post((nvtx_name + "postsolve (device)").c_str());
  std::vector<HipBatchPost> hpost((size_t)count);
  for (int k = 0; k < count; k++) {
    HipBatchPost& q = hpost[k];
    const b200pdlp_result& o = outs[src[k]];
    q.col_value = o.col_value; q.col_dual = o.col_dual; q.row_value = o.row_value; q.row_dual = o.row_dual;
    q.sol = runs[k].converged ? runs[k].sol : -1;
    q.pad = 0;
  }
  DevBuf<HipBatchPost> dpost;
  dpost.alloc(count, false);
  CUDA_OK(cudaMemcpyAsync(dpost.p, hpost.data(), (size_t)count * sizeof(HipBatchPost), cudaMemcpyHostToDevice, s));
  if (nord > 0) launch_hip_batch_post(s, nord, O.prep.p, O.dhx.p, dpost.p, scaled ? 1 : 0);
  if (ntree > 0) launch_hip_tree_post(s, ntree, T.prep.p, T.dhx.p, T.dht.p, dpost.p + nord, scaled ? 1 : 0);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaStreamSynchronize(s));
  const double setup_seconds = std::chrono::duration<double>(loop.t_loop - t_begin).count();
  for (int k = 0; k < count; k++) hip_batch_result(outs + src[k], runs[k], loop, setup_seconds);
  lap("batch device", "postsolve (device)");
}

// ---- b200pdlp_debug_hipdlp_tree_prep_compare: the tree members' device prologue and postsolve against
// formulate_hipdlp + scale_hipdlp + build_layout(ordered_max = -1) and hip_host_postsolve
static const int kHipTreePrepItems = 31;

// one matrix's long rows (descriptors, entries) from the device against the host's: r[0..3] (all -1 when the counts differ)
static void long_mismatches(const SellMatrix& H, int nseg, int nlong, long long lcount, const int4* segs, const int4* longs,
                            const int* lcol, const double* lval, double* r) {
  if (nseg != (int)H.segs.size() || nlong != (int)H.long_rows.size() || lcount != H.lcount) {
    r[0] = r[1] = r[2] = r[3] = -1.0;
    return;
  }
  r[0] = dev_mismatches(segs, reinterpret_cast<const int4*>(H.segs.data()), H.segs.size());
  r[1] = dev_mismatches(longs, reinterpret_cast<const int4*>(H.long_rows.data()), H.long_rows.size());
  r[2] = dev_mismatches(lcol, H.lcol.data(), H.lcol.size());
  r[3] = dev_mismatches(lval, H.lval.data(), H.lval.size());
}

static void hipdlp_tree_prep_compare(int count, const b200pdlp_lp* lps, int scaling_mode, int ruiz_iterations, double* report) {
  using V = HipBatchVec;
  const char* who = "b200pdlp_debug_hipdlp_tree_prep_compare";
  device_count_checked();
  RawLps raw(count, lps);
  StreamHolder sh;
  DeviceBatch D;
  PrepMode mode;
  mode.hip = true;
  device_batch_size(sh.s, count, raw.dl.data(), nullptr, mode, D);
  std::vector<int> ids((size_t)count);
  for (int i = 0; i < count; i++) {
    const BatchSize& z = D.size[i];
    if (z.err != kPrepOk) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": member " + std::to_string(i) + ": " + prep_error_text(z.err));
    if (std::max(z.n, lps[i].num_row) > kTreeMemberMax)
      throw Error(B200PDLP_ERR_ARG, std::string(who) + ": member " + std::to_string(i) + ": exceeds max(n, m) = " +
                                        std::to_string(kTreeMemberMax) + " of a tree member");
    ids[i] = i;
  }
  TreeBatch T;
  tree_batch_plan(sh.s, D.hp, D.size, ids, who, T);
  tree_batch_prep(sh.s, scaling_mode, ruiz_iterations, T);
  const bool scaled = (scaling_mode & 7) != 0;
  std::vector<StdForm> F((size_t)count);
  std::vector<HostLayout> Ls((size_t)count);
  for (int i = 0; i < count; i++) {
    const BatchPrep& P = T.hp[i];
    const HipTreePrep& H = T.ht[i];
    const HipTreePlan& Z = T.plan[i];
    StdForm& f = F[i];
    HostLayout& L = Ls[i];
    formulate_hipdlp(lps[i], f);
    scale_hipdlp(f, scaling_mode, ruiz_iterations);
    build_layout(f, 0, 1, -1, L);
    double* rep = report + (size_t)kHipTreePrepItems * i;
    for (int k = 0; k < kHipTreePrepItems; k++) rep[k] = 0.0;
    rep[0] = (P.n != f.n) + (P.m != f.m) + (P.nnz != f.nnz) + (P.neq != f.neq) + L.ordered;
    if (rep[0] != 0.0) {   // nothing else lines up
      for (int k = 1; k < kHipTreePrepItems; k++) rep[k] = -1.0;
      continue;
    }
    const int n = f.n, m = f.m;
    const double* v = P.vec;
    auto by_col = [&](const std::vector<double>& x) { std::vector<double> o(n); for (int k = 0; k < n; k++) o[k] = x[L.cperm[k]]; return o; };
    auto by_row = [&](const std::vector<double>& x) { std::vector<double> o(m); for (int k = 0; k < m; k++) o[k] = x[L.rperm[k]]; return o; };
    rep[1] = dev_mismatches(V::col(v, n, V::kCost), by_col(f.cost).data(), n);
    rep[2] = dev_mismatches(V::col(v, n, V::kLower), by_col(f.lower).data(), n);
    rep[3] = dev_mismatches(V::col(v, n, V::kUpper), by_col(f.upper).data(), n);
    rep[4] = dev_mismatches(V::row(v, n, m, V::kRlo), by_row(f.rhs).data(), m);
    rep[5] = dev_mismatches(V::row(v, n, m, V::kRup), by_row(f.row_upper).data(), m);
    rep[6] = dev_mismatches(V::col(v, n, V::kColscale), by_col(f.col_scale).data(), n);
    rep[7] = dev_mismatches(V::row(v, n, m, V::kRowscale), by_row(f.row_scale).data(), m);
    rep[8] = dev_mismatches(H.rperm, L.rperm.data(), m);
    rep[9] = dev_mismatches(H.cperm, L.cperm.data(), n);
    sell_mismatches(L.A, P.a_slices, P.a_col, P.a_val, rep + 10);
    sell_mismatches(L.AT, P.at_slices, P.at_col, P.at_val, rep + 13);
    long_mismatches(L.A, Z.nseg_a, Z.nlong_a, Z.lcount_a, H.a_segs, H.a_long, H.a_lcol, H.a_lval, rep + 16);
    long_mismatches(L.AT, Z.nseg_at, Z.nlong_at, Z.lcount_at, H.at_segs, H.at_long, H.at_lcol, H.at_lval, rep + 20);
    const double* r = T.rec.data() + (size_t)kPrepRec * i;
    const double got[2] = {std::sqrt(r[kRecCostSq]), std::sqrt(r[kRecRhsSq])};
    const double want[2] = {f.norm_cost, f.norm_rhs};
    for (int k = 0; k < 2; k++) rep[24 + k] = memcmp(got + k, want + k, sizeof(double)) != 0;
    rep[26] = scaled != f.scaled;
  }
  // the postsolve of a probe iterate (x, y, sp, sn in device order; a converged member at the iteration-0 check)
  std::vector<HipBatchPost> hpost;
  DevBuf<double> dout;
  DeviceBatch shape;   // probe_outputs reads the dimensions only
  shape.hp = T.hp;
  probe_outputs(shape, dout, hpost);
  std::vector<std::vector<double>> probes((size_t)count);
  for (int i = 0; i < count; i++) {
    const BatchPrep& P = T.hp[i];
    const int n = P.n, m = P.m;
    std::vector<double>& pr = probes[i];   // x, sp, sn (n each), y (m)
    pr.resize(3 * (size_t)n + m);
    for (size_t k = 0; k < pr.size(); k++) pr[k] = batch_probe(i, (int)k);
    double* v = P.vec;
    CUDA_OK(cudaMemcpy(V::col(v, n, V::kX), pr.data(), n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(V::col(v, n, V::kSp), pr.data() + n, n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(V::col(v, n, V::kSn), pr.data() + 2 * n, n * sizeof(double), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(V::row(v, n, m, V::kY), pr.data() + 3 * n, m * sizeof(double), cudaMemcpyHostToDevice));
  }
  DevBuf<HipBatchPost> dpost;
  dpost.alloc(count, false);
  dpost.upload(hpost.data(), count);
  launch_hip_tree_post(sh.s, count, T.prep.p, T.dhx.p, T.dht.p, dpost.p, scaled ? 1 : 0);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaStreamSynchronize(sh.s));
  for (int i = 0; i < count; i++) {
    double* rep = report + (size_t)kHipTreePrepItems * i;
    if (rep[0] != 0.0) continue;
    const StdForm& f = F[i];
    const HostLayout& L = Ls[i];
    const int n = f.n, m = f.m, n0 = f.n_orig;
    const double* pr = probes[i].data();
    std::vector<double> cv(std::max(n0, 1)), cd(std::max(n0, 1)), rv(std::max(m, 1)), rdual(std::max(m, 1));
    b200pdlp_result res{};
    res.col_value = cv.data(); res.col_dual = cd.data(); res.row_value = rv.data(); res.row_dual = rdual.data();
    hip_host_postsolve(lps[i], f, L.cperm.data(), L.rperm.data(), pr, pr + 3 * n, pr + n, pr + 2 * n, &res);
    const HipBatchPost& q = hpost[i];
    rep[27] = dev_mismatches(q.col_value, cv.data(), n0);
    rep[28] = dev_mismatches(q.col_dual, cd.data(), n0);
    rep[29] = dev_mismatches(q.row_value, rv.data(), m);
    rep[30] = dev_mismatches(q.row_dual, rdual.data(), m);
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
  const int dev = select_device(device);
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
      const b200pdlp_solution& x = sols[i];
      check_device_lp(lps[i], dev, i, who);
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

// The four batch solves' entry: the caller's device restored on return, count < 0 an error, count == 0 nothing to do, and
// no NULL argument (args_ok); then solve(), and any CUDA error it left behind
template <class F>
static int batch_entry(const char* who, int count, bool args_ok, F&& solve) {
  DeviceGuard dg;
  return guarded([&] {
    if (count < 0) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": count < 0");
    if (count == 0) return;
    if (!args_ok) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": null argument");
    solve();
    CUDA_OK(cudaGetLastError());
  });
}

// The three prologue comparisons' entry: the caller's device restored on return, count >= 0, no NULL argument and every LP
// well-formed (check_lp), then compare() when there is a member
template <class F>
static int prep_compare_entry(const char* who, int count, const b200pdlp_lp* lps, const double* report, F&& compare) {
  DeviceGuard dg;
  return guarded([&] {
    if (count < 0 || (count > 0 && (!lps || !report))) throw Error(B200PDLP_ERR_ARG, std::string(who) + ": bad arguments");
    for (int i = 0; i < count; i++) check_lp(&lps[i]);
    if (count > 0) compare();
  });
}

}  // namespace b200

extern "C" {

int b200pdlp_solve_batch(int32_t count, const b200pdlp_lp* lps, const b200pdlp_params* params, const b200pdlp_warm* warms,
                         b200pdlp_result* outs) {
  const char* who = "b200pdlp_solve_batch";
  return batch_entry(who, count, lps && params && outs, [&] {
    check_params(*params);
    for (int i = 0; i < count; i++) check_ordered_member(&lps[i], params->ordered_max, 1e20, i, who);
    solve_batch(count, lps, *params, warms, outs);
  });
}

int b200pdlp_solve_batch_device(int32_t count, const b200pdlp_lp* lps, const b200pdlp_params* params, const b200pdlp_warm* warms,
                                b200pdlp_result* outs) {
  const char* who = "b200pdlp_solve_batch_device";
  return batch_entry(who, count, lps && params && outs, [&] {
    check_params(*params);
    for (int i = 0; i < count; i++) check_batch_device_member(&lps[i], params->ordered_max, i, who);
    solve_batch_device(count, lps, *params, warms, outs);
  });
}

int b200pdlp_debug_batch_prep_compare(int32_t count, const b200pdlp_lp* lps, int32_t scaling, double* report) {
  return prep_compare_entry("b200pdlp_debug_batch_prep_compare", count, lps, report,
                            [&] { batch_prep_compare(count, lps, scaling, report); });
}

int b200pdlp_solve_hipdlp_batch(int32_t count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params* params,
                                b200pdlp_result* outs) {
  const char* who = "b200pdlp_solve_hipdlp_batch";
  return batch_entry(who, count, lps && params && outs, [&] {
    for (int i = 0; i < count; i++)
      check_ordered_member(&lps[i], params->ordered_max, std::numeric_limits<double>::infinity(), i, who);
    std::vector<int> src((size_t)count);
    for (int i = 0; i < count; i++) src[i] = i;
    solve_hipdlp_batch(count, lps, *params, outs, src, 0, false);
  });
}

int b200pdlp_solve_hipdlp_batch_mixed(int32_t count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params* params,
                                      b200pdlp_result* outs) {
  const char* who = "b200pdlp_solve_hipdlp_batch_mixed";
  return batch_entry(who, count, lps && params && outs, [&] {
    std::vector<int> src, tree;   // the ordered members first, then the tree members, each group in the caller's order
    for (int i = 0; i < count; i++) (check_mixed_member(&lps[i], params->ordered_max, i, who) ? tree : src).push_back(i);
    const int ntree = (int)tree.size();
    src.insert(src.end(), tree.begin(), tree.end());
    solve_hipdlp_batch(count, lps, *params, outs, src, ntree, true);
  });
}

int b200pdlp_solve_hipdlp_batch_device(int32_t count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params* params,
                                       b200pdlp_result* outs) {
  const char* who = "b200pdlp_solve_hipdlp_batch_device";
  return batch_entry(who, count, lps && params && outs, [&] {
    for (int i = 0; i < count; i++) check_batch_device_member(&lps[i], params->ordered_max, i, who);
    solve_hipdlp_batch_device(count, lps, *params, outs, false);
  });
}

int b200pdlp_solve_hipdlp_batch_mixed_device(int32_t count, const b200pdlp_lp* lps, const b200pdlp_hipdlp_params* params,
                                             b200pdlp_result* outs) {
  const char* who = "b200pdlp_solve_hipdlp_batch_mixed_device";
  return batch_entry(who, count, lps && params && outs, [&] {
    for (int i = 0; i < count; i++) check_batch_device_member(&lps[i], 0, i, who);   // (any ordered_max: tree members)
    solve_hipdlp_batch_device(count, lps, *params, outs, true);
  });
}

int b200pdlp_debug_hipdlp_tree_prep_compare(int32_t count, const b200pdlp_lp* lps, int32_t scaling_mode, int32_t ruiz_iterations,
                                            double* report) {
  return prep_compare_entry("b200pdlp_debug_hipdlp_tree_prep_compare", count, lps, report,
                            [&] { hipdlp_tree_prep_compare(count, lps, scaling_mode, ruiz_iterations, report); });
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
  return prep_compare_entry("b200pdlp_debug_hipdlp_batch_prep_compare", count, lps, report,
                            [&] { hipdlp_batch_prep_compare(count, lps, scaling_mode, ruiz_iterations, report); });
}

}  // extern "C"
