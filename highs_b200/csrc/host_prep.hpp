// highs_b200/csrc/host_prep.hpp -- host-side preparation of the PDLP standard form.
//
// Product code (C++), no CUDA.  Replaces, for the CUDA engine, what the reference
// does on the host before its solver starts:
//   formulateLP_highs            /root/reference/highs/pdlp/CupdlpWrapper.cpp:280-448
//   Init_Scaling/PDHG_Scale_Data highs/pdlp/cupdlp/cupdlp_scaling.c:233-425
//   csc2csr                      highs/pdlp/cupdlp/cupdlp_utils.c:1222-1254
// and then builds the row-blocked layouts the SpMV kernels stream.
#pragma once
#include <cstdint>
#include <functional>
#include <memory>
#include <utility>
#include <vector>

#include "../../include/b200pdlp.h"

namespace b200 {

// std::vector whose resize() leaves new elements uninitialised: the big arrays of the prologue are written exactly
// once by the threads that fill them, so the pages are first touched in parallel (and on the writer's NUMA node)
// instead of being zero-filled by one thread beforehand.
template <class T>
struct DefaultInitAlloc : std::allocator<T> {
  template <class U> struct rebind { using other = DefaultInitAlloc<U>; };
  DefaultInitAlloc() = default;
  template <class U> DefaultInitAlloc(const DefaultInitAlloc<U>&) {}
  template <class U> void construct(U* p) { ::new (static_cast<void*>(p)) U; }
  template <class U, class... A> void construct(U* p, A&&... a) { ::new (static_cast<void*>(p)) U(std::forward<A>(a)...); }
};
template <class T> using RawVec = std::vector<T, DefaultInitAlloc<T>>;

enum RowClass : int { kEq = 0, kLeq = 1, kGeq = 2, kBound = 3, kFreeRow = 4 };  // cupdlp_defs.h numbering (+ HiPDLP's FREE)

// min c'x  s.t.  A x = b (rows < neq),  A x >= b (rows >= neq),  l <= x <= u
struct StdForm {
  int n = 0, m = 0, nnz = 0, neq = 0, n_orig = 0;
  std::vector<double> cost, lower, upper, rhs;
  std::vector<int> cbeg;         // column-wise copy (scaled in place)
  RawVec<int> cidx;
  RawVec<double> cval;
  std::vector<double> col_scale, row_scale;
  std::vector<int> row_new_idx, row_class;  // by ORIGINAL row
  double sense = 1.0, offset = 0.0;
  double norm_cost = 0.0, norm_rhs = 0.0;   // 2-norms of the unscaled cost / rhs
  double amax = 0.0;                        // max |a_ij| after scaling
  // HiPDLP mode (host_prep_hipdlp.cpp): rows carry an upper bound as well (rhs = lower), `scaled` = any scaling applied
  bool hipdlp = false, scaled = false;
  std::vector<double> row_upper;
  // row-major index of the nonzeros (built once, by scale() or on demand): row i owns positions
  // rpos[rptr[i] .. rptr[i+1]) of cidx/cval, columns ascending
  std::vector<int> rptr;
  RawVec<int> rpos, rcol;   // rcol[q] = column of position rpos[q]
};

// plain row-major matrix (CSR); entries of a row keep the order the reference's scatter SpMV adds them in
struct Csr {
  int nrows = 0, ncols = 0, nnz = 0;
  std::vector<int> rowptr;
  RawVec<int> col;
  RawVec<double> val;
};

// Device layout of one matrix: sliced ELL body + split long rows.
//  * body: rows (in `perm` order) are grouped in slices of 32; slice s stores its entries k-major /
//    lane-minor (element (k, lane) at ptr + 32 k + lane), padded with (col 0, val 0) to the longest
//    row of the slice, so a warp reads col/val fully coalesced and each lane accumulates ITS row in
//    registers, in the row's own entry order.  Rows are sorted by length inside windows of
//    kSortWindow rows (never across the equality / inequality boundary) to keep the padding small.
//  * rows longer than `long_threshold` are left out of the body (their lanes are masked) and cut into
//    segments of kNnzPerBlock nonzeros; the last segment CTA to finish combines the partial sums.
struct SellMatrix {
  int nrows = 0, ncols = 0;
  long long nnz = 0, padded = 0;
  struct Slice { int ptr, len; unsigned skipmask; int pad; };
  std::vector<Slice> slices;
  RawVec<int> col;
  RawVec<double> val;
  struct Seg { int row, nnz_begin, nnz_end, long_id; };
  struct LongRow { int row, first_seg, nseg, partial_offset; };
  std::vector<Seg> segs;
  std::vector<LongRow> long_rows;
  std::vector<int> lcol;
  std::vector<double> lval;
  int n_partials = 0;
  long long lcount = 0;      // entries of lcol / lval (rows padded to multiples of 4, + 8)
};

constexpr int kNnzPerBlock = 2048;   // long-row segment size (== kernels.cuh kNnzBlk)
constexpr int kSortWindow = 8192;

void formulate(const b200pdlp_lp& lp, StdForm& f);
// HiPDLP's own prologue (pdhg.cc:152-358, scaling.cc, pdhg.cc:1529-1671): scaling_mode bits 1 Ruiz, 4 PC, 2 L2
void formulate_hipdlp(const b200pdlp_lp& lp, StdForm& f);
void scale_hipdlp(StdForm& f, int scaling_mode, int ruiz_iterations);
double power_method_hipdlp(const StdForm& f);
// Host control of the HiPDLP loop between blocks of 40 Halpern steps (PDLPSolver::solve, hipdlp/pdhg.cc:494-707):
// step sizes from the power method, fixed-point error, convergence test, restart criteria and the PID primal weight.
// The device (or, in the CPU tests, the oracle's trace) supplies nine sums per check:
//   s[0] |x_next - refl_x|^2  s[1] |y_next - refl_y|^2  s[2] (x_next - refl_x).A'(y_next - refl_y)
//   s[3] |primal residual|^2  s[4] |dual residual|^2    s[5] primal objective   s[6] dual objective
//   s[7] |x_next - x_anchor|^2  s[8] |y_next - y_anchor|^2
struct HipController {
  double tol = 1e-7, norm_cost = 0.0, norm_rhs = 0.0, eta = 0.0;
  int strategy = 3;                        // 0: fixed primal weight, otherwise PID
  double omega = 1.0, primal_weight = 1.0, best_primal_weight = 1.0, best_gap = 0.0, err_sum = 0.0, last_err = 0.0;
  double primal_step = 0.0, dual_step = 0.0;
  int iters = 0, halpern_iteration = 0, restarts = 0;
  bool pending_restart_fpe = false;        // the next block's first step defines the restart's reference error
  double fpe = 0.0, fpe0 = 0.0, last_trial = 0.0;
  double pfeas = 0.0, dfeas = 0.0, pobj = 0.0, dobj = 0.0, relgap = 0.0;
  void init(double norm_cost_, double norm_rhs_, double op_norm_sq, double tol_, int strategy_);   // initializeStepSizes, :1944-1977
  double fixed_point_error(const double* s) const;                                                 // :733-739
  bool converged(const double* s);                                                                 // checkConvergence, :1474-1527
  // the convergence test on the measures of the last check (converged() sets them, and so does after_block())
  bool block_converged() const { return pfeas < tol * (1.0 + norm_rhs) && dfeas < tol * (1.0 + norm_cost) && relgap < tol; }
  void restart_reference(const double* s) { fpe = fixed_point_error(s); fpe0 = fpe; pending_restart_fpe = false; }   // :600-608
  // after steps 2..40 of a block (s = the block-end check); returns true if the loop restarts now (anchors <- iterate),
  // with the primal weight and the step sizes already updated
  bool after_block(const double* s);
};
void build_row_index(StdForm& f);   // fills f.rptr / f.rpos (parallel counting sort)
// fn(chunk_index, begin, end) over [0, count) cut into contiguous chunks, one per host thread of the persistent pool
void parallel_chunks(long long count, const std::function<void(int, long long, long long)>& fn, long long min_per_thread = 1 << 15);
void scale(StdForm& f, bool do_scale);
// nnz-balanced contiguous partition of the m rows into `world` parts
std::vector<int> partition_rows(const StdForm& f, int world);
// rows [r0,r1) of A, row-major (columns ascending within a row)
void build_row_major(const StdForm& f, int r0, int r1, Csr& a);
// transpose of rows [r0,r1): n rows, (r1-r0) columns, local row ids ascending
void build_col_major(const StdForm& f, int r0, int r1, Csr& at);
// new -> old ordering of `count` rows: identity, or (sort) by descending length inside windows that
// do not straddle `boundary`
std::vector<int> make_perm(const std::vector<int>& rowptr, int boundary, bool sort);
std::vector<int> invert_perm(const std::vector<int>& perm);
// rows of `a` taken in `perm` order, column ids mapped through `colmap` (old -> new)
void build_sell(const Csr& a, const std::vector<int>& perm, const std::vector<int>& colmap, int long_threshold,
                SellMatrix& out);
// the two halves of build_sell: the plan (descriptors only; needs nothing but the row lengths) and the host fill
void plan_sell(int nrows, int ncols, long long nnz, const std::vector<int>& perm, const std::function<int(int)>& old_row_len,
               int long_threshold, SellMatrix& out);
void fill_sell_host(const Csr& a, const std::vector<int>& perm, const std::vector<int>& colmap, SellMatrix& out);

// Everything the device needs to know about one rank's share of the matrix (host side of
// b200pdlp_problem_create; also what b200pdlp_form_layout_eval evaluates without a GPU).
//  * rank g of `world` owns rows [r0, r1) (partition_rows) and, when world > 1, the device columns
//    [c0, c0 + nl_real); n-vectors are held in segments of shard_len entries, full vectors in `world`
//    segments of seg_len = shard_len + 2 doubles (the tail carries the pass's scalar sums);
//  * ordered (single GPU, max(m, n) <= ordered_max): rows/columns keep the reference's order and no row is
//    split, so that every sum can run in the reference's order; otherwise they are sorted by length in windows.
struct HostLayout {
  int rank = 0, world = 1;
  int r0 = 0, r1 = 0, ml = 0, neq_local = 0;
  std::vector<int> bounds;        // row offsets of every rank's block (world + 1 entries)
  bool ordered = false;
  Csr csr_local;                  // rows [r0, r1) in standard-form order
  std::vector<int> rperm, rinv;   // device row order: rperm[new] = old local row
  std::vector<int> cperm, cinv;   // device column order: cperm[new] = old column (same on every rank)
  int nl = 0, nl_real = 0, c0 = 0, shard_len = 0, seg_len = 0;
  SellMatrix A, AT;               // A_g (rows = local device rows; columns = positions in the segmented x)
                                  // A_g^T (rows = device columns in AT order; columns = local device rows)
  std::vector<int> at_outpos;     // world > 1: A_g^T body row -> position in the segmented partial vector
  // position of device column j in a segmented full vector
  size_t seg_pos(int j) const { return world == 1 ? (size_t)j : (size_t)(j / shard_len) * seg_len + (size_t)(j % shard_len); }
};
// `lap`, if given, is called with a stage name after every stage (timing hook)
// plan_only (world == 1): only the orderings and the sliced-ELL PLANS (A.col/val and csr_local stay empty) -- the
// arrays are then filled on the device from the scaled matrix resident there
void build_layout(StdForm& f, int rank, int world, int ordered_max, HostLayout& L,
                  const std::function<void(const char*)>& lap = nullptr, bool plan_only = false);
// HiPDLP on several GPUs: the ONE-GPU device orders (build_layout(f, 0, 1, ...): rperm / cperm, ordered or tree mode
// decided on the whole problem) cut into `world` contiguous, nnz-balanced blocks.  Rank g computes whole rows: device
// rows [rb[g], rb[g+1]) of A and device columns [cb[g], cb[g+1]) of A (rows of A'), each in the one-GPU entry order, so
// every value it produces has the one-GPU bits.  A rank may own no rows or no columns.
struct HipShards {
  int world = 1;
  bool ordered = false;
  int long_threshold = 512;
  Csr a, at;                                  // the whole matrix, row-major and column-major (standard-form order)
  std::vector<int> rperm, rinv, cperm, cinv;  // the one-GPU device orders
  std::vector<int> rb, cb;                    // world + 1 block offsets in device row / column order
};
void plan_hipdlp_shards(StdForm& f, int world, int ordered_max, HipShards& S);
// rank g's matrices: A_g (rows = device rows [rb[g], rb[g+1]); column ids = device column positions 0..n-1) and
// A_g' (rows = device columns [cb[g], cb[g+1]); column ids = device row positions 0..m-1)
void build_hipdlp_shard(const HipShards& S, int rank, SellMatrix& A, SellMatrix& AT);
// host evaluation of a sliced-ELL matrix exactly as the kernels traverse it (body: lane = row, k ascending;
// long rows: per-segment partial sums, added in segment order): out[row] for row < nrows
void sell_apply_host(const SellMatrix& a, const double* xin, double* out);

}  // namespace b200
