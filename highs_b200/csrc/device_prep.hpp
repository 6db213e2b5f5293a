// highs_b200/csrc/device_prep.hpp -- the whole prologue of a solve on the device (one GPU, tree mode).
//
// What the reference does on the host before its first iteration -- formulateLP_highs
// (/root/reference/highs/pdlp/CupdlpWrapper.cpp:280-448), Init_Scaling + PDHG_Scale_Data
// (highs/pdlp/cupdlp/cupdlp_scaling.c:233-425), csc2csr (cupdlp_utils.c:1222-1254) -- and what host_prep.cpp does for
// the engine on host threads (its tested twin: same arithmetic, same orders), here as kernels over the caller's
// HighsLp arrays, copied once to HBM or (inputs_on_device) read where they are.  The host touches O(1) data: three small read-backs (sizes of the standard form,
// sizes of the layouts + scalars, long-row totals; block mode adds the partition's 2 (world + 1) offsets).  Scans, stable radix sorts and the stream compaction come from CUB
// (part of the CUDA toolkit); everything that computes is a kernel of device_prep.cu / setup_kernels.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../include/b200pdlp.h"
#include "kernels.cuh"

namespace b200 {

// Process-wide cache of device blocks: a solve allocates ~60 buffers and frees them a few milliseconds later; cudaMalloc /
// cudaFree (which also synchronises the device) would cost more than the prologue itself.  Blocks go back to the cache,
// not to the driver (whole cudaMalloc blocks, never sub-allocations, so CUDA-IPC export keeps working);
// b200pdlp_release_cache() empties it.  B200PDLP_CACHE_MB caps what is kept (default 16 GiB).
void* dev_cache_alloc(size_t bytes);
void dev_cache_free(void* p);
void dev_cache_release();
void* pinned_cache_alloc(size_t bytes, bool mapped);
void pinned_cache_free(void* p);

// sizes / scalars the host learns from the device during the prologue
struct PrepScalars {
  int neq = 0, nbound = 0, cols_sorted = 1, bad_index = 0;   // read-back 1
  long long a_padded = 0, at_padded = 0;                     // sliced-ELL slots of A and A' (read-back 2)
  int a_nlong = 0, a_nsegs = 0, at_nlong = 0, at_nsegs = 0;
  long long a_lcount = 8, at_lcount = 8;
  double norm_cost_sq = 0, norm_rhs_sq = 0;                  // unscaled cost (x sense) and rhs: sums of squares
                                                             // (HiPDLP mode: cost not x sense, added in index order)
  int scaled = 0;                                            // HiPDLP mode: some scaling pass ran (StdForm::scaled)
  float norms_ms = 0.f;                                      // HiPDLP mode: device time of the ordered norm sums
  double beta_cost_sq = 0, beta_rhs_sq = 0;                  // the same sums over the SCALED data (PDHG_Init_Step_Sizes)
  double amax = 0;                                           // max |a_ij| after scaling
  // sector sharing of the SpMV gathers, sampled over <= 4096 slices of each layout: distinct 32-byte sectors among the first
  // column ids of a slice's live lanes, and the number of those lanes (1.0 = every gather its own sector, 0.25 = consecutive)
  int a_sectors = 0, a_lanes = 0, at_sectors = 0, at_lanes = 0;
};

// what the prologue leaves on the device for the solve
struct DevProblemArrays {
  int n = 0, m = 0, nnz = 0, neq = 0, n0 = 0, nbound = 0;
  // by ORIGINAL row
  int* row_new_idx = nullptr;   // [m] standard-form row
  int* row_class = nullptr;     // [m] EQ 0, LEQ 1, GEQ 2, BOUND 3 (HiPDLP mode: FREE 4)
  int* bound_ord = nullptr;     // [m + 1] exclusive count of BOUND rows: slack column of BOUND row i = n0 + bound_ord[i]
                                // (HiPDLP mode: BOUND and FREE rows)
  int* row_old = nullptr;       // [m] original row of a standard-form row
  int* slack_row = nullptr;     // [nbound] original row of slack column n0 + k
  // device orderings (length-sorted in windows): perm[new] = old, inv[old] = new
  int *rperm = nullptr, *rinv = nullptr, *cperm = nullptr, *cinv = nullptr;
  // vectors in device order
  double *cost = nullptr, *lower = nullptr, *upper = nullptr, *colscale = nullptr, *rhs = nullptr, *rowscale = nullptr;
  // HiPDLP mode only
  double* rup = nullptr;        // [m] row upper bounds, device order
  int* orow_ptr = nullptr;      // [m + 1] the caller's matrix, row-major (a row's entries in column order): row pointer,
  int* orow_col = nullptr;      // [nnz0]  column ids,
  double* orow_val = nullptr;   // [nnz0]  values (for the postsolve's row_value = A x)
};

struct DevSellOwned {   // one sliced-ELL matrix, blocks owned through the cache
  int nrows = 0, ncols = 0, nslices = 0, nlong = 0, nsegs = 0;
  long long padded = 0, lcount = 0;
  int4* slices = nullptr;
  int* col = nullptr;
  double* val = nullptr;
  int4* segs = nullptr;
  int4* long_rows = nullptr;
  int* lcol = nullptr;
  double* lval = nullptr;
  double* long_partial = nullptr;
  unsigned* long_counter = nullptr;
  // tiled SpMV shape (kernels.cuh DevSell::tiled): per tile of kTileSlices slices the window of the input vector its rows touch
  int ntiles = 0, tiles_staged = 0;   // tiles_staged: tiles whose window fits the staging buffer
  int* tile_lo = nullptr;
  int* tile_w = nullptr;
  void release();
};

struct DevStdForm {     // tests only (keep_form): the scaled standard form, standard-form order
  int *cbeg = nullptr, *cidx = nullptr, *rptr = nullptr, *rpos = nullptr, *rcol = nullptr;   // rcol[q] = column of position rpos[q]
  double *cval = nullptr, *cost = nullptr, *lower = nullptr, *upper = nullptr, *colscale = nullptr, *rhs = nullptr,
         *rowscale = nullptr;
  double* row_upper = nullptr;   // HiPDLP mode
};

struct DevicePrologue {
  PrepScalars sc;
  DevProblemArrays arr;
  DevSellOwned A, AT;
  DevStdForm form;
  bool keep_form = false;
  bool stop_after_scaling = false;   // formulate + row index + scaling only (several GPUs: the layouts are built per rank by the host)
  // HiPDLP mode (solver=hipdlp): its own formulate and scaling (host twin host_prep_hipdlp.cpp), the same orderings and
  // layouts; `do_scale` is then ignored in favour of scaling_mode (bits 1 Ruiz, 4 Pock-Chambolle, 2 L2) / ruiz_iterations
  bool hipdlp = false;
  int scaling_mode = 0, ruiz_iterations = 0;
  // Block mode (HiPDLP mode on several GPUs, world > 1): the HiPDLP front and the one-GPU orderings as above, then the
  // nnz-balanced partition of the device rows and columns into `world` contiguous blocks (host twin: balanced_blocks in
  // host_prep.cpp) and, for every rank in `ranks`, A_g (device rows [rb[g], rb[g+1]), columns through cinv) and A_g'
  // (device columns [cb[g], cb[g+1]), columns through rinv) -- what build_hipdlp_shard builds on the host.  The one-GPU A / A',
  // the sector sampling and the tile windows are not built.  block_A[k] / block_AT[k] belong to rank ranks[k].
  int world = 1;
  std::vector<int> ranks;
  std::vector<int> rb, cb;                        // world + 1 block offsets each (read back)
  std::vector<DevSellOwned> block_A, block_AT;
  // The caller's eight LP arrays are device memory of this device (b200pdlp_solve_device, _hipdlp_device): the kernels read
  // them in place, with no staging copy and nothing on the side stream but the HiPDLP norms; h2d_bytes stays 0.  The host
  // cannot read a_start[num_col] then: device_nnz holds it.  Every kernel of the prologue only reads these arrays.
  bool inputs_on_device = false;
  int device_nnz = 0;
  size_t h2d_bytes = 0;   // bytes of the caller's arrays copied to the device
  // formulate + scale + row index + orderings + sliced-ELL layouts, all on stream `s`; returns with the stream idle.
  // Throws std::exception on bad input / CUDA errors (the caller releases what was produced so far).
  void run(cudaStream_t s, const b200pdlp_lp& lp, bool do_scale, int long_threshold);
  void release_arrays();
  void release_form();
  void release_blocks();   // whatever block_A / block_AT still own
};

// solve boundary for a device-resident problem: initial point (hot start / proj(0), start of the running sums) and
// PDHG_PostSolve into original-order arrays on the device (w* = hot-start vectors in original order, or nullptr)
void launch_init_point(cudaStream_t s, const DevProblemArrays& a, double sense, const double* wcol, const double* wrowval,
                       const double* wdual, const double* colscale, const double* lower, const double* upper,
                       const double* rowscale, double* x0, double* xsum, double* y0);
void launch_postsolve(cudaStream_t s, const DevProblemArrays& a, double sense, int have_check, const double* x, const double* aty,
                      const double* y, const double* ax, const double* cost, const double* lower, const double* upper,
                      const double* colscale, const double* rowscale, double* col_value, double* col_dual, double* row_value,
                      double* row_dual);
// HiPDLP mode (host twins: engine_hipdlp.cu solve_hipdlp_on_device).  Initial point x = xa = proj_[l,u](0) (upper bound first,
// then lower, pdhg.cc:512-552), device order.
void launch_hip_init_point(cudaStream_t s, int n, const double* lower, const double* upper, double* x, double* xa);
// unscaleSolution + postprocess (pdhg.cc:1883-1897, :359-492) into original-order arrays on the device: x, y only when
// `converged` (else 0), divided by their scales only when `scaled`; s+ and s- always times col_scale; LEQ row duals negated;
// col_dual = (s+ - s-) sense; row_value = A x over the caller's matrix, each row from 0.0 with the columns ascending
void launch_hip_postsolve(cudaStream_t s, const DevProblemArrays& a, double sense, int converged, int scaled, const double* x,
                          const double* y, const double* sp, const double* sn, const double* colscale, const double* rowscale,
                          double* col_value, double* col_dual, double* row_value, double* row_dual);

}  // namespace b200
