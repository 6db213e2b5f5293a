// highs_b200/csrc/kkt_check.cu -- HiGHS's post-solve KKT assessment on the device (SURVEY.md 8(f) rank 4) and its host twin.
//
// After solveLpCupdlp returns, Highs::run() evaluates the HighsSolution with lpKktCheck
// (/root/reference/highs/lp_data/HighsSolution.cpp:1043-1327 -> getKktFailures :73-495): A x and A'y in quad precision,
// two sweeps over all columns and rows, complementarity, dual objective -- single-threaded, about as long as a
// 20-iteration GPU solve at 1M x 1M.  Here: the same quantities from the original (unscaled) HighsLp arrays and the
// solution vectors copied to HBM; per-variable arithmetic shared with the host twin through kkt_logic.hpp.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/b200pdlp.h"
#include "device_prep.hpp"
#include "kkt_batch.hpp"
#include "kkt_logic.hpp"

namespace b200 {

// ---- shared epilogue (also of the batch, kkt_batch.hpp): HighsInfo fields + lpKktCheck's status rules for a solution
// without a basis (:1207-1323)
void finalize_kkt(const KktSums& s, double offset, const KktTolerances& t, b200pdlp_kkt_info* out) {
  out->objective_function_value = offset + s.objective;
  out->num_primal_infeasibilities = s.num_primal_infeasibility;
  out->max_primal_infeasibility = s.max_primal_infeasibility;
  out->sum_primal_infeasibilities = s.sum_primal_infeasibility;
  out->num_dual_infeasibilities = s.num_dual_infeasibility;
  out->max_dual_infeasibility = s.max_dual_infeasibility;
  out->sum_dual_infeasibilities = s.sum_dual_infeasibility;
  out->num_relative_primal_infeasibilities = s.num_relative_primal_infeasibility;
  out->max_relative_primal_infeasibility = s.max_relative_primal_infeasibility;
  out->num_relative_dual_infeasibilities = s.num_relative_dual_infeasibility;
  out->max_relative_dual_infeasibility = s.max_relative_dual_infeasibility;
  out->num_primal_residual_errors = s.num_primal_residual_error;
  out->max_primal_residual_error = s.max_primal_residual_error;
  out->num_dual_residual_errors = s.num_dual_residual_error;
  out->max_dual_residual_error = s.max_dual_residual_error;
  out->num_relative_primal_residual_errors = s.num_relative_primal_residual_error;
  out->max_relative_primal_residual_error = s.max_relative_primal_residual_error;
  out->num_relative_dual_residual_errors = s.num_relative_dual_residual_error;
  out->max_relative_dual_residual_error = s.max_relative_dual_residual_error;
  out->num_complementarity_violations = s.num_complementarity_violation;
  out->max_complementarity_violation = s.max_complementarity_violation;
  const double dual_objective = offset + s.dual_objective;               // computeDualObjectiveValue :1345-1386
  out->dual_objective_value = dual_objective;
  out->primal_dual_objective_error = std::fabs(out->objective_function_value - dual_objective) /
                                     (1.0 + std::fabs(out->objective_function_value) + std::fabs(dual_objective));   // :468-495
  // lpKktCheck (no basis): kUnboundedOrInfeasible (9) -> kUnbounded (10) if primal feasible with no residual errors (:1074-1077)
  int status = out->model_status;
  if (status == 9 && out->num_primal_infeasibilities == 0 && out->num_primal_residual_errors == 0) status = 10;
  double max_primal = 0, max_dual = 0, pd = 0;
  max_primal = std::max(out->max_relative_primal_infeasibility / t.primal_feasibility, max_primal);
  max_dual = std::max(out->max_relative_dual_infeasibility / t.dual_feasibility, max_dual);
  max_primal = std::max(out->max_relative_primal_residual_error / t.primal_residual, max_primal);
  max_dual = std::max(out->max_relative_dual_residual_error / t.dual_residual, max_dual);
  if (out->primal_dual_objective_error > t.optimality) pd = out->primal_dual_objective_error / t.optimality;
  const double allowed = 1e2;   // max_allowed_tolerance_relative_violation
  out->primal_solution_status = max_primal > allowed ? 1 : 2;   // kSolutionStatusInfeasible / Feasible
  out->dual_solution_status = max_dual > allowed ? 1 : 2;
  const double worst = std::max(pd, std::max(max_primal, max_dual));
  if (status == 7) { if (worst > allowed) status = 15; }          // kOptimal -> kUnknown
  else if (status == 15 && worst <= allowed) status = 7;          // kUnknown -> kOptimal
  out->model_status = status;
}

KktTolerances tolerances_of(const b200pdlp_kkt_tolerances* t) {
  return KktTolerances{t->primal_feasibility_tolerance, t->dual_feasibility_tolerance, t->primal_residual_tolerance,
                       t->dual_residual_tolerance, t->optimality_tolerance};
}

// ---- host twin (sequential; the reference's loop order)
static void kkt_host(const b200pdlp_lp& lp, const double* cv, const double* cd, const double* rv, const double* rd,
                     const KktTolerances& t, b200pdlp_kkt_info* out) {
  const int n = lp.num_col, m = lp.num_row;
  std::vector<DD> acc(m);
  std::vector<double> pact(m), dact(n);
  for (int j = 0; j < n; j++)
    for (int p = lp.a_start[j]; p < lp.a_start[j + 1]; p++) acc[lp.a_index[p]].add(cv[j] * lp.a_value[p]);
  for (int i = 0; i < m; i++) pact[i] = acc[i].value();
  for (int j = 0; j < n; j++) {
    DD v;
    for (int p = lp.a_start[j]; p < lp.a_start[j + 1]; p++) v.add(rd[lp.a_index[p]] * lp.a_value[p]);
    dact[j] = v.value() - lp.col_cost[j];
  }
  double norm_bounds = 0, norm_costs = 0;
  for (int j = 0; j < n; j++) kkt_pass0(t, true, lp.col_cost[j], lp.col_lower[j], lp.col_upper[j], cv[j], cd[j], lp.sense, norm_bounds, norm_costs);
  for (int i = 0; i < m; i++) kkt_pass0(t, false, 0.0, lp.row_lower[i], lp.row_upper[i], rv[i], rd[i], lp.sense, norm_bounds, norm_costs);
  KktSums s;
  for (int j = 0; j < n; j++)
    kkt_pass1(t, true, lp.col_cost[j], lp.col_lower[j], lp.col_upper[j], cv[j], cd[j], lp.sense, norm_bounds, norm_costs,
              std::fabs(dact[j] + cd[j]), s);
  for (int i = 0; i < m; i++)
    kkt_pass1(t, false, 0.0, lp.row_lower[i], lp.row_upper[i], rv[i], rd[i], lp.sense, norm_bounds, norm_costs,
              std::fabs(pact[i] - rv[i]), s);
  out->norm_bounds = norm_bounds; out->norm_costs = norm_costs;
  finalize_kkt(s, lp.offset, t, out);
}

// ---- device
namespace {
constexpr int kTpb = 256;
inline int grid_for(long long work) {
  long long g = (work + kTpb - 1) / kTpb;
  if (g < 1) g = 1;
  return (int)(g > kGridUnit * 16LL ? kGridUnit * 16LL : g);
}
inline int warp_grid(long long rows) { return (int)std::max<long long>(1, (rows * 32 + kTpb - 1) / kTpb); }

__device__ __forceinline__ DD warp_dd_sum(DD v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    DD w;
    w.hi = __shfl_down_sync(0xffffffffu, v.hi, o);
    w.lo = __shfl_down_sync(0xffffffffu, v.lo, o);
    v.add(w);
  }
  return v;
}
__global__ void __launch_bounds__(kTpb) iota_k(int len, int* v) {
  const int stride = gridDim.x * kTpb;
  for (int i = blockIdx.x * kTpb + threadIdx.x; i < len; i += stride) v[i] = i;
}
__global__ void __launch_bounds__(kTpb) hist_k(int nnz, const int* __restrict__ idx, int* __restrict__ cnt) {
  const int stride = gridDim.x * kTpb;
  for (int p = blockIdx.x * kTpb + threadIdx.x; p < nnz; p += stride) atomicAdd(&cnt[idx[p]], 1);
}
__global__ void __launch_bounds__(kTpb) colof_k(int n, const int* __restrict__ beg, int* __restrict__ colof) {
  const int j = (blockIdx.x * kTpb + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (j >= n) return;
  for (int p = beg[j] + lane; p < beg[j + 1]; p += 32) colof[p] = j;
}
// |A x - row_value| per row: productQuad (one warp per row over the row-major index)
__global__ void __launch_bounds__(kTpb)
row_residual_k(int m, const int* __restrict__ rptr, const int* __restrict__ rpos, const int* __restrict__ colof,
               const double* __restrict__ aval, const double* __restrict__ x, const double* __restrict__ rv, double* __restrict__ res) {
  const int i = (blockIdx.x * kTpb + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= m) return;
  DD v;
  for (int q = rptr[i] + lane; q < rptr[i + 1]; q += 32) { const int p = rpos[q]; v.add(x[colof[p]] * aval[p]); }
  v = warp_dd_sum(v);
  if (lane == 0) res[i] = fabs(v.value() - rv[i]);
}
// |A'y - c + col_dual| per column: productTransposeQuad
__global__ void __launch_bounds__(kTpb)
col_residual_k(int n, const int* __restrict__ beg, const int* __restrict__ idx, const double* __restrict__ aval,
               const double* __restrict__ y, const double* __restrict__ cost, const double* __restrict__ cd, double* __restrict__ res) {
  const int j = (blockIdx.x * kTpb + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (j >= n) return;
  DD v;
  for (int p = beg[j] + lane; p < beg[j + 1]; p += 32) v.add(y[idx[p]] * aval[p]);
  v = warp_dd_sum(v);
  if (lane == 0) { const double da = v.value() - cost[j]; res[j] = fabs(da + cd[j]); }
}
__device__ __forceinline__ void atomic_max_nonneg(double* addr, double v) {
  atomicMax(reinterpret_cast<unsigned long long*>(addr), (unsigned long long)__double_as_longlong(v));
}
struct KktVecs {
  int n, m;
  const double *cost, *cl, *cu, *rl, *ru, *cv, *cd, *rv, *rd, *cres, *rres;
  double sense;
};
__global__ void __launch_bounds__(kTpb) pass0_k(KktVecs a, KktTolerances t, double* __restrict__ norms) {
  double nb = 0, nc = 0;
  const int stride = gridDim.x * kTpb, total = a.n + a.m;
  for (int v = blockIdx.x * kTpb + threadIdx.x; v < total; v += stride) {
    if (v < a.n) kkt_pass0(t, true, a.cost[v], a.cl[v], a.cu[v], a.cv[v], a.cd[v], a.sense, nb, nc);
    else { const int i = v - a.n; kkt_pass0(t, false, 0.0, a.rl[i], a.ru[i], a.rv[i], a.rd[i], a.sense, nb, nc); }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    nb = kmax(nb, __shfl_down_sync(0xffffffffu, nb, o));
    nc = kmax(nc, __shfl_down_sync(0xffffffffu, nc, o));
  }
  if ((threadIdx.x & 31) == 0) { atomic_max_nonneg(norms, nb); atomic_max_nonneg(norms + 1, nc); }
}
__global__ void __launch_bounds__(kTpb) pass1_k(KktVecs a, KktTolerances t, const double* __restrict__ norms, KktSums* __restrict__ part) {
  __shared__ KktSums sm[kTpb / 32];
  const double nb = norms[0], nc = norms[1];
  KktSums s;
  const int stride = gridDim.x * kTpb, total = a.n + a.m;
  for (int v = blockIdx.x * kTpb + threadIdx.x; v < total; v += stride) {
    if (v < a.n) kkt_pass1(t, true, a.cost[v], a.cl[v], a.cu[v], a.cv[v], a.cd[v], a.sense, nb, nc, a.cres[v], s);
    else { const int i = v - a.n; kkt_pass1(t, false, 0.0, a.rl[i], a.ru[i], a.rv[i], a.rd[i], a.sense, nb, nc, a.rres[i], s); }
  }
  // warp tree, then the block's warps in order: deterministic
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int o = 16; o > 0; o >>= 1) {
    KktSums w;
    int* wi = reinterpret_cast<int*>(&w);
    const int* si = reinterpret_cast<const int*>(&s);
    for (int k = 0; k < (int)(sizeof(KktSums) / sizeof(int)); k++) wi[k] = __shfl_down_sync(0xffffffffu, si[k], o);
    kkt_merge(s, w);
  }
  if (lane == 0) sm[wid] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    KktSums tot = sm[0];
    for (int w = 1; w < kTpb / 32; w++) kkt_merge(tot, sm[w]);
    part[blockIdx.x] = tot;
  }
}
__global__ void merge_k(int nb, const KktSums* __restrict__ part, KktSums* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  KktSums tot = part[0];
  for (int b = 1; b < nb; b++) kkt_merge(tot, part[b]);
  *out = tot;
}
#define KKT_OK(call)                                                                                       \
  do {                                                                                                     \
    cudaError_t e_ = (call);                                                                               \
    if (e_ != cudaSuccess)                                                                                 \
      throw std::runtime_error(std::string(#call) + ": " + cudaGetErrorString(e_) + " at kkt_check.cu:" + \
                               std::to_string(__LINE__));                                                  \
  } while (0)
struct Tmp {
  cudaStream_t stream = nullptr;
  std::vector<void*> blocks;
  template <class T> T* get(size_t count) {
    void* p = dev_cache_alloc(std::max<size_t>(count, 1) * sizeof(T));
    blocks.push_back(p);
    return static_cast<T*>(p);
  }
  ~Tmp() { if (stream) cudaStreamSynchronize(stream); for (void* p : blocks) dev_cache_free(p); }
};
}  // namespace

static void kkt_device(const b200pdlp_lp& lp, const double* cv, const double* cd, const double* rv, const double* rd,
                       const KktTolerances& t, b200pdlp_kkt_info* out) {
  NvtxRange nvtx("b200pdlp: KKT check (device)");
  const int n = lp.num_col, m = lp.num_row, nnz = lp.a_start[n];
  cudaStream_t s = nullptr;
  KKT_OK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  struct StreamGuard { cudaStream_t s; ~StreamGuard() { cudaStreamDestroy(s); } } sg{s};
  Tmp tmp;
  tmp.stream = s;
  auto up_d = [&](const double* h, size_t cnt) { double* d = tmp.get<double>(cnt); if (cnt) KKT_OK(cudaMemcpyAsync(d, h, cnt * 8, cudaMemcpyHostToDevice, s)); return d; };
  auto up_i = [&](const int* h, size_t cnt) { int* d = tmp.get<int>(cnt); if (cnt) KKT_OK(cudaMemcpyAsync(d, h, cnt * 4, cudaMemcpyHostToDevice, s)); return d; };
  int* beg = up_i(lp.a_start, n + 1);
  int* idx = up_i(lp.a_index, nnz);
  double* aval = up_d(lp.a_value, nnz);
  KktVecs a{};
  a.n = n; a.m = m; a.sense = lp.sense;
  a.cost = up_d(lp.col_cost, n); a.cl = up_d(lp.col_lower, n); a.cu = up_d(lp.col_upper, n);
  a.rl = up_d(lp.row_lower, m); a.ru = up_d(lp.row_upper, m);
  a.cv = up_d(cv, n); a.cd = up_d(cd, n); a.rv = up_d(rv, m); a.rd = up_d(rd, m);
  // row-major index of the nonzeros (stable sort of the positions by row: columns ascending within a row, the order in
  // which productQuad adds into a row)
  int* rptr = tmp.get<int>(m + 2);
  int* rpos = tmp.get<int>(nnz);
  int* colof = tmp.get<int>(nnz);
  {
    int* cnt = tmp.get<int>(m + 2);
    KKT_OK(cudaMemsetAsync(cnt, 0, (size_t)(m + 2) * sizeof(int), s));
    if (nnz > 0) hist_k<<<grid_for(nnz), kTpb, 0, s>>>(nnz, idx, cnt);
    size_t bytes = 0;
    KKT_OK(cub::DeviceScan::ExclusiveSum(nullptr, bytes, cnt, rptr, m + 1, s));
    void* w = tmp.get<char>(bytes);
    KKT_OK(cub::DeviceScan::ExclusiveSum(w, bytes, cnt, rptr, m + 1, s));
    if (n > 0) colof_k<<<warp_grid(n), kTpb, 0, s>>>(n, beg, colof);
    if (nnz > 0) {
      int* k_out = tmp.get<int>(nnz);
      int* v_in = tmp.get<int>(nnz);
      iota_k<<<grid_for(nnz), kTpb, 0, s>>>(nnz, v_in);
      int end_bit = 1;
      while ((1LL << end_bit) <= (long long)std::max(m - 1, 1) && end_bit < 31) end_bit++;
      bytes = 0;
      KKT_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, idx, k_out, v_in, rpos, nnz, 0, end_bit, s));
      void* w2 = tmp.get<char>(bytes);
      KKT_OK(cub::DeviceRadixSort::SortPairs(w2, bytes, idx, k_out, v_in, rpos, nnz, 0, end_bit, s));
    }
  }
  double* rres = tmp.get<double>(m);
  double* cres = tmp.get<double>(n);
  if (m > 0) row_residual_k<<<warp_grid(m), kTpb, 0, s>>>(m, rptr, rpos, colof, aval, a.cv, a.rv, rres);
  if (n > 0) col_residual_k<<<warp_grid(n), kTpb, 0, s>>>(n, beg, idx, aval, a.rd, a.cost, a.cd, cres);
  a.rres = rres; a.cres = cres;
  double* norms = tmp.get<double>(2);
  KKT_OK(cudaMemsetAsync(norms, 0, 2 * sizeof(double), s));
  const int g = grid_for((long long)n + m);
  pass0_k<<<g, kTpb, 0, s>>>(a, t, norms);
  KktSums* part = tmp.get<KktSums>(g + 1);
  pass1_k<<<g, kTpb, 0, s>>>(a, t, norms, part);
  merge_k<<<1, 32, 0, s>>>(g, part, part + g);
  KktSums hs;
  double hn[2];
  KKT_OK(cudaMemcpyAsync(&hs, part + g, sizeof(KktSums), cudaMemcpyDeviceToHost, s));
  KKT_OK(cudaMemcpyAsync(hn, norms, sizeof(hn), cudaMemcpyDeviceToHost, s));
  KKT_OK(cudaStreamSynchronize(s));
  KKT_OK(cudaGetLastError());
  out->norm_bounds = hn[0]; out->norm_costs = hn[1];
  finalize_kkt(hs, lp.offset, t, out);
}

}  // namespace b200

extern "C" {

void b200pdlp_kkt_default_tolerances(b200pdlp_kkt_tolerances* t, double kkt_tolerance) {
  const double v = kkt_tolerance > 0 ? kkt_tolerance : 1e-7;   // kDefaultKktTolerance
  t->primal_feasibility_tolerance = t->dual_feasibility_tolerance = t->primal_residual_tolerance = t->dual_residual_tolerance =
      t->optimality_tolerance = v;
}

static int kkt_entry(bool device, const b200pdlp_lp* lp, const double* cv, const double* cd, const double* rv, const double* rd,
                     const b200pdlp_kkt_tolerances* tol, b200pdlp_kkt_info* out) {
  if (!lp || !cv || !cd || !rv || !rd || !tol || !out || lp->num_col < 0 || lp->num_row < 0 || !lp->a_start) return B200PDLP_ERR_ARG;
  try {
    const b200::KktTolerances t = b200::tolerances_of(tol);
    if (device) {
      int ndev = 0;
      if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return B200PDLP_ERR_CUDA; }   // no CPU fallback
      b200::kkt_device(*lp, cv, cd, rv, rd, t, out);
    } else {
      b200::kkt_host(*lp, cv, cd, rv, rd, t, out);
    }
    return B200PDLP_OK;
  } catch (const std::bad_alloc&) {
    return B200PDLP_ERR_ALLOC;
  } catch (const std::exception&) {
    return device ? B200PDLP_ERR_CUDA : B200PDLP_ERR_STATE;
  }
}

int b200pdlp_kkt_check(const b200pdlp_lp* lp, const double* col_value, const double* col_dual, const double* row_value,
                       const double* row_dual, const b200pdlp_kkt_tolerances* tol, b200pdlp_kkt_info* out) {
  return kkt_entry(true, lp, col_value, col_dual, row_value, row_dual, tol, out);
}
int b200pdlp_kkt_check_host(const b200pdlp_lp* lp, const double* col_value, const double* col_dual, const double* row_value,
                            const double* row_dual, const b200pdlp_kkt_tolerances* tol, b200pdlp_kkt_info* out) {
  return kkt_entry(false, lp, col_value, col_dual, row_value, row_dual, tol, out);
}

}  // extern "C"
