// highs_b200/csrc/pdhg_kernels.hpp -- launcher declarations (host-callable) of pdhg_kernels.cu
#pragma once
#include "kernels.cuh"

namespace b200 {

struct ColIter { const double* x; const double* aty; };   // one primal-side iterate (n-vectors)
struct RowIter { const double* y; const double* ax; };    // one dual-side iterate (m-vectors)

void launch_primal_step(cudaStream_t s, int n, PdhgState* st, double* x0, double* x1, const double* aty0,
                        const double* aty1, const double* c, const double* lo, const double* up, double* xsum,
                        ReduceScratch rs, unsigned* xnz = nullptr, int l2_hints = 0);
// xnz / ynz: where K1 / K2 write the nonzero bitmap of x' / y' (DevSell::nzmap of A / A'), nullptr: nowhere
void launch_nz_bitmap(cudaStream_t s, int len, const double* v, unsigned* out);
int zskip_ctas_per_sm(int nz_bytes);
void launch_spmv_plain(cudaStream_t s, const DevSell& A, const double* in, double* out, const PdhgState* due = nullptr);
void launch_spmv_dual(cudaStream_t s, const DevSell& A, PdhgState* st, const double* x0, const double* x1,
                      double* y0, double* y1, double* ax0, double* ax1, const double* b, double* ysum,
                      int neq, int row_offset, ReduceScratch rs, double* axsum = nullptr, unsigned* ynz = nullptr);
void launch_spmv_primal(cudaStream_t s, const DevSell& A, PdhgState* st, const double* y0, const double* y1,
                        const double* x0, const double* x1, double* aty0, double* aty1, ReduceScratch rs,
                        double* atysum = nullptr);
void launch_spmv_partial_aty(cudaStream_t s, const DevSell& A, PdhgState* st, const double* y0, const double* y1,
                             double* part, const int* outpos, const PdhgState* due = nullptr);
void launch_spmv_dual_mg(cudaStream_t s, const DevSell& A, PdhgState* st, const double* xfull, double* y0, double* y1,
                         double* ax0, double* ax1, const double* b, double* ysum, int neq, ReduceScratch rs,
                         double* axsum = nullptr);
void launch_primal_shard(cudaStream_t s, int len, PdhgState* st, double* xs0, double* xs1, double* aty_s,
                         const double* red, const double* c, const double* lo, const double* up, double* xsum,
                         double* send, ReduceScratch rs);
int primal_shard_grid(int len);
int primal_shard_p2p_grid(int len);
void launch_stash_scalars(cudaStream_t s, int nv, PdhgState* st, const double* partials, int nb, double* dst, int copies,
                          int stride);
void launch_primal_shard_p2p(cudaStream_t s, int len, PdhgState* st, double* xs0, double* xs1, double* aty_s,
                             const PeerPtrs& pp, int world, int rank, int seg_len, const double* c,
                             const double* lo, const double* up, double* xsum, ReduceScratch rs, double* atysum = nullptr);
void launch_push_shard(cudaStream_t s, const double* src, int len, const PeerPtrs& pp, int world, int rank, int seg_len,
                       const PdhgState* due = nullptr);
void launch_push_rows(cudaStream_t s, const double* src, int len, const PeerPtrs& pp, int world, int rank, int seg_len);
void launch_p2p_exchange(cudaStream_t s, double* vals, int k, const PeerPtrs& pp, int world, int rank,
                         unsigned long long* epochs, int* fault, const PdhgState* due = nullptr,
                         const SolveCtl* only_if_restart = nullptr /* skip (on every rank alike) unless the check chose a restart */);
// pull 1: add the peers' `part` segments (a pass's partial A_g^T y'); 2: their `recv` (a check's partial A_g^T ybar)
void launch_reduce_part_p2p(cudaStream_t s, int len, double* dst, const PeerPtrs& pp, int world, int rank, int seg_len,
                            int pull, const PdhgState* due = nullptr, int only_if_accepted = 0);
void launch_p2p_barrier(cudaStream_t s, int mode, PdhgState* st, const double* partials, int nb, const PeerPtrs& pp,
                        int world, int rank, int seg_len, int shard_len, unsigned long long* epochs, int* fault);
void launch_step_rule_mg(cudaStream_t s, PdhgState* st, const double* xfull, int world, int seg_len, int shard_len,
                         const double* red);
void launch_step_rule(cudaStream_t s, PdhgState* st, ReduceScratch r1, int nb1, ReduceScratch r2, int nb2,
                      ReduceScratch r3, int nb3, const double* dy2_override);
int primal_step_grid(int n);
// load every kernel of the multi-GPU path now (see pdhg_kernels.cu: lazy module loading vs. spinning barrier kernels)
void preload_multi_gpu_kernels();
void launch_average(cudaStream_t s, int len, const double* v, double* sum, double* avg, int pending, double w,
                    double scale);
void launch_col_check_a(cudaStream_t s, int n, int nit, ColIter a, ColIter b, const double* c, const double* lo,
                        const double* up, const double* cs, ReduceScratch rs, double* out);
void launch_col_check_fused(cudaStream_t s, int n, ColIter a, ColIter b, const double* c, const double* lo,
                            const double* up, const double* cs, ReduceScratch rs, double* out,
                            const PdhgState* st = nullptr, ColIter alt = ColIter{nullptr, nullptr});
void launch_row_check_fused(cudaStream_t s, int m, RowIter a, RowIter b, const double* rhs, const double* rsca, int neq,
                            ReduceScratch rs, double* out);
void launch_average_dev(cudaStream_t s, int len, const double* v0, const double* v1, double* sum, double* avg,
                        const PdhgState* st);
void launch_row_check_a(cudaStream_t s, int m, int nit, RowIter a, RowIter b, const double* rhs,
                        const double* rsca, int neq, int row_offset, ReduceScratch rs, double* out);
void launch_col_check_b(cudaStream_t s, int n, int nit, ColIter a, ColIter b, const double inv_d[2],
                        const double inv_p[2], const double* c, const double* lo, const double* up,
                        const double* cs, ReduceScratch rs, double* out);
void launch_row_check_b(cudaStream_t s, int m, int nit, RowIter a, RowIter b, const double inv_p[2],
                        const double* rsca, int neq, int row_offset, ReduceScratch rs, double* out);
void launch_diff_norm2(cudaStream_t s, int len, const double* a, const double* b, ReduceScratch rs, double* out);
void launch_scale(cudaStream_t s, int len, double* v, double w);
void launch_fill(cudaStream_t s, int len, double* v, double w);

// ---- device-side check iteration (tree mode, one GPU): see pdhg_kernels.cu "device-side check iteration"
void launch_check_avg_x(cudaStream_t s, int n, const double* x0, const double* x1, double* xsum, double* xavg,
                        const PdhgState* st, const SolveCtl* ctl);
void launch_check_decide(cudaStream_t s, PdhgState* st, SolveCtl* ctl, const double* prow, int nbr, const double* pcol,
                         int nbc, unsigned* ticket /* zero-initialised, self-resetting */);
int restart_sweep_grid(int n, int m);
void launch_restart_sweep(cudaStream_t s, int n, int m, double* x0, double* x1, double* aty0, double* aty1,
                          const double* xavg, const double* atyavg, double* xsum, double* xlr, double* y0, double* y1,
                          double* ax0, double* ax1, const double* yavg, const double* axavg, double* ysum, double* ylr,
                          const PdhgState* st, const SolveCtl* ctl, ReduceScratch rs, double* atysum = nullptr,
                          double* axsum = nullptr);
// the residual sweeps as plain vector kernels: given = true (split check: xbar/ybar from launch_check_avg_xy, A xbar / A'ybar
// from two plain SpMV) or false (light check of the dense-check phase: from the carried A xSum / A'ySum); partial-sum layout
// [20][check_light_grid(n, true)], [8][check_light_grid(m, false)]
int check_light_grid(int len, bool cols);
void launch_check_cols_sweep(cudaStream_t s, bool given, int n, const double* x0, const double* x1, const double* aty0,
                             const double* aty1, double* xsum, double* atysum, double* xavg, double* atyavg, const double* c,
                             const double* lo, const double* up, const double* cs, const PdhgState* st, const SolveCtl* ctl,
                             ReduceScratch rs);
void launch_check_rows_sweep(cudaStream_t s, bool given, int m, int neq, const double* y0, const double* y1, const double* ax0,
                             const double* ax1, double* ysum, double* axsum, double* yavg, double* axavg, const double* b,
                             const double* rsc, const PdhgState* st, const SolveCtl* ctl, ReduceScratch rs);
void launch_check_light_off(cudaStream_t s, PdhgState* st, const SolveCtl* ctl);
void launch_check_avg_xy(cudaStream_t s, int n, int m, const double* x0, const double* x1, double* xsum, double* xavg,
                         const double* y0, const double* y1, double* ysum, double* yavg, const PdhgState* st, const SolveCtl* ctl);
void launch_check_finish(cudaStream_t s, PdhgState* st, SolveCtl* ctl, const double* prst, int nbs, const double* sums2 = nullptr);
// several GPUs (fused peer-memory path): row side with ybar already formed, partial sums -> scalars, decision from all-reduced sums
void launch_spmv_check_rows_mg(cudaStream_t s, const DevSell& A, const PdhgState* st, const SolveCtl* ctl, const double* xfull,
                               const double* y0, const double* y1, const double* ax0, const double* ax1, const double* yavg,
                               double* axavg, const double* b, const double* rsc, int neq, ReduceScratch rs);
void launch_reduce_partials(cudaStream_t s, const PdhgState* st, const SolveCtl* ctl, int nacc, const double* partials, int nb,
                            double* out, int flag_slot /* in the LAST output array, or -1 */, int need_restart, int nacc2 = 0,
                            const double* partials2 = nullptr, int nb2 = 0, double* out2 = nullptr);
void launch_check_decide_sums(cudaStream_t s, PdhgState* st, SolveCtl* ctl, const double* outs);

// ---- HiPDLP mode (reflected Halpern PDHG; pdhg_kernels.cu, last section)
struct HipCheckArgs {
  int n, m, neq, scaled;
  double offset;
  const double *x, *y, *ax, *aty;
  const double *rx, *ry, *atdy;
  const double *xa, *ya;
  const double *c, *lo, *up, *rlo, *colscale, *rowscale, *sp, *sn;
};
void launch_hip_primal(cudaStream_t s, int n, const HipState* st, int k_offset, int is_major, double* x, const double* xa,
                       const double* c, const double* aty, const double* lo, const double* up, double* rx, double* xn,
                       double* hslack);
void launch_hip_dual(cudaStream_t s, const DevSell& A, const HipState* st, int k_offset, int is_major, const double* rx,
                     double* y, const double* ya, const double* rlo, const double* rup, double* yn, double* ry);
void launch_hip_diff(cudaStream_t s, int len, const double* a, const double* b, double* out);
void launch_hip_slack(cudaStream_t s, int n, int use_cached, const double* hslack, const double* c, const double* aty,
                      const double* lo, const double* up, double* sp, double* sn);
void launch_hip_check(cudaStream_t s, const HipCheckArgs& a, int with_fpe, int ordered, ReduceScratch rs, double* out);
void launch_hip_dot(cudaStream_t s, int len, const double* a, const double* b, int ordered, ReduceScratch rs, double* out);
void launch_hip_div_norm(cudaStream_t s, int len, double* v, const double* norm_sq);

// ---- HiPDLP on several GPUs (pdhg_kernels.cu, "HiPDLP shards"): every rank holds full-length vectors in the one-GPU
// device order; peers' copies of one vector, by rank (this rank's own entry included)
struct PeerVec { double* v[kMaxPeers]; };
struct PeerFlags { unsigned long long* f[kMaxPeers]; };   // every rank's kMaxPeers arrival words
constexpr int kMaxGather = 4;
struct HipGather {   // entries [lo, hi) of up to kMaxGather vectors, copied from this rank into every peer
  const double* src[kMaxGather];
  PeerVec dst[kMaxGather];
  int nv, lo, hi;
};
void launch_hip_primal_shard(cudaStream_t s, int c0, int c1, const HipState* st, int k_offset, int is_major, double* x,
                             const double* xa, const double* c, const double* aty, const double* lo, const double* up,
                             double* rx, double* xn, double* hslack, const PeerVec& rx_peers, int world, int rank);
void launch_hip_dual_shard(cudaStream_t s, const DevSell& A, const HipState* st, int k_offset, int is_major, const double* rx,
                           double* y, const double* ya, const double* rlo, const double* rup, double* yn, double* ry,
                           const PeerVec& y_peers, int world, int rank);
void launch_hip_gather(cudaStream_t s, const HipGather& g, int world, int rank);
void launch_hip_barrier(cudaStream_t s, const PeerFlags& flags, int world, int rank, unsigned long long* epoch, int* fault);
void preload_hipdlp_shard_kernels();

}  // namespace b200
