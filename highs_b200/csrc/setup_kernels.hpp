// highs_b200/csrc/setup_kernels.hpp -- device-side PDHG_Scale_Data (see setup_kernels.cu).
#pragma once
#include <cuda_runtime.h>

namespace b200 {

// the standard form's column-major matrix and vectors, resident on the device (standard-form order)
struct DevForm {
  int n, m, nnz;
  const int* cbeg;   // [n+1]
  const int* cidx;   // [nnz] row of each nonzero
  int* colof;        // [nnz] column of each nonzero
  double* cval;      // [nnz] scaled in place
  double *cost, *lower, *upper, *colscale;   // [n]
  double *rhs, *rowscale;                    // [m]
};
struct DevScaleScratch {
  double *cs, *cnorm;   // [n]
  double *rs, *rnorm;   // [m]
  double* amax;         // [1] max |a_ij| of the scaled matrix
};

// the 10 Ruiz passes (cupdlp_scaling.c:47-120); needs nothing but the column-major matrix (and its colof)
void device_scale_ruiz(cudaStream_t s, const DevForm& F, DevScaleScratch& w);
// *amax = max |val[p]|
void device_abs_max(cudaStream_t s, int nnz, const double* val, double* amax);
// the Pock-Chambolle pass (:174-231); rptr[m+1] / rpos[nnz] = device copy of the row-major index of the nonzeros
void device_scale_pock_chambolle(cudaStream_t s, const DevForm& F, DevScaleScratch& w, const int* rptr, const int* rpos);

// HiPDLP mode: Scaling::scaleProblem (hipdlp/scaling.cc:23-263), bit-identical to host_prep_hipdlp.cpp::scale_hipdlp.
// scaling_mode bits: 1 Ruiz (inf-norm) x ruiz_iterations, then 4 Pock-Chambolle (alpha = 1), then 2 L2.  Every pass divides
// a_ij by (r_i * c_j), scales only finite bounds and rhs / row_upper entries, and accumulates the scales.  Column sums run in
// a column's storage order, row sums in the order of the row-major index (rptr / rpos).  w.amax = max |a_ij| at the end.
// Returns true if any pass ran (the host's StdForm::scaled).
bool device_scale_hipdlp(cudaStream_t s, const DevForm& F, DevScaleScratch& w, const int* rptr, const int* rpos,
                         double* row_upper, int scaling_mode, int ruiz_iterations);

// where a sliced-ELL fill reads a row's entries from: entries [beg[r], end[r]) of the OLD row r, optionally through an
// index (pos), column id = colmap[idx[.] - idx_offset], value = val[.]
struct SellSource {
  const int* beg;
  const int* end;
  const int* pos;      // nullptr: direct
  const int* idx;
  const double* val;
  int idx_offset;
  const int* colmap;
};
// fills col/val[0 .. padded + 32) and, for n_long > 0, lcol/lval (which must be zero-initialised) from the plan's
// descriptors (all pointers are device pointers; perm[new row] = old row)
void device_fill_sell(cudaStream_t s, int nrows, int nslices, const int4* slices, const int* perm, const SellSource& S,
                      int* col, double* val, long long padded, int n_long, const int4* long_rows, const int4* segs,
                      int* lcol, double* lval);

}  // namespace b200
