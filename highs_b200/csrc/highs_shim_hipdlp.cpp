// highs_b200/csrc/highs_shim_hipdlp.cpp -- replaces /root/reference/highs/pdlp/HiPdlpWrapper.cpp when HiGHS is linked
// against the CUDA engine's HiPDLP mode (solver=hipdlp; sole call site highs/lp_data/HighsSolve.cpp:107-117).
//
// Defines  HighsStatus solveLpHiPdlp(HighsLpSolverObject&)  and the 8-reference overload (HiPdlpWrapper.h) with the
// behaviour of HiPdlpWrapper.cpp:26-141 -- reset status/info, read the options PDLPSolver::setup reads
// (hipdlp/pdhg.cc:1783-1874), fill the HighsSolution, pdlp_iteration_count, invalidate the basis, map the termination
// status -- and forwards the numerical work to b200pdlp_solve_hipdlp (include/b200pdlp.h).
// STATUS (round 2): runs on hardware (tests/test_gpu_dropin.py drives Highs::run() with solver=hipdlp through this shim);
// oracle/build_ref.py --shim links it into a SEPARATE library (oracle/_ref/libhighs_b200_hipdlp.so) next to the solver=pdlp
// drop-in (libhighs_b200.so).
#include <algorithm>
#include <cmath>
#include <cstdlib>

#include "lp_data/HighsLpSolverObject.h"
#include "lp_data/HighsSolution.h"

#include "b200pdlp.h"

HighsStatus solveLpHiPdlp(const HighsOptions& options, HighsTimer& timer, const HighsLp& lp, HighsBasis& highs_basis,
                          HighsSolution& highs_solution, HighsModelStatus& model_status, HighsInfo& highs_info,
                          HighsCallback& callback) {
  (void)callback;
  (void)timer;
  resetModelStatusAndHighsInfo(model_status, highs_info);
  static_assert(sizeof(HighsInt) == 4, "the engine uses 32-bit indices (build HiGHS without HIGHSINT64)");
  b200pdlp_lp clp;
  clp.num_col = lp.num_col_;
  clp.num_row = lp.num_row_;
  clp.a_start = lp.a_matrix_.start_.data();
  clp.a_index = lp.a_matrix_.index_.data();
  clp.a_value = lp.a_matrix_.value_.data();
  clp.col_cost = lp.col_cost_.data();
  clp.col_lower = lp.col_lower_.data();
  clp.col_upper = lp.col_upper_.data();
  clp.row_lower = lp.row_lower_.data();
  clp.row_upper = lp.row_upper_.data();
  clp.sense = lp.sense_ == ObjSense::kMaximize ? -1.0 : 1.0;
  clp.offset = lp.offset_;

  b200pdlp_hipdlp_params prm;   // PDLPSolver::setup, hipdlp/pdhg.cc:1820-1863
  b200pdlp_hipdlp_default_params(&prm);
  prm.tolerance = options.pdlp_optimality_tolerance;
  if (options.kkt_tolerance != kDefaultKktTolerance) prm.tolerance = options.kkt_tolerance;
  prm.iter_limit = (int32_t)std::min<int64_t>((int64_t)options.pdlp_iteration_limit, (int64_t)kHighsIInf32);
  prm.time_limit = options.time_limit < kHighsInf ? options.time_limit : -1.0;   // < 0 = none; 0 ends the run at the first check
  prm.scaling_mode = (options.pdlp_features_off & kPdlpScalingOff) == 0 ? (int32_t)options.pdlp_scaling_mode : 0;
  prm.ruiz_iterations = (int32_t)options.pdlp_ruiz_iterations;
  prm.step_size_strategy = options.pdlp_step_size_strategy == kPdlpStepSizeStrategyFixed ? 0 : 3;
  prm.log_level = options.output_flag ? (options.log_dev_level ? 2 : 1) : 0;

  highs_solution.clear();
  highs_solution.col_value.resize(lp.num_col_);
  highs_solution.row_value.resize(lp.num_row_);
  highs_solution.col_dual.resize(lp.num_col_);
  highs_solution.row_dual.resize(lp.num_row_);
  b200pdlp_result res{};
  res.col_value = highs_solution.col_value.data();
  res.col_dual = highs_solution.col_dual.data();
  res.row_value = highs_solution.row_value.data();
  res.row_dual = highs_solution.row_dual.data();
  // B200PDLP_GPUS=N: N devices of this process (blocks of the device rows and columns, peer memory; the same bits as one GPU
  // with the host prologue)
  int ngpus = 1;
  if (const char* e = getenv("B200PDLP_GPUS")) ngpus = std::max(1, std::min(atoi(e), b200pdlp_device_count()));
  const int rc = ngpus > 1 ? b200pdlp_solve_hipdlp_multi(&clp, &prm, &res, ngpus, nullptr) : b200pdlp_solve_hipdlp(&clp, &prm, &res);
  model_status = HighsModelStatus::kUnknown;
  highs_basis.valid = false;
  if (rc != B200PDLP_OK) {
    highsLogUser(options.log_options, HighsLogType::kError, "B200 HiPDLP engine failed: %s\n", b200pdlp_last_error());
    return HighsStatus::kError;
  }
  highs_info.pdlp_iteration_count = res.iters;
  if (res.term_code == B200PDLP_OPTIMAL) model_status = HighsModelStatus::kOptimal;          // HiPdlpWrapper.cpp:96-127
  else if (res.term_iterate == 2) model_status = HighsModelStatus::kTimeLimit;
  else model_status = HighsModelStatus::kIterationLimit;
  highs_solution.value_valid = true;
  highs_solution.dual_valid = true;
  return HighsStatus::kOk;
}

HighsStatus solveLpHiPdlp(HighsLpSolverObject& solver_object) {
  return solveLpHiPdlp(solver_object.options_, solver_object.timer_, solver_object.lp_, solver_object.basis_,
                       solver_object.solution_, solver_object.model_status_, solver_object.highs_info_,
                       solver_object.callback_);
}
