"""ctypes binding of libb200pdlp.so (C ABI: include/b200pdlp.h).

Plumbing only: it marshals numpy arrays into the C structs.  There is no CPU
fallback -- if the CUDA extension is missing or no device is visible every compute
entry point raises `EngineError`.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .lp import HighsLp

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200pdlp.so")

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)

TERM_NAMES = {0: "OPTIMAL", 1: "INFEASIBLE", 2: "UNBOUNDED", 3: "INFEASIBLE_OR_UNBOUNDED",
              4: "TIMELIMIT_OR_ITERLIMIT", 5: "FEASIBLE"}


class EngineError(RuntimeError):
    pass


class CLp(C.Structure):
    _fields_ = [("num_col", C.c_int32), ("num_row", C.c_int32), ("a_start", _ip), ("a_index", _ip),
                ("a_value", _dp), ("col_cost", _dp), ("col_lower", _dp), ("col_upper", _dp),
                ("row_lower", _dp), ("row_upper", _dp), ("sense", C.c_double), ("offset", C.c_double)]


class CParams(C.Structure):
    _fields_ = [("iter_limit", C.c_int32), ("tol_primal", C.c_double), ("tol_dual", C.c_double),
                ("tol_gap", C.c_double), ("time_limit", C.c_double), ("scaling", C.c_int32),
                ("adaptive_step", C.c_int32), ("restart", C.c_int32), ("log_level", C.c_int32),
                ("check_interval", C.c_int32), ("device", C.c_int32), ("graph_passes", C.c_int32),
                ("ordered_max", C.c_int32), ("device_scaling", C.c_int32), ("reserved", C.c_int32 * 2)]


class CHipdlpParams(C.Structure):
    _fields_ = [("tolerance", C.c_double), ("iter_limit", C.c_int32), ("scaling_mode", C.c_int32),
                ("ruiz_iterations", C.c_int32), ("step_size_strategy", C.c_int32), ("time_limit", C.c_double),
                ("ordered_max", C.c_int32), ("device", C.c_int32), ("log_level", C.c_int32), ("device_prep", C.c_int32),
                ("reserved", C.c_int32 * 2)]


class CCheckIn(C.Structure):
    """b200pdlp_check_in: the PdhgState and SolveCtl scalars of one device check (b200pdlp_check_device)"""
    _fields_ = [("iter", C.c_int32), ("step_iter", C.c_int32), ("adaptive", C.c_int32), ("pending", C.c_int32),
                ("beta", C.c_double), ("tau", C.c_double), ("sigma", C.c_double), ("sum_step", C.c_double),
                ("w_pending", C.c_double), ("tol_p", C.c_double), ("tol_d", C.c_double), ("tol_gap", C.c_double),
                ("iter_limit", C.c_int32), ("interval", C.c_int32), ("restart_on", C.c_int32), ("time_flag", C.c_int32),
                ("pf_lr", C.c_double), ("df_lr", C.c_double), ("gap_lr", C.c_double), ("pf_lc", C.c_double),
                ("df_lc", C.c_double), ("gap_lc", C.c_double), ("last_restart_iter", C.c_int32), ("light", C.c_int32)]


class CCheckOut(C.Structure):
    """b200pdlp_check_out: what one device check leaves behind"""
    _fields_ = [("sums", C.c_double * 28), ("res", (C.c_double * 10) * 2), ("term", C.c_int32), ("term_iterate", C.c_int32),
                ("restart_choice", C.c_int32), ("restarts", C.c_int32), ("checks", C.c_int32), ("trace_len", C.c_int32),
                ("done", C.c_int32), ("stop_iter", C.c_int32), ("pending", C.c_int32), ("pow_base", C.c_int32),
                ("pf_lr", C.c_double), ("df_lr", C.c_double), ("gap_lr", C.c_double), ("pf_lc", C.c_double),
                ("df_lc", C.c_double), ("gap_lc", C.c_double), ("last_restart_iter", C.c_int32), ("reserved", C.c_int32),
                ("beta", C.c_double), ("tau", C.c_double), ("sigma", C.c_double), ("eta", C.c_double), ("tau_try", C.c_double),
                ("sigma_try", C.c_double), ("sum_step", C.c_double), ("restart_sq", C.c_double * 2),
                ("pow_red", C.c_double * 128), ("pow_grow", C.c_double * 128), ("trace", C.c_double * 16)]


class CPassOut(C.Structure):
    """b200pdlp_pass_out: K4's sums and the sizes of what b200pdlp_pass_partials returned"""
    _fields_ = [("dx2", C.c_double), ("dy2", C.c_double), ("inter", C.c_double), ("slots", C.c_int32 * 3),
                ("long_a", C.c_int32), ("long_at", C.c_int32)]


CHECK_VECTORS = ("x", "y", "ax", "aty", "xsum", "ysum", "xlr", "ylr", "axsum", "atysum", "xavg", "yavg", "axavg", "atyavg")
RESIDUAL_NAMES = ("pobj", "dobj", "pfeas", "dfeas", "gap", "relgap", "pinf_obj", "pinf_res", "dinf_obj", "dinf_res")


class CWarm(C.Structure):
    _fields_ = [("col_value", _dp), ("row_value", _dp), ("row_dual", _dp)]


class CResult(C.Structure):
    _fields_ = [("col_value", _dp), ("col_dual", _dp), ("row_value", _dp), ("row_dual", _dp),
                ("value_valid", C.c_int32), ("dual_valid", C.c_int32), ("term_code", C.c_int32),
                ("term_iterate", C.c_int32), ("iters", C.c_int32), ("passes", C.c_int32),
                ("restarts", C.c_int32), ("kernel_launches", C.c_int32),
                ("primal_obj", C.c_double), ("dual_obj", C.c_double), ("primal_feas", C.c_double),
                ("dual_feas", C.c_double), ("gap", C.c_double), ("rel_gap", C.c_double),
                ("setup_seconds", C.c_double), ("solve_seconds", C.c_double), ("iter_device_ms", C.c_double), ("loop_device_ms", C.c_double),
                ("form_cols", C.c_int32), ("form_rows", C.c_int32), ("form_nnz", C.c_int32),
                ("form_neq", C.c_int32), ("trace", _dp), ("trace_cap", C.c_int32), ("trace_len", C.c_int32)]


# every symbol include/b200pdlp.h declares (tests/test_abi.py checks the library exports them all)
ABI_SYMBOLS = [
    "b200pdlp_default_params", "b200pdlp_solve", "b200pdlp_problem_create", "b200pdlp_problem_destroy",
    "b200pdlp_problem_dims", "b200pdlp_problem_get_vector", "b200pdlp_problem_get_csr", "b200pdlp_spmv_ax",
    "b200pdlp_spmv_aty", "b200pdlp_bench_spmv", "b200pdlp_bench_pass", "b200pdlp_p2p_export", "b200pdlp_p2p_import", "b200pdlp_p2p_timeline", "b200pdlp_p2p_release", "b200pdlp_problem_solve", "b200pdlp_nccl_unique_id",
    "b200pdlp_comm_init", "b200pdlp_partition_rows", "b200pdlp_last_error", "b200pdlp_version",
    "b200pdlp_device_count", "b200pdlp_form_create", "b200pdlp_form_destroy", "b200pdlp_form_dims",
    "b200pdlp_form_get_vector", "b200pdlp_form_get_csc", "b200pdlp_form_get_csr", "b200pdlp_form_get_row_map",
    "b200pdlp_form_layout_eval", "b200pdlp_p2p_link_local", "b200pdlp_solve_multi",
    "b200pdlp_hipdlp_form_create", "b200pdlp_hipdlp_power_method", "b200pdlp_hipdlp_default_params",
    "b200pdlp_solve_hipdlp", "b200pdlp_solve_hipdlp_multi", "b200pdlp_hipdlp_shard_layout_eval",
    "b200pdlp_hipdlp_controller_replay", "b200pdlp_debug_prep_compare",
    "b200pdlp_debug_prep_compare_hipdlp", "b200pdlp_debug_hipdlp_shard_prep_compare", "b200pdlp_release_cache",
    "b200pdlp_host_register", "b200pdlp_host_unregister", "b200pdlp_primal_step", "b200pdlp_dual_step", "b200pdlp_residuals",
    "b200pdlp_kkt_check", "b200pdlp_kkt_check_host", "b200pdlp_kkt_default_tolerances", "b200pdlp_solve_batch",
    "b200pdlp_solve_hipdlp_batch", "b200pdlp_solve_batch_device", "b200pdlp_debug_batch_prep_compare",
    "b200pdlp_solve_hipdlp_batch_device", "b200pdlp_debug_hipdlp_batch_prep_compare", "b200pdlp_kkt_check_batch",
    "b200pdlp_kkt_check_batch_device", "b200pdlp_hipdlp_problem_create", "b200pdlp_hipdlp_step", "b200pdlp_hipdlp_check",
    "b200pdlp_hipdlp_problem_power_method", "b200pdlp_solve_hipdlp_batch_mixed",
    "b200pdlp_solve_hipdlp_batch_mixed_device", "b200pdlp_debug_hipdlp_tree_prep_compare", "b200pdlp_check_device",
    "b200pdlp_solve_device", "b200pdlp_solve_hipdlp_device", "b200pdlp_pass_partials",
]
HIP_TRACE_COLS = 16   # B200PDLP_HIP_TRACE_COLS: the per-block trace of the HiPDLP solves

_lib = None


def _preload_nccl():
    """The engine binds NCCL at run time by SONAME (dlopen "libnccl.so.2").  If PyTorch's bundled,
    newer NCCL is installed, load THAT copy first so that the engine and a later `import torch` share
    one NCCL (the system libnccl lacks symbols torch needs)."""
    import importlib.util
    import sys
    if "torch" in sys.modules:
        return
    try:
        spec = importlib.util.find_spec("nvidia.nccl")
        if spec and spec.submodule_search_locations:
            cand = os.path.join(list(spec.submodule_search_locations)[0], "lib", "libnccl.so.2")
            if os.path.exists(cand):
                C.CDLL(cand, mode=C.RTLD_GLOBAL)
    except Exception:
        pass


def lib():
    """Load the CUDA extension; raise loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EngineError(f"{LIB_PATH} is missing: run `python -m highs_b200.build` (nvcc, sm_90a). "
                              "There is no CPU fallback.")
        _preload_nccl()
        L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        L.b200pdlp_last_error.restype = C.c_char_p
        L.b200pdlp_default_params.argtypes = [C.POINTER(CParams)]
        L.b200pdlp_default_params.restype = None
        L.b200pdlp_solve.argtypes = [C.POINTER(CLp), C.POINTER(CParams), C.POINTER(CWarm), C.POINTER(CResult)]
        L.b200pdlp_solve_batch.argtypes = [C.c_int32, C.POINTER(CLp), C.POINTER(CParams), C.POINTER(CWarm), C.POINTER(CResult)]
        L.b200pdlp_problem_create.argtypes = [C.POINTER(CLp), C.POINTER(CParams), C.c_int32, C.c_int32,
                                              C.POINTER(C.c_void_p)]
        L.b200pdlp_problem_destroy.argtypes = [C.c_void_p]
        L.b200pdlp_problem_destroy.restype = None
        L.b200pdlp_problem_dims.argtypes = [C.c_void_p, _ip]
        L.b200pdlp_problem_get_vector.argtypes = [C.c_void_p, C.c_int32, _dp, C.c_int32]
        L.b200pdlp_problem_get_csr.argtypes = [C.c_void_p, _ip, _ip, _dp]
        L.b200pdlp_spmv_ax.argtypes = [C.c_void_p, _dp, _dp]
        L.b200pdlp_spmv_aty.argtypes = [C.c_void_p, _dp, _dp]
        L.b200pdlp_bench_spmv.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_float)]
        L.b200pdlp_bench_pass.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_float)]
        L.b200pdlp_problem_solve.argtypes = [C.c_void_p, C.POINTER(CParams), C.POINTER(CWarm), C.POINTER(CResult)]
        L.b200pdlp_nccl_unique_id.argtypes = [C.POINTER(C.c_uint8)]
        L.b200pdlp_comm_init.argtypes = [C.c_void_p, C.POINTER(C.c_uint8)]
        L.b200pdlp_p2p_export.argtypes = [C.c_void_p, C.POINTER(C.c_uint8)]
        L.b200pdlp_p2p_import.argtypes = [C.c_void_p, C.POINTER(C.c_uint8)]
        L.b200pdlp_p2p_timeline.argtypes = [C.c_void_p, _dp]
        L.b200pdlp_p2p_release.argtypes = [C.c_void_p]
        L.b200pdlp_p2p_link_local.argtypes = [C.POINTER(C.c_void_p), C.c_int32]
        L.b200pdlp_partition_rows.argtypes = [C.POINTER(CLp), C.c_int32, _ip]
        L.b200pdlp_form_create.argtypes = [C.POINTER(CLp), C.c_int32, C.POINTER(C.c_void_p)]
        L.b200pdlp_form_destroy.argtypes = [C.c_void_p]
        L.b200pdlp_form_destroy.restype = None
        L.b200pdlp_form_dims.argtypes = [C.c_void_p, _ip, _dp]
        L.b200pdlp_form_get_vector.argtypes = [C.c_void_p, C.c_int32, _dp, C.c_int32]
        L.b200pdlp_form_get_csc.argtypes = [C.c_void_p, _ip, _ip, _dp]
        L.b200pdlp_form_get_row_map.argtypes = [C.c_void_p, _ip, _ip]
        L.b200pdlp_form_get_csr.argtypes = [C.c_void_p, _ip, _ip, _dp]
        L.b200pdlp_form_layout_eval.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, _dp, _dp, _dp, _dp, _dp]
        L.b200pdlp_debug_prep_compare.argtypes = [C.POINTER(CLp), C.c_int32, _dp]
        L.b200pdlp_release_cache.argtypes = []
        L.b200pdlp_release_cache.restype = None
        L.b200pdlp_host_register.argtypes = [C.c_void_p, C.c_size_t]
        L.b200pdlp_host_unregister.argtypes = [C.c_void_p]
        L.b200pdlp_primal_step.argtypes = [C.c_void_p, _dp, _dp, C.c_double, _dp, _dp]
        L.b200pdlp_dual_step.argtypes = [C.c_void_p, _dp, _dp, _dp, C.c_double, _dp, _dp, _dp]
        L.b200pdlp_residuals.argtypes = [C.c_void_p, _dp, _dp, _dp]
        L.b200pdlp_check_device.argtypes = [C.c_void_p, C.POINTER(CCheckIn)] + [_dp] * 14 + [C.POINTER(CCheckOut)]
        L.b200pdlp_pass_partials.argtypes = ([C.c_void_p] + [_dp] * 4 + [C.c_double] * 2 + [_dp] * 5 +
                                             [C.c_int32, _ip, C.c_int32, C.POINTER(CPassOut)])
        _lib = L
    return _lib


def _check(rc: int, what: str):
    if rc != 0:
        raise EngineError(f"{what} failed ({rc}): {lib().b200pdlp_last_error().decode()}")


def _p(a, t):
    return a.ctypes.data_as(t)


def make_clp(lp: HighsLp):
    a = lp.a_matrix_
    keep = (a.start_, a.index_, a.value_, lp.col_cost_, lp.col_lower_, lp.col_upper_, lp.row_lower_, lp.row_upper_)
    c = CLp(lp.num_col_, lp.num_row_, _p(a.start_, _ip), _p(a.index_, _ip), _p(a.value_, _dp), _p(lp.col_cost_, _dp),
            _p(lp.col_lower_, _dp), _p(lp.col_upper_, _dp), _p(lp.row_lower_, _dp), _p(lp.row_upper_, _dp),
            float(lp.sense_), float(lp.offset_))
    return c, keep


def make_params(**kw) -> CParams:
    p = CParams()
    lib().b200pdlp_default_params(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise TypeError(f"unknown parameter {k}")
        setattr(p, k, v)
    return p


def _result_dict(res: CResult, arrays) -> dict:
    cv, cd, rv, rd = arrays[:4]
    skip = ("col_value", "col_dual", "row_value", "row_dual", "trace")
    out = {k: getattr(res, k) for k, _ in CResult._fields_ if k not in skip}
    out.update(col_value=cv, col_dual=cd, row_value=rv, row_dual=rd, term_name=TERM_NAMES.get(res.term_code, "?"))
    if len(arrays) > 4:
        out["trace"] = arrays[4][: res.trace_len].copy()
    return out


def _mk_result(lp: HighsLp, trace_cap: int = 0):
    n, m = lp.num_col_, lp.num_row_
    arrays = (np.zeros(n), np.zeros(n), np.zeros(m), np.zeros(m))
    res = CResult()
    res.col_value, res.col_dual, res.row_value, res.row_dual = (_p(a, _dp) for a in arrays)
    if trace_cap > 0:
        tr = np.zeros((trace_cap, 16))
        res.trace, res.trace_cap = _p(tr, _dp), trace_cap
        arrays = arrays + (tr,)
    return res, arrays


def _mk_warm(warm):
    if warm is None:
        return None, None
    arrs = tuple(np.ascontiguousarray(w, dtype=np.float64) for w in warm)  # (col_value, row_value, row_dual)
    return CWarm(_p(arrs[0], _dp), _p(arrs[1], _dp), _p(arrs[2], _dp)), arrs


def solve(lp: HighsLp, warm=None, trace_cap: int = 0, out_arrays=None, **params) -> dict:
    """b200pdlp_solve: host buffers in, host buffers out (prologue + upload + PDHG + download).
    out_arrays = (col_value, col_dual, row_value, row_dual): caller-owned (e.g. page-locked) result storage."""
    L = lib()
    clp, keep = make_clp(lp)
    prm = make_params(**params)
    res, arrays = _mk_result(lp, trace_cap)
    if out_arrays is not None:
        arrays = tuple(out_arrays) + arrays[4:]
        res.col_value, res.col_dual, res.row_value, res.row_dual = (_p(a, _dp) for a in arrays[:4])
    w, wk = _mk_warm(warm)
    _check(L.b200pdlp_solve(C.byref(clp), C.byref(prm), C.byref(w) if w else None, C.byref(res)), "b200pdlp_solve")
    return _result_dict(res, arrays)


def solve_batch(lps, warms=None, trace_cap: int = 0, **params) -> list:
    """b200pdlp_solve_batch: every LP of `lps` (ordered-mode problems) solved on one GPU in one call, one CTA per LP.
    warms: None, or one entry per LP -- None (cold start) or (col_value, row_value, row_dual).  Returns the dicts solve()
    returns, in order; each holds the bits solve() returns for that LP alone (the timings and kernel_launches are the
    batch's)."""
    lps = list(lps)
    if warms is not None:
        warms = list(warms)
        if len(warms) != len(lps):
            raise ValueError(f"solve_batch: {len(warms)} warm starts for {len(lps)} LPs")
    L = lib()
    count = len(lps)
    clps, cres, keep, arrays = (CLp * max(count, 1))(), (CResult * max(count, 1))(), [], []
    cwarm = (CWarm * max(count, 1))() if warms is not None and any(w is not None for w in warms) else None
    for i, lp in enumerate(lps):
        clps[i], k = make_clp(lp)
        keep.append(k)
        cres[i], a = _mk_result(lp, trace_cap)
        arrays.append(a)
        if cwarm is not None and warms[i] is not None:
            cwarm[i], wk = _mk_warm(warms[i])
            keep.append(wk)
    prm = make_params(**params)
    _check(L.b200pdlp_solve_batch(count, clps, C.byref(prm), cwarm, cres), "b200pdlp_solve_batch")
    return [_result_dict(cres[i], arrays[i]) for i in range(count)]


_LP_INDEX_ARRAYS = ("a_start", "a_index")
_LP_VALUE_ARRAYS = ("a_value", "col_cost", "col_lower", "col_upper", "row_lower", "row_upper")


def lp_to_device(lp: HighsLp, device: int = 0) -> dict:
    """The arrays of `lp` as torch CUDA tensors on `device` (int32 indices, float64 values), with num_col, num_row, sense and
    offset: one member of solve_batch_device."""
    import torch
    dev = torch.device("cuda", device)
    arrs = dict(zip(_LP_INDEX_ARRAYS + _LP_VALUE_ARRAYS, lp_arrays(lp)))
    out = {k: torch.as_tensor(np.ascontiguousarray(v, dtype=np.int32 if k in _LP_INDEX_ARRAYS else np.float64)).to(dev)
           for k, v in arrs.items()}
    out.update(num_col=int(lp.num_col_), num_row=int(lp.num_row_), sense=float(lp.sense_), offset=float(lp.offset_))
    return out


def _dev_ptr(t, dtype, ptype, what):
    """the device address of a contiguous CUDA tensor of `dtype` (NULL when empty)"""
    if t is None:
        return None
    if not (t.is_cuda and t.dtype == dtype and t.is_contiguous()):
        raise TypeError(f"{what} must be a contiguous CUDA tensor of {dtype}")
    return C.cast(C.c_void_p(t.data_ptr() if t.numel() else 0), ptype)


def make_clp_device(d: dict) -> CLp:
    """the b200pdlp_lp of an lp_to_device dict: every array pointer is device memory"""
    import torch
    ptrs = [_dev_ptr(d[k], torch.int32, _ip, k) for k in _LP_INDEX_ARRAYS] + \
           [_dev_ptr(d[k], torch.float64, _dp, k) for k in _LP_VALUE_ARRAYS]
    return CLp(d["num_col"], d["num_row"], *ptrs, float(d["sense"]), float(d["offset"]))


def solve_batch_device(dlps, warms=None, trace_cap: int = 0, **params) -> list:
    """b200pdlp_solve_batch_device: solve_batch for LPs already in GPU memory (dicts of lp_to_device), prologue and postsolve
    on the device.  warms: None, or one entry per LP -- None or (col_value, row_value, row_dual) as float64 CUDA tensors.
    Returns the dicts solve_batch returns, with the four vectors as float64 CUDA tensors; each member's bits are those
    solve_batch returns for it.  `device` defaults to the device of the first LP's tensors.  torch's current stream is
    synchronised first, so that inputs it is still writing are complete."""
    dlps = list(dlps)
    if warms is not None:
        warms = list(warms)
        if len(warms) != len(dlps):
            raise ValueError(f"solve_batch_device: {len(warms)} warm starts for {len(dlps)} LPs")
    L = lib()
    L.b200pdlp_solve_batch_device.argtypes = [C.c_int32, C.POINTER(CLp), C.POINTER(CParams), C.POINTER(CWarm), C.POINTER(CResult)]
    count = len(dlps)
    if count == 0:
        _check(L.b200pdlp_solve_batch_device(0, None, C.byref(make_params(**params)), None, None), "b200pdlp_solve_batch_device")
        return []
    import torch
    dev = dlps[0]["a_start"].device
    params.setdefault("device", dev.index)
    prm = make_params(**params)
    dev = torch.device("cuda", prm.device if prm.device >= 0 else torch.cuda.current_device())
    clps, cres, arrays = (CLp * count)(), (CResult * count)(), []
    cwarm = (CWarm * count)() if warms is not None and any(w is not None for w in warms) else None
    for i, d in enumerate(dlps):
        clps[i] = make_clp_device(d)
        vecs = (torch.empty(d["num_col"], dtype=torch.float64, device=dev), torch.empty(d["num_col"], dtype=torch.float64, device=dev),
                torch.empty(d["num_row"], dtype=torch.float64, device=dev), torch.empty(d["num_row"], dtype=torch.float64, device=dev))
        res = CResult()
        res.col_value, res.col_dual, res.row_value, res.row_dual = (_dev_ptr(v, torch.float64, _dp, "result") for v in vecs)
        if trace_cap > 0:
            tr = np.zeros((trace_cap, 16))
            res.trace, res.trace_cap = _p(tr, _dp), trace_cap
            vecs = vecs + (tr,)
        cres[i] = res
        arrays.append(vecs)
        if cwarm is not None and warms[i] is not None:
            cwarm[i] = CWarm(*(_dev_ptr(w, torch.float64, _dp, "warm start") for w in warms[i]))
    torch.cuda.current_stream(dev).synchronize()
    _check(L.b200pdlp_solve_batch_device(count, clps, C.byref(prm), cwarm, cres), "b200pdlp_solve_batch_device")
    return [_result_dict(cres[i], arrays[i]) for i in range(count)]


def _device_result(d: dict, dev, trace_cap: int, trace_cols: int):
    """a CResult whose four vectors are new float64 CUDA tensors on `dev` for the LP of lp_to_device dict `d` (at least one
    element each, so that an LP without rows or columns still gets four non-NULL vectors), with a host trace array of
    trace_cap rows; and the arrays the result dict returns"""
    import torch
    n, m = d["num_col"], d["num_row"]
    vecs = [torch.empty(max(k, 1), dtype=torch.float64, device=dev) for k in (n, n, m, m)]
    res = CResult()
    res.col_value, res.col_dual, res.row_value, res.row_dual = (_dev_ptr(v, torch.float64, _dp, "result") for v in vecs)
    out = tuple(v[:k] for v, k in zip(vecs, (n, n, m, m)))
    if trace_cap > 0:
        tr = np.zeros((trace_cap, trace_cols))
        res.trace, res.trace_cap = _p(tr, _dp), trace_cap
        out = out + (tr,)
    return res, out


def solve_device(dlp: dict, warm=None, trace_cap: int = 0, **params) -> dict:
    """b200pdlp_solve_device: solve() for an LP already in GPU memory (a dict of lp_to_device), at any size.  warm: None or
    (col_value, row_value, row_dual) as float64 CUDA tensors.  Returns the dict solve() returns for host copies of the same
    arrays, bit for bit, with the four vectors as float64 CUDA tensors (kkt_check_batch_device takes them as they are).  A
    tree-mode LP's prologue reads the tensors in place; an ordered-mode LP is solved as a batch of one (solve_batch_device),
    whose timings and kernel_launches it returns.  `device` defaults to the device of the LP's tensors; torch's current
    stream is synchronised first, so that inputs it is still writing are complete."""
    import torch
    L = lib()
    L.b200pdlp_solve_device.argtypes = [C.POINTER(CLp), C.POINTER(CParams), C.POINTER(CWarm), C.POINTER(CResult)]
    params.setdefault("device", dlp["a_start"].device.index)
    prm = make_params(**params)
    dev = torch.device("cuda", prm.device if prm.device >= 0 else torch.cuda.current_device())
    clp = make_clp_device(dlp)
    res, arrays = _device_result(dlp, dev, trace_cap, 16)
    cw = None
    if warm is not None:   # (an empty vector gets one element: a NULL pointer would mean a cold start)
        keep = [w if w.numel() else torch.zeros(1, dtype=torch.float64, device=dev) for w in warm]
        cw = CWarm(*(_dev_ptr(w, torch.float64, _dp, "warm start") for w in keep))
    torch.cuda.current_stream(dev).synchronize()
    _check(L.b200pdlp_solve_device(C.byref(clp), C.byref(prm), C.byref(cw) if cw else None, C.byref(res)),
           "b200pdlp_solve_device")
    return _result_dict(res, arrays)


def _prep_compare(name: str, items, lps, *ints) -> list:
    """the call of a batch prologue comparison `name` on host LPs, with the int arguments `ints`: one dict of mismatch counts
    per LP (`items`)"""
    lps = list(lps)
    fn = getattr(lib(), name)
    fn.argtypes = [C.c_int32, C.POINTER(CLp)] + [C.c_int32] * len(ints) + [_dp]
    count = len(lps)
    clps, keep = (CLp * max(count, 1))(), []
    for i, lp in enumerate(lps):
        clps[i], k = make_clp(lp)
        keep.append(k)
    k = len(items)
    rep = np.zeros(max(count, 1) * k)
    _check(fn(count, clps, *ints, _p(rep, _dp)), name)
    return [dict(zip(items, rep[k * i:k * (i + 1)].tolist())) for i in range(count)]


BATCH_PREP_ITEMS = ["dims", "cost", "lower", "upper", "rhs", "col_scale", "row_scale", "row_new_idx", "row_class", "A.slices",
                    "A.col", "A.val", "AT.slices", "AT.col", "AT.val", "x0", "y0", "xsum", "norm_cost", "norm_rhs", "amax",
                    "beta_cost_sq", "beta_rhs_sq", "col_value", "col_dual", "row_value", "row_dual"]


def batch_prep_compare(lps, scaling: int = 1) -> list:
    """b200pdlp_debug_batch_prep_compare: the device prologue and postsolve of solve_batch_device against their host twins on
    host LPs; one dict of mismatch counts per LP (BATCH_PREP_ITEMS)."""
    return _prep_compare("b200pdlp_debug_batch_prep_compare", BATCH_PREP_ITEMS, lps, scaling)


PREP_ITEMS = ["n", "m", "nnz", "neq", "cbeg", "cidx", "cval", "cost", "lower", "upper", "col_scale", "rhs", "row_scale", "rptr",
              "rpos", "row_new_idx", "row_class", "rperm", "cperm", "A.slices", "A.col", "A.val", "AT.slices", "AT.col", "AT.val",
              "A.long", "AT.long", "amax", "norm_cost_relerr", "norm_rhs_relerr", "device_order_vectors", "cols_sorted"]


def prep_compare(lp: HighsLp, scaling: int = 1) -> dict:
    """b200pdlp_debug_prep_compare: the device-resident prologue against its host twin, mismatches per array."""
    clp, keep = make_clp(lp)
    rep = np.zeros(32)
    _check(lib().b200pdlp_debug_prep_compare(C.byref(clp), scaling, _p(rep, _dp)), "b200pdlp_debug_prep_compare")
    return dict(zip(PREP_ITEMS, rep.tolist()))


PREP_ITEMS_HIPDLP = PREP_ITEMS[:28] + ["norm_cost_bits", "norm_rhs_bits"] + PREP_ITEMS[30:] + [
    "row_upper", "row_upper_device_order", "orig_row_ptr", "orig_row_entries", "scaled", "unused37", "unused38", "unused39"]


def prep_compare_hipdlp(lp: HighsLp, scaling_mode: int = 5, ruiz_iterations: int = 10) -> dict:
    """b200pdlp_debug_prep_compare_hipdlp: the HiPDLP mode's device prologue against its host twin, mismatches per array."""
    L = lib()
    L.b200pdlp_debug_prep_compare_hipdlp.argtypes = [C.POINTER(CLp), C.c_int32, C.c_int32, _dp]
    clp, keep = make_clp(lp)
    rep = np.zeros(40)
    _check(L.b200pdlp_debug_prep_compare_hipdlp(C.byref(clp), scaling_mode, ruiz_iterations, _p(rep, _dp)),
           "b200pdlp_debug_prep_compare_hipdlp")
    return dict(zip(PREP_ITEMS_HIPDLP, rep.tolist()))


SHARD_PREP_ITEMS = ["dims", "device_order_vectors", "row_upper_device_order", "norm_cost_bits", "norm_rhs_bits", "scaled",
                    "orderings", "unused7"]
SHARD_PREP_RANK_ITEMS = ["bounds", "A.slices", "A.col", "A.val", "A.long", "AT.slices", "AT.col", "AT.val", "AT.long"]


def hipdlp_shard_prep_compare(lp: HighsLp, world: int, scaling_mode: int = 5, ruiz_iterations: int = 10) -> dict:
    """b200pdlp_debug_hipdlp_shard_prep_compare: the device prologue of solve_hipdlp_multi (every rank's A_g and A_g' on the
    current device) against the host prologue and build_hipdlp_shard, mismatches per array; "ranks" holds one dict per rank."""
    L = lib()
    L.b200pdlp_debug_hipdlp_shard_prep_compare.argtypes = [C.POINTER(CLp), C.c_int32, C.c_int32, C.c_int32, _dp]
    clp, keep = make_clp(lp)
    rep = np.zeros(8 + 9 * max(world, 1))
    _check(L.b200pdlp_debug_hipdlp_shard_prep_compare(C.byref(clp), scaling_mode, ruiz_iterations, world, _p(rep, _dp)),
           "b200pdlp_debug_hipdlp_shard_prep_compare")
    out = dict(zip(SHARD_PREP_ITEMS, rep[:8].tolist()))
    out["ranks"] = [dict(zip(SHARD_PREP_RANK_ITEMS, rep[8 + 9 * g:17 + 9 * g].tolist())) for g in range(world)]
    return out


def lp_arrays(lp: HighsLp):
    a = lp.a_matrix_
    return [a.start_, a.index_, a.value_, lp.col_cost_, lp.col_lower_, lp.col_upper_, lp.row_lower_, lp.row_upper_]


def pin_arrays(arrays) -> list:
    """cudaHostRegister the given numpy arrays (b200pdlp_host_register); returns the ones that were pinned."""
    done = []
    for a in arrays:
        if a.nbytes and lib().b200pdlp_host_register(a.ctypes.data_as(C.c_void_p), a.nbytes) == 0:
            done.append(a)
    return done


def unpin_arrays(arrays):
    for a in arrays:
        lib().b200pdlp_host_unregister(a.ctypes.data_as(C.c_void_p))


class CKktTolerances(C.Structure):
    _fields_ = [(k, C.c_double) for k in ("primal_feasibility_tolerance", "dual_feasibility_tolerance", "primal_residual_tolerance",
                                          "dual_residual_tolerance", "optimality_tolerance")]


class CKktInfo(C.Structure):
    _fields_ = ([(k, C.c_double) for k in (
        "objective_function_value", "dual_objective_value", "primal_dual_objective_error", "max_primal_infeasibility",
        "sum_primal_infeasibilities", "max_dual_infeasibility", "sum_dual_infeasibilities", "max_relative_primal_infeasibility",
        "max_relative_dual_infeasibility", "max_primal_residual_error", "max_dual_residual_error",
        "max_relative_primal_residual_error", "max_relative_dual_residual_error", "max_complementarity_violation",
        "norm_bounds", "norm_costs")] + [(k, C.c_int32) for k in (
            "num_primal_infeasibilities", "num_dual_infeasibilities", "num_relative_primal_infeasibilities",
            "num_relative_dual_infeasibilities", "num_primal_residual_errors", "num_dual_residual_errors",
            "num_relative_primal_residual_errors", "num_relative_dual_residual_errors", "num_complementarity_violations",
            "primal_solution_status", "dual_solution_status", "model_status")])


class CSolution(C.Structure):
    _fields_ = [("col_value", _dp), ("col_dual", _dp), ("row_value", _dp), ("row_dual", _dp)]


_SOLUTION_VECTORS = ("col_value", "col_dual", "row_value", "row_dual")


def _kkt_tolerances(kkt_tolerance: float) -> CKktTolerances:
    L = lib()
    tol = CKktTolerances()
    L.b200pdlp_kkt_default_tolerances.argtypes = [C.POINTER(CKktTolerances), C.c_double]
    L.b200pdlp_kkt_default_tolerances.restype = None
    L.b200pdlp_kkt_default_tolerances(C.byref(tol), float(kkt_tolerance))
    return tol


def kkt_check(lp: HighsLp, solution, kkt_tolerance: float = 0.0, model_status: int = 7, on_device: bool = True) -> dict:
    """lpKktCheck of a HighsSolution (b200pdlp_kkt_check on the GPU, b200pdlp_kkt_check_host = its host twin).
    `solution`: mapping with col_value, col_dual, row_value, row_dual; model_status: HighsModelStatus code from the solver."""
    L = lib()
    clp, keep = make_clp(lp)
    tol = _kkt_tolerances(kkt_tolerance)
    info = CKktInfo()
    info.model_status = int(model_status)
    arrs = [np.ascontiguousarray(solution[k], dtype=np.float64) for k in _SOLUTION_VECTORS]
    fn = L.b200pdlp_kkt_check if on_device else L.b200pdlp_kkt_check_host
    fn.argtypes = [C.POINTER(CLp), _dp, _dp, _dp, _dp, C.POINTER(CKktTolerances), C.POINTER(CKktInfo)]
    rc = fn(C.byref(clp), *(_p(a, _dp) for a in arrs), C.byref(tol), C.byref(info))
    if rc != 0:
        raise EngineError(f"b200pdlp_kkt_check{'_host' if not on_device else ''} failed ({rc})")
    return {k: getattr(info, k) for k, _ in CKktInfo._fields_}


def _kkt_statuses(model_status, count: int, what: str) -> list:
    """model_status (one int, or one per LP) as a list of `count` ints"""
    if isinstance(model_status, (int, np.integer)):
        return [int(model_status)] * count
    statuses = [int(s) for s in model_status]
    if len(statuses) != count:
        raise ValueError(f"{what}: {len(statuses)} model statuses for {count} LPs")
    return statuses


def _kkt_batch_call(name: str, count: int, clps, csols, kkt_tolerance: float, statuses, device: int) -> list:
    L = lib()
    fn = getattr(L, name)
    fn.argtypes = [C.c_int32, C.POINTER(CLp), C.POINTER(CSolution), C.POINTER(CKktTolerances), C.c_int32, C.POINTER(CKktInfo)]
    infos = (CKktInfo * max(count, 1))()
    for i, s in enumerate(statuses):
        infos[i].model_status = s
    _check(fn(count, clps, csols, C.byref(_kkt_tolerances(kkt_tolerance)), device, infos), name)
    return [{k: getattr(infos[i], k) for k, _ in CKktInfo._fields_} for i in range(count)]


def kkt_check_batch(lps, sols, kkt_tolerance: float = 0.0, model_status=7, device: int = -1) -> list:
    """b200pdlp_kkt_check_batch: kkt_check for every (LP, solution) pair in one call on one GPU, one CTA per LP.  `sols`:
    mappings holding the four vectors as numpy arrays (the dicts of solve_batch and solve_hipdlp_batch work as they are);
    model_status: one HighsModelStatus code for all, or one per LP.  Returns the dicts kkt_check returns, in order; each
    equals kkt_check(lp, sol, on_device=False) for that pair, bit for bit (any NaN matching any NaN)."""
    lps, sols = list(lps), list(sols)
    if len(sols) != len(lps):
        raise ValueError(f"kkt_check_batch: {len(sols)} solutions for {len(lps)} LPs")
    count = len(lps)
    statuses = _kkt_statuses(model_status, count, "kkt_check_batch")
    clps, csols, keep = (CLp * max(count, 1))(), (CSolution * max(count, 1))(), []
    for i, (lp, sol) in enumerate(zip(lps, sols)):
        clps[i], k = make_clp(lp)
        arrs = [np.ascontiguousarray(sol[v], dtype=np.float64) for v in _SOLUTION_VECTORS]
        csols[i] = CSolution(*(_p(a, _dp) for a in arrs))
        keep += [k, arrs]
    return _kkt_batch_call("b200pdlp_kkt_check_batch", count, clps, csols, kkt_tolerance, statuses, device)


def kkt_check_batch_device(dlps, sols, kkt_tolerance: float = 0.0, model_status=7) -> list:
    """b200pdlp_kkt_check_batch_device: kkt_check_batch for LPs and solutions already in GPU memory -- `dlps` from
    lp_to_device, `sols` mappings holding the four vectors as float64 CUDA tensors (the dicts of solve_batch_device and
    solve_hipdlp_batch_device work as they are).  The device is that of the tensors.  torch's current stream is synchronised
    first, so that inputs it is still writing are complete.  Returns the dicts kkt_check_batch returns."""
    dlps, sols = list(dlps), list(sols)
    if len(sols) != len(dlps):
        raise ValueError(f"kkt_check_batch_device: {len(sols)} solutions for {len(dlps)} LPs")
    count = len(dlps)
    statuses = _kkt_statuses(model_status, count, "kkt_check_batch_device")
    if count == 0:
        return _kkt_batch_call("b200pdlp_kkt_check_batch_device", 0, None, None, kkt_tolerance, [], -1)
    import torch
    dev = dlps[0]["a_start"].device
    clps, csols = (CLp * count)(), (CSolution * count)()
    for i, (d, sol) in enumerate(zip(dlps, sols)):
        clps[i] = make_clp_device(d)
        csols[i] = CSolution(*(_dev_ptr(sol[v], torch.float64, _dp, v) for v in _SOLUTION_VECTORS))
    torch.cuda.current_stream(dev).synchronize()
    return _kkt_batch_call("b200pdlp_kkt_check_batch_device", count, clps, csols, kkt_tolerance, statuses, dev.index)


def hipdlp_controller_replay(norm_cost, norm_rhs, op_norm_sq, tolerance, strategy, sums, restart_sums) -> np.ndarray:
    """Host-only: replay the HiPDLP host control over recorded per-block sums (b200pdlp_hipdlp_controller_replay)."""
    L = lib()
    L.b200pdlp_hipdlp_controller_replay.argtypes = [C.c_double, C.c_double, C.c_double, C.c_double, C.c_int32, C.c_int32, _dp, _dp, _dp]
    sums = np.ascontiguousarray(sums, dtype=np.float64).reshape(-1, 9)
    rs = np.ascontiguousarray(restart_sums, dtype=np.float64).reshape(-1, 3)
    nb = sums.shape[0]
    out = np.zeros((max(nb, 1), 8))
    _check(L.b200pdlp_hipdlp_controller_replay(norm_cost, norm_rhs, op_norm_sq, tolerance, strategy, nb,
                                               _p(sums if nb else np.zeros(9), _dp), _p(rs if nb else np.zeros(3), _dp), _p(out, _dp)),
           "b200pdlp_hipdlp_controller_replay")
    return out[:nb]


def _hipdlp_params(params) -> CHipdlpParams:
    L = lib()
    L.b200pdlp_hipdlp_default_params.argtypes = [C.POINTER(CHipdlpParams)]
    L.b200pdlp_hipdlp_default_params.restype = None
    prm = CHipdlpParams()
    L.b200pdlp_hipdlp_default_params(C.byref(prm))
    for k, v in params.items():
        if not hasattr(prm, k):
            raise TypeError(f"unknown parameter {k}")
        setattr(prm, k, v)
    return prm


def solve_hipdlp(lp: HighsLp, trace_cap: int = 0, out_arrays=None, **params) -> dict:
    """b200pdlp_solve_hipdlp: the HiPDLP mode (reflected Halpern PDHG, solver=hipdlp) on one GPU; parameters are the
    HighsOptions of the same meaning (tolerance, iter_limit, scaling_mode, ruiz_iterations, step_size_strategy ...), and
    device_prep=-1 for the host prologue instead of the device-resident one.  trace_cap > 0: "trace" holds one row of
    HIP_TRACE_COLS per block of 40 steps (include/b200pdlp.h, B200PDLP_HIP_TRACE_COLS).
    out_arrays = (col_value, col_dual, row_value, row_dual): caller-owned (e.g. page-locked) result storage, as in solve()."""
    L = lib()
    L.b200pdlp_solve_hipdlp.argtypes = [C.POINTER(CLp), C.POINTER(CHipdlpParams), C.POINTER(CResult)]
    clp, keep = make_clp(lp)
    prm = _hipdlp_params(params)
    res, arrays = _mk_result(lp, trace_cap)
    if out_arrays is not None:
        arrays = tuple(out_arrays) + arrays[4:]
        res.col_value, res.col_dual, res.row_value, res.row_dual = (_p(a, _dp) for a in arrays[:4])
    _check(L.b200pdlp_solve_hipdlp(C.byref(clp), C.byref(prm), C.byref(res)), "b200pdlp_solve_hipdlp")
    return _result_dict(res, arrays)


def solve_hipdlp_device(dlp: dict, trace_cap: int = 0, **params) -> dict:
    """b200pdlp_solve_hipdlp_device: solve_hipdlp() for an LP already in GPU memory (a dict of lp_to_device), at any size.
    Returns the dict solve_hipdlp() returns for host copies of the same arrays, bit for bit, with the four vectors as
    float64 CUDA tensors.  A tree-mode LP's prologue reads the tensors in place; an ordered-mode LP is solved as a batch of
    one (solve_hipdlp_batch_mixed_device), whose timings and kernel_launches it returns.  `device` defaults to the device of
    the LP's tensors; torch's current stream is synchronised first."""
    import torch
    L = lib()
    L.b200pdlp_solve_hipdlp_device.argtypes = [C.POINTER(CLp), C.POINTER(CHipdlpParams), C.POINTER(CResult)]
    params.setdefault("device", dlp["a_start"].device.index)
    prm = _hipdlp_params(params)
    dev = torch.device("cuda", prm.device if prm.device >= 0 else torch.cuda.current_device())
    clp = make_clp_device(dlp)
    res, arrays = _device_result(dlp, dev, trace_cap, HIP_TRACE_COLS)
    torch.cuda.current_stream(dev).synchronize()
    _check(L.b200pdlp_solve_hipdlp_device(C.byref(clp), C.byref(prm), C.byref(res)), "b200pdlp_solve_hipdlp_device")
    return _result_dict(res, arrays)


def _hipdlp_batch(name: str, lps, trace_cap: int, params: dict) -> list:
    """the call of the host-array HiPDLP batch `name`: the result dicts, in order"""
    lps = list(lps)
    fn = getattr(lib(), name)
    fn.argtypes = [C.c_int32, C.POINTER(CLp), C.POINTER(CHipdlpParams), C.POINTER(CResult)]
    count = len(lps)
    clps, cres, keep, arrays = (CLp * max(count, 1))(), (CResult * max(count, 1))(), [], []
    for i, lp in enumerate(lps):
        clps[i], k = make_clp(lp)
        keep.append(k)
        cres[i], a = _mk_result(lp, trace_cap)
        arrays.append(a)
    prm = _hipdlp_params(params)
    _check(fn(count, clps, C.byref(prm), cres), name)
    return [_result_dict(cres[i], arrays[i]) for i in range(count)]


def _hipdlp_batch_device(name: str, dlps, trace_cap: int, params: dict) -> list:
    """the call of the device-array HiPDLP batch `name`: the result dicts, in order, their vectors float64 CUDA tensors"""
    dlps = list(dlps)
    fn = getattr(lib(), name)
    fn.argtypes = [C.c_int32, C.POINTER(CLp), C.POINTER(CHipdlpParams), C.POINTER(CResult)]
    count = len(dlps)
    if count == 0:
        _check(fn(0, None, C.byref(_hipdlp_params(params)), None), name)
        return []
    import torch
    if getattr(dlps[0]["a_start"], "is_cuda", False):
        params.setdefault("device", dlps[0]["a_start"].device.index)
    prm = _hipdlp_params(params)
    clps, cres, arrays = (CLp * count)(), (CResult * count)(), []
    for i, d in enumerate(dlps):
        clps[i] = make_clp_device(d)
    dev = torch.device("cuda", prm.device if prm.device >= 0 else torch.cuda.current_device())
    for i, d in enumerate(dlps):
        # at least one element each, so that an LP without rows (or columns) still gets four non-NULL vectors
        n, m = d["num_col"], d["num_row"]
        vecs = [torch.empty(max(k, 1), dtype=torch.float64, device=dev) for k in (n, n, m, m)]
        res = CResult()
        res.col_value, res.col_dual, res.row_value, res.row_dual = (_dev_ptr(v, torch.float64, _dp, "result") for v in vecs)
        out = tuple(v[:k] for v, k in zip(vecs, (n, n, m, m)))
        if trace_cap > 0:
            tr = np.zeros((trace_cap, HIP_TRACE_COLS))
            res.trace, res.trace_cap = _p(tr, _dp), trace_cap
            out = out + (tr,)
        cres[i] = res
        arrays.append(out)
    torch.cuda.current_stream(dev).synchronize()
    _check(fn(count, clps, C.byref(prm), cres), name)
    return [_result_dict(cres[i], arrays[i]) for i in range(count)]


def solve_hipdlp_batch(lps, **params) -> list:
    """b200pdlp_solve_hipdlp_batch: every LP of `lps` (ordered-mode problems under HiPDLP's classification) solved in the
    HiPDLP mode on one GPU in one call, one CTA per LP.  Takes the parameters of solve_hipdlp (device_prep is ignored) and
    returns the dicts solve_hipdlp returns, in order; each holds the bits solve_hipdlp returns for that LP alone (the timings
    and kernel_launches are the batch's)."""
    return _hipdlp_batch("b200pdlp_solve_hipdlp_batch", lps, 0, params)


def solve_hipdlp_batch_mixed(lps, trace_cap: int = 0, **params) -> list:
    """b200pdlp_solve_hipdlp_batch_mixed: solve_hipdlp_batch for LPs of any size up to max(n, m) = 262144, in any order.
    Ordered-mode members return what solve_hipdlp_batch returns for them; every other member (a tree member: one
    thread-block cluster of the GPU per LP) returns what solve_hipdlp returns for it alone, bit for bit, and with
    trace_cap > 0 its "trace" rows too.  ordered_max=-1 makes every member a tree member."""
    return _hipdlp_batch("b200pdlp_solve_hipdlp_batch_mixed", lps, trace_cap, params)


def solve_hipdlp_batch_device(dlps, **params) -> list:
    """b200pdlp_solve_hipdlp_batch_device: solve_hipdlp_batch for LPs already in GPU memory (dicts of lp_to_device), prologue
    and postsolve on the device.  Returns the dicts solve_hipdlp_batch returns, with the four vectors as float64 CUDA tensors;
    each member's bits are those solve_hipdlp_batch returns for it.  `device` defaults to the device of the first LP's
    tensors.  torch's current stream is synchronised first, so that inputs it is still writing are complete."""
    return _hipdlp_batch_device("b200pdlp_solve_hipdlp_batch_device", dlps, 0, params)


HIPDLP_BATCH_PREP_ITEMS = ["dims", "cost", "lower", "upper", "rhs", "row_upper", "col_scale", "row_scale", "row_new_idx",
                           "row_class", "A.slices", "A.col", "A.val", "AT.slices", "AT.col", "AT.val", "norm_cost", "norm_rhs",
                           "scaled", "orderings", "col_value", "col_dual", "row_value", "row_dual"]


def hipdlp_batch_prep_compare(lps, scaling_mode: int = 5, ruiz_iterations: int = 10) -> list:
    """b200pdlp_debug_hipdlp_batch_prep_compare: the device prologue and postsolve of solve_hipdlp_batch_device against their
    host twins on host LPs; one dict of mismatch counts per LP (HIPDLP_BATCH_PREP_ITEMS)."""
    return _prep_compare("b200pdlp_debug_hipdlp_batch_prep_compare", HIPDLP_BATCH_PREP_ITEMS, lps, scaling_mode,
                         ruiz_iterations)


def solve_hipdlp_batch_mixed_device(dlps, trace_cap: int = 0, **params) -> list:
    """b200pdlp_solve_hipdlp_batch_mixed_device: solve_hipdlp_batch_mixed for LPs already in GPU memory (dicts of
    lp_to_device), every member's prologue and postsolve on the device.  Returns the dicts solve_hipdlp_batch_device returns,
    with the four vectors as float64 CUDA tensors (and with trace_cap > 0 a host "trace" array); each member's bits are those
    solve_hipdlp_batch_mixed returns for it.  `device` defaults to the device of the first LP's tensors.  torch's current
    stream is synchronised first, so that inputs it is still writing are complete."""
    return _hipdlp_batch_device("b200pdlp_solve_hipdlp_batch_mixed_device", dlps, trace_cap, params)


HIPDLP_TREE_PREP_ITEMS = ["dims", "cost", "lower", "upper", "rhs", "row_upper", "col_scale", "row_scale", "rperm", "cperm",
                          "A.slices", "A.col", "A.val", "AT.slices", "AT.col", "AT.val", "A.segs", "A.long_rows", "A.lcol",
                          "A.lval", "AT.segs", "AT.long_rows", "AT.lcol", "AT.lval", "norm_cost", "norm_rhs", "scaled",
                          "col_value", "col_dual", "row_value", "row_dual"]


def hipdlp_tree_prep_compare(lps, scaling_mode: int = 5, ruiz_iterations: int = 10) -> list:
    """b200pdlp_debug_hipdlp_tree_prep_compare: the tree-mode device prologue and postsolve of solve_hipdlp_batch_mixed_device
    against formulate_hipdlp + scale_hipdlp + build_layout(ordered_max=-1) and the host postsolve, on host LPs (every one
    treated as a tree member); one dict of mismatch counts per LP (HIPDLP_TREE_PREP_ITEMS)."""
    return _prep_compare("b200pdlp_debug_hipdlp_tree_prep_compare", HIPDLP_TREE_PREP_ITEMS, lps, scaling_mode,
                         ruiz_iterations)


def solve_hipdlp_multi(lp: HighsLp, ngpus: int, devices=None, out_arrays=None, **params) -> dict:
    """b200pdlp_solve_hipdlp_multi: the HiPDLP mode on `ngpus` ranks of this process (devices may repeat: logical shards
    on one device).  device_prep is passed through: 0 (default) runs the device prologue once per device where it applies,
    -1 the host prologue; either way the bits are those of solve_hipdlp(lp, device_prep=-1, **params).
    out_arrays = (col_value, col_dual, row_value, row_dual): caller-owned (e.g. page-locked) result storage."""
    L = lib()
    L.b200pdlp_solve_hipdlp_multi.argtypes = [C.POINTER(CLp), C.POINTER(CHipdlpParams), C.POINTER(CResult), C.c_int32, _ip]
    clp, keep = make_clp(lp)
    prm = _hipdlp_params(params)
    res, arrays = _mk_result(lp, 0)
    if out_arrays is not None:
        arrays = tuple(out_arrays)
        res.col_value, res.col_dual, res.row_value, res.row_dual = (_p(a, _dp) for a in arrays)
    dev = None if devices is None else np.ascontiguousarray(devices, dtype=np.int32)
    _check(L.b200pdlp_solve_hipdlp_multi(C.byref(clp), C.byref(prm), C.byref(res), ngpus,
                                         _p(dev, _ip) if dev is not None else None), "b200pdlp_solve_hipdlp_multi")
    return _result_dict(res, arrays)


def hipdlp_shard_layout_eval(lp: HighsLp, world: int, ordered_max: int = 0, x=None, y=None, scaling_mode: int = 5,
                             ruiz_iterations: int = 10, seed: int = 0) -> dict:
    """Host-only: every rank's A_g and A_g' of solve_hipdlp_multi evaluated on the host (b200pdlp_hipdlp_shard_layout_eval).
    Returns x, y, the per-rank ax / aty (NaN outside the rank's rows / columns, standard-form order), stats, and the
    one-GPU layout's A x and A'y of the same form (b200pdlp_form_layout_eval, world = 1) as ref_ax / ref_aty."""
    L = lib()
    L.b200pdlp_hipdlp_form_create.argtypes = [C.POINTER(CLp), C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
    L.b200pdlp_hipdlp_shard_layout_eval.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, _dp, _dp, _dp, _dp, _dp]
    clp, keep = make_clp(lp)
    h = C.c_void_p()
    _check(L.b200pdlp_hipdlp_form_create(C.byref(clp), scaling_mode, ruiz_iterations, C.byref(h)), "b200pdlp_hipdlp_form_create")
    try:
        d = (C.c_int32 * 5)()
        sc = (C.c_double * 3)()
        _check(L.b200pdlp_form_dims(h, d, sc), "b200pdlp_form_dims")
        n, m = d[0], d[1]
        rng = np.random.default_rng(seed)
        x = rng.standard_normal(max(n, 1)) if x is None else np.ascontiguousarray(x, dtype=np.float64)
        y = rng.standard_normal(max(m, 1)) if y is None else np.ascontiguousarray(y, dtype=np.float64)
        ax, aty, stats = [], [], []
        for g in range(world):
            a, b, st = np.full(max(m, 1), np.nan), np.full(max(n, 1), np.nan), np.zeros(7)
            _check(L.b200pdlp_hipdlp_shard_layout_eval(h, g, world, ordered_max, _p(x, _dp), _p(y, _dp), _p(a, _dp), _p(b, _dp),
                                                       _p(st, _dp)), "b200pdlp_hipdlp_shard_layout_eval")
            ax.append(a[:m])
            aty.append(b[:n])
            stats.append(st)
        ref_ax, ref_aty, st = np.full(max(m, 1), np.nan), np.full(max(n, 1), np.nan), np.zeros(12)
        _check(L.b200pdlp_form_layout_eval(h, 0, 1, ordered_max, _p(x, _dp), _p(y, _dp), _p(ref_ax, _dp), _p(ref_aty, _dp),
                                           _p(st, _dp)), "b200pdlp_form_layout_eval")
        return dict(n=n, m=m, x=x[:n], y=y[:m], ax=ax, aty=aty, stats=stats, ref_ax=ref_ax[:m], ref_aty=ref_aty[:n],
                    ref_ordered=bool(st[2]))
    finally:
        L.b200pdlp_form_destroy(h)


def solve_multi(lp: HighsLp, ngpus: int, devices=None, warm=None, **params) -> dict:
    """b200pdlp_solve_multi: the whole solve on `ngpus` devices of this process (in-process peer linking, no NCCL)."""
    L = lib()
    L.b200pdlp_solve_multi.argtypes = [C.POINTER(CLp), C.POINTER(CParams), C.POINTER(CWarm), C.POINTER(CResult), C.c_int32, _ip]
    clp, keep = make_clp(lp)
    prm = make_params(**params)
    res, arrays = _mk_result(lp, 0)
    w, wk = _mk_warm(warm)
    dev = None if devices is None else np.ascontiguousarray(devices, dtype=np.int32)
    _check(L.b200pdlp_solve_multi(C.byref(clp), C.byref(prm), C.byref(w) if w else None, C.byref(res), ngpus,
                                  _p(dev, _ip) if dev is not None else None), "b200pdlp_solve_multi")
    return _result_dict(res, arrays)


class Problem:
    """Persistent device-resident problem (b200pdlp_problem_*)."""

    def __init__(self, lp: HighsLp, rank: int = 0, world: int = 1, **params):
        L = lib()
        self.lp = lp
        self._clp, self._keep = make_clp(lp)
        self._prm = make_params(**params)
        self._h = C.c_void_p()
        _check(L.b200pdlp_problem_create(C.byref(self._clp), C.byref(self._prm), rank, world, C.byref(self._h)),
               "b200pdlp_problem_create")
        d = (C.c_int32 * 8)()
        _check(L.b200pdlp_problem_dims(self._h, d), "b200pdlp_problem_dims")
        (self.n, self.m, self.nnz, self.neq, self.m_local, self.row_offset, self.nnz_local, self.n_orig) = list(d)

    def close(self):
        if self._h:
            lib().b200pdlp_problem_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def vector(self, which: str) -> np.ndarray:
        idx = {"cost": 0, "lower": 1, "upper": 2, "rhs": 3, "col_scale": 4, "row_scale": 5}[which]
        cap = self.n if idx in (0, 1, 2, 4) else self.m
        out = np.zeros(cap)
        k = lib().b200pdlp_problem_get_vector(self._h, idx, _p(out, _dp), cap)
        if k < 0:
            raise EngineError("b200pdlp_problem_get_vector failed")
        return out[:k]

    def csr(self):
        rp = np.zeros(self.m_local + 1, dtype=np.int32)
        col = np.zeros(max(self.nnz_local, 1), dtype=np.int32)
        val = np.zeros(max(self.nnz_local, 1))
        _check(lib().b200pdlp_problem_get_csr(self._h, _p(rp, _ip), _p(col, _ip), _p(val, _dp)), "get_csr")
        return rp, col[: self.nnz_local], val[: self.nnz_local]

    def spmv_ax(self, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float64)
        assert x.shape == (self.n,)
        out = np.zeros(self.m_local)
        _check(lib().b200pdlp_spmv_ax(self._h, _p(x, _dp), _p(out, _dp)), "b200pdlp_spmv_ax")
        return out

    def spmv_aty(self, y: np.ndarray) -> np.ndarray:
        y = np.ascontiguousarray(y, dtype=np.float64)
        assert y.shape == (self.m_local,)
        out = np.zeros(self.n)
        _check(lib().b200pdlp_spmv_aty(self._h, _p(y, _dp), _p(out, _dp)), "b200pdlp_spmv_aty")
        return out

    def primal_step(self, x, aty, tau):
        """K1 on host vectors (standard-form order): returns (x_new, |x - x_new|^2)"""
        x, aty = (np.ascontiguousarray(v, dtype=np.float64) for v in (x, aty))
        out, d = np.zeros(self.n), C.c_double()
        _check(lib().b200pdlp_primal_step(self._h, _p(x, _dp), _p(aty, _dp), float(tau), _p(out, _dp), C.byref(d)), "b200pdlp_primal_step")
        return out, d.value

    def dual_step(self, x_new, y, ax, sigma):
        """K2 on host vectors: returns (y_new, ax_new = A x_new, |y - y_new|^2)"""
        x_new, y, ax = (np.ascontiguousarray(v, dtype=np.float64) for v in (x_new, y, ax))
        yn, axn, d = np.zeros(self.m), np.zeros(self.m), C.c_double()
        _check(lib().b200pdlp_dual_step(self._h, _p(x_new, _dp), _p(y, _dp), _p(ax, _dp), float(sigma), _p(yn, _dp), _p(axn, _dp),
                                        C.byref(d)), "b200pdlp_dual_step")
        return yn, axn, d.value

    def residuals(self, x, y) -> dict:
        x, y = (np.ascontiguousarray(v, dtype=np.float64) for v in (x, y))
        out = np.zeros(10)
        _check(lib().b200pdlp_residuals(self._h, _p(x, _dp), _p(y, _dp), _p(out, _dp)), "b200pdlp_residuals")
        return dict(zip(("pobj", "dobj", "pfeas", "dfeas", "gap", "relgap", "pinf_obj", "pinf_res", "dinf_obj", "dinf_res"), out.tolist()))

    def check_device(self, x, y, ax, aty, xsum, ysum, xlr, ylr, axsum=None, atysum=None, **scalars) -> dict:
        """One device check of a tree-mode solve (b200pdlp_check_device).  Vectors in standard-form order; scalars are the
        fields of b200pdlp_check_in (iter, tau, ..., light, time_flag).  Returns the fields of b200pdlp_check_out as numbers
        and arrays ("res" as two dicts keyed by RESIDUAL_NAMES) and every vector of CHECK_VECTORS after the check (axsum /
        atysum only for light = 1)."""
        n, m = self.n, self.m
        cin = CCheckIn()
        for k, v in scalars.items():
            if not hasattr(cin, k):
                raise TypeError(f"unknown check_device field {k}")
            setattr(cin, k, v)
        light = bool(cin.light)
        vec = lambda v, ln: np.array(v, dtype=np.float64, copy=True).reshape(ln)
        v = dict(x=vec(x, n), y=vec(y, m), ax=vec(ax, m), aty=vec(aty, n), xsum=vec(xsum, n), ysum=vec(ysum, m),
                 xlr=vec(xlr, n), ylr=vec(ylr, m), xavg=np.zeros(n), yavg=np.zeros(m), axavg=np.zeros(m), atyavg=np.zeros(n))
        if light:
            v["axsum"], v["atysum"] = vec(axsum, m), vec(atysum, n)
        out = CCheckOut()
        ptrs = [_p(v[k], _dp) if k in v else None for k in CHECK_VECTORS]
        _check(lib().b200pdlp_check_device(self._h, C.byref(cin), *ptrs, C.byref(out)), "b200pdlp_check_device")
        r = {}
        for k, t in CCheckOut._fields_:
            a = getattr(out, k)
            r[k] = np.ctypeslib.as_array(a).copy() if hasattr(t, "_length_") else a
        r["res"] = [dict(zip(RESIDUAL_NAMES, r["res"][t].tolist())) for t in range(2)]
        r.update(v)
        return r

    def pass_partials(self, x, y, ax, aty, tau, sigma) -> dict:
        """One PDHG pass of a tree-mode solve and its partial sums (b200pdlp_pass_partials).  Vectors in standard-form order.
        Returns x_new, y_new, ax_new, aty_new; k1, k2, k3, the slot arrays of the three pass kernels; long_a and long_at, one
        row (standard-form row, first slot, segments) per long row of A and of A'; dx2, dy2 and inter as K4 left them."""
        n, m = self.n, self.m
        x, aty = (np.array(v, dtype=np.float64, copy=True).reshape(n) for v in (x, aty))
        y, ax = (np.array(v, dtype=np.float64, copy=True).reshape(m) for v in (y, ax))
        r = dict(x_new=np.zeros(n), y_new=np.zeros(m), ax_new=np.zeros(m), aty_new=np.zeros(n))
        # bounds of the slot counts: K1's grid is capped at 16 x 148 CTAs; K2 and K3 have at most one CTA per 256 rows and
        # one per started 2048 entries of a long row (longer than 512 entries)
        nlong = self.nnz // 513 + 1
        cap = max(16 * 148, (max(n, m) + 255) // 256 + self.nnz // 2048 + nlong)
        slots = np.zeros((3, cap))
        lr = np.zeros((2 * nlong, 3), dtype=np.int32)
        out = CPassOut()
        _check(lib().b200pdlp_pass_partials(self._h, _p(x, _dp), _p(y, _dp), _p(ax, _dp), _p(aty, _dp), float(tau), float(sigma),
                                            *(_p(r[k], _dp) for k in ("x_new", "y_new", "ax_new", "aty_new")), _p(slots, _dp),
                                            cap, _p(lr, _ip), lr.shape[0], C.byref(out)), "b200pdlp_pass_partials")
        for k in range(3):
            r[f"k{k + 1}"] = slots[k, : out.slots[k]].copy()
        r["long_a"], r["long_at"] = lr[: out.long_a].copy(), lr[out.long_a: out.long_a + out.long_at].copy()
        r.update(dx2=out.dx2, dy2=out.dy2, inter=out.inter)
        return r

    def bench_spmv(self, which: int, reps: int) -> float:
        ms = C.c_float()
        _check(lib().b200pdlp_bench_spmv(self._h, which, reps, C.byref(ms)), "b200pdlp_bench_spmv")
        return float(ms.value)

    def bench_pass(self, reps: int):
        ms = (C.c_float * 4)()
        _check(lib().b200pdlp_bench_pass(self._h, reps, ms), "b200pdlp_bench_pass")
        return [float(v) for v in ms]

    def comm_init(self, unique_id: bytes):
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        _check(lib().b200pdlp_comm_init(self._h, buf), "b200pdlp_comm_init")

    def p2p_timeline(self) -> dict:
        out = np.zeros(8)
        _check(lib().b200pdlp_p2p_timeline(self._h, _p(out, _dp)), "b200pdlp_p2p_timeline")
        keys = ["primal_shard_phase", "barrier0_total", "barrier0_wait", "ax_aty_phase", "barrier1_total", "barrier1_wait", "passes"]
        return dict(zip(keys, out[:7].tolist()))

    def p2p_release(self):
        _check(lib().b200pdlp_p2p_release(self._h), "b200pdlp_p2p_release")

    def p2p_export(self) -> bytes:
        buf = (C.c_uint8 * 256)()
        _check(lib().b200pdlp_p2p_export(self._h, buf), "b200pdlp_p2p_export")
        return bytes(buf)

    def p2p_import(self, all_handles: bytes):
        buf = (C.c_uint8 * len(all_handles)).from_buffer_copy(all_handles)
        _check(lib().b200pdlp_p2p_import(self._h, buf), "b200pdlp_p2p_import")

    def solve(self, warm=None, trace_cap: int = 0, **params) -> dict:
        prm = make_params(**params)
        res, arrays = _mk_result(self.lp, trace_cap)
        w, wk = _mk_warm(warm)
        _check(lib().b200pdlp_problem_solve(self._h, C.byref(prm), C.byref(w) if w else None, C.byref(res)),
               "b200pdlp_problem_solve")
        return _result_dict(res, arrays)


class HipProblem:
    """Persistent HiPDLP problem for kernel-level tests (b200pdlp_hipdlp_problem_create): built as solve_hipdlp builds it
    (same prologue choice and SpMV launch shapes), one GPU.  Vectors are numpy arrays in standard-form order."""

    def __init__(self, lp: HighsLp, **params):
        L = lib()
        L.b200pdlp_hipdlp_problem_create.argtypes = [C.POINTER(CLp), C.POINTER(CHipdlpParams), C.POINTER(C.c_void_p)]
        L.b200pdlp_hipdlp_step.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_int32, C.c_int32, C.c_int32] + [_dp] * 10
        L.b200pdlp_hipdlp_check.argtypes = [C.c_void_p, C.c_int32] + [_dp] * 13
        L.b200pdlp_hipdlp_problem_power_method.argtypes = [C.c_void_p, _dp]
        self.lp = lp
        self._clp, self._keep = make_clp(lp)
        self._prm = _hipdlp_params(params)
        self._h = C.c_void_p()
        _check(L.b200pdlp_hipdlp_problem_create(C.byref(self._clp), C.byref(self._prm), C.byref(self._h)),
               "b200pdlp_hipdlp_problem_create")
        d = (C.c_int32 * 8)()
        _check(L.b200pdlp_problem_dims(self._h, d), "b200pdlp_problem_dims")
        self.n, self.m, self.nnz, self.neq = list(d)[:4]

    def close(self):
        if self._h:
            lib().b200pdlp_problem_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _vec(self, v, length):
        v = np.array(v, dtype=np.float64, copy=True)
        assert v.shape == (length,), (v.shape, length)
        return v

    def step(self, primal_step, dual_step, halpern_iteration, k_offset, is_major, x, xa, aty, y, ya, xn=None, hslack=None,
             yn=None, ry=None) -> dict:
        """One Halpern step (b200pdlp_hipdlp_step).  xn, hslack, yn, ry default to NaN, which a minor step returns as
        given.  Returns x, rx, xn, hslack, y, yn, ry and aty (= A'y of the new y)."""
        n, m = self.n, self.m
        v = dict(x=self._vec(x, n), xa=self._vec(xa, n), aty=self._vec(aty, n), y=self._vec(y, m), ya=self._vec(ya, m),
                 rx=np.zeros(n), xn=self._vec(np.full(n, np.nan) if xn is None else xn, n),
                 hslack=self._vec(np.full(n, np.nan) if hslack is None else hslack, n),
                 yn=self._vec(np.full(m, np.nan) if yn is None else yn, m), ry=self._vec(np.full(m, np.nan) if ry is None else ry, m))
        _check(lib().b200pdlp_hipdlp_step(self._h, float(primal_step), float(dual_step), int(halpern_iteration), int(k_offset),
                                          int(is_major), *(_p(v[k], _dp) for k in ("x", "xa", "aty", "y", "ya", "rx", "xn",
                                                                                   "hslack", "yn", "ry"))), "b200pdlp_hipdlp_step")
        return {k: v[k] for k in ("x", "rx", "xn", "hslack", "y", "yn", "ry", "aty")}

    def check(self, major, x, y, xa, ya, rx=None, ry=None, hslack=None) -> dict:
        """One check (b200pdlp_hipdlp_check): "sums" = the nine sums, and the vectors sp, sn, ax, aty, atdy."""
        n, m = self.n, self.m
        ins = [self._vec(x, n), self._vec(y, m), self._vec(xa, n), self._vec(ya, m)]
        ins += [self._vec(v, ln) if v is not None else None for v, ln in ((rx, n), (ry, m), (hslack, n))]
        out = dict(sums=np.zeros(9), sp=np.zeros(n), sn=np.zeros(n), ax=np.zeros(m), aty=np.zeros(n), atdy=np.zeros(n))
        _check(lib().b200pdlp_hipdlp_check(self._h, int(major), *(_p(v, _dp) if v is not None else None for v in ins),
                                           *(_p(out[k], _dp) for k in ("sums", "sp", "sn", "ax", "aty", "atdy"))),
               "b200pdlp_hipdlp_check")
        return out

    def power_method(self) -> float:
        lam = C.c_double()
        _check(lib().b200pdlp_hipdlp_problem_power_method(self._h, C.byref(lam)), "b200pdlp_hipdlp_problem_power_method")
        return lam.value


def nccl_unique_id() -> bytes:
    buf = (C.c_uint8 * 128)()
    _check(lib().b200pdlp_nccl_unique_id(buf), "b200pdlp_nccl_unique_id")
    return bytes(buf)


def partition_rows(lp: HighsLp, world: int) -> np.ndarray:
    clp, keep = make_clp(lp)
    out = np.zeros(world + 1, dtype=np.int32)
    _check(lib().b200pdlp_partition_rows(C.byref(clp), world, _p(out, _ip)), "b200pdlp_partition_rows")
    return out


def host_form(lp: HighsLp, scaling: int = 1) -> dict:
    """Host-only standard form (formulate + scale) as numpy arrays; needs no GPU."""
    L = lib()
    clp, keep = make_clp(lp)
    h = C.c_void_p()
    _check(L.b200pdlp_form_create(C.byref(clp), scaling, C.byref(h)), "b200pdlp_form_create")
    try:
        d = (C.c_int32 * 5)()
        sc = (C.c_double * 3)()
        _check(L.b200pdlp_form_dims(h, d, sc), "b200pdlp_form_dims")
        n, m, nnz, neq, n_orig = list(d)
        out = dict(n=n, m=m, nnz=nnz, neq=neq, n_orig=n_orig, norm_cost=sc[0], norm_rhs=sc[1], amax=sc[2])
        for idx, (name, ln) in enumerate([("cost", n), ("lower", n), ("upper", n), ("rhs", m), ("col_scale", n), ("row_scale", m)]):
            v = np.zeros(max(ln, 1))
            k = L.b200pdlp_form_get_vector(h, idx, _p(v, _dp), ln)
            out[name] = v[:k].copy()
        cbeg = np.zeros(n + 1, dtype=np.int32)
        cidx = np.zeros(max(nnz, 1), dtype=np.int32)
        cval = np.zeros(max(nnz, 1))
        _check(L.b200pdlp_form_get_csc(h, _p(cbeg, _ip), _p(cidx, _ip), _p(cval, _dp)), "form_get_csc")
        rni = np.zeros(max(m, 1), dtype=np.int32)
        rcl = np.zeros(max(m, 1), dtype=np.int32)
        _check(L.b200pdlp_form_get_row_map(h, _p(rni, _ip), _p(rcl, _ip)), "form_get_row_map")
        rbeg = np.zeros(m + 1, dtype=np.int32)
        ridx = np.zeros(max(nnz, 1), dtype=np.int32)
        rval = np.zeros(max(nnz, 1))
        _check(L.b200pdlp_form_get_csr(h, _p(rbeg, _ip), _p(ridx, _ip), _p(rval, _dp)), "form_get_csr")
        out.update(cbeg=cbeg, cidx=cidx[:nnz], cval=cval[:nnz], row_new_idx=rni[:m], row_type=rcl[:m],
                   rbeg=rbeg, ridx=ridx[:nnz], rval=rval[:nnz])
        return out
    finally:
        L.b200pdlp_form_destroy(h)


def host_form_hipdlp(lp: HighsLp, scaling_mode: int = 5, ruiz_iterations: int = 10) -> dict:
    """Host-only HiPDLP standard form (preprocess + scale) and its power-method estimate; needs no GPU."""
    L = lib()
    L.b200pdlp_hipdlp_form_create.argtypes = [C.POINTER(CLp), C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
    L.b200pdlp_hipdlp_power_method.argtypes = [C.c_void_p, _dp]
    clp, keep = make_clp(lp)
    h = C.c_void_p()
    _check(L.b200pdlp_hipdlp_form_create(C.byref(clp), scaling_mode, ruiz_iterations, C.byref(h)), "b200pdlp_hipdlp_form_create")
    try:
        d = (C.c_int32 * 5)()
        sc = (C.c_double * 3)()
        _check(L.b200pdlp_form_dims(h, d, sc), "b200pdlp_form_dims")
        n, m, nnz, neq, n_orig = list(d)
        out = dict(n=n, m=m, nnz=nnz, neq=neq, n_orig=n_orig, c_norm=sc[0], rhs_norm=sc[1], amax=sc[2])
        for idx, (name, ln) in enumerate([("cost", n), ("lower", n), ("upper", n), ("rlo", m), ("col_scale", n), ("row_scale", m), ("rup", m)]):
            v = np.zeros(max(ln, 1))
            k = L.b200pdlp_form_get_vector(h, idx, _p(v, _dp), ln)
            out[name] = v[:k].copy()
        cbeg = np.zeros(n + 1, dtype=np.int32)
        cidx = np.zeros(max(nnz, 1), dtype=np.int32)
        cval = np.zeros(max(nnz, 1))
        _check(L.b200pdlp_form_get_csc(h, _p(cbeg, _ip), _p(cidx, _ip), _p(cval, _dp)), "form_get_csc")
        rni = np.zeros(max(m, 1), dtype=np.int32)
        rcl = np.zeros(max(m, 1), dtype=np.int32)
        _check(L.b200pdlp_form_get_row_map(h, _p(rni, _ip), _p(rcl, _ip)), "form_get_row_map")
        lam = np.zeros(1)
        _check(L.b200pdlp_hipdlp_power_method(h, _p(lam, _dp)), "b200pdlp_hipdlp_power_method")
        out.update(cbeg=cbeg, cidx=cidx[:nnz], cval=cval[:nnz], new_idx=rni[:m], ctype=rcl[:m], op_norm_sq=float(lam[0]))
        return out
    finally:
        L.b200pdlp_form_destroy(h)


def host_layout_eval(lp: HighsLp, world: int = 1, ordered_max: int = 0, x=None, y=None, scaling: int = 1, seed: int = 0) -> dict:
    """Host-only: build every rank's device layout of `lp` (as b200pdlp_problem_create would) and evaluate the
    sliced-ELL data on the host.  Returns ax (assembled over ranks), aty (summed over ranks in rank order), the
    per-rank partial A_g'y, the per-rank stats and the standard form's column-wise matrix for checking."""
    L = lib()
    clp, keep = make_clp(lp)
    h = C.c_void_p()
    _check(L.b200pdlp_form_create(C.byref(clp), scaling, C.byref(h)), "b200pdlp_form_create")
    try:
        d = (C.c_int32 * 5)()
        sc = (C.c_double * 3)()
        _check(L.b200pdlp_form_dims(h, d, sc), "b200pdlp_form_dims")
        n, m, nnz = d[0], d[1], d[2]
        rng = np.random.default_rng(seed)
        x = rng.standard_normal(max(n, 1)) if x is None else np.ascontiguousarray(x, dtype=np.float64)
        y = rng.standard_normal(max(m, 1)) if y is None else np.ascontiguousarray(y, dtype=np.float64)
        ax = np.full(max(m, 1), np.nan)
        aty = np.zeros(max(n, 1))
        parts, stats = [], []
        for g in range(world):
            part = np.full(max(n, 1), np.nan)
            st = np.zeros(12)
            _check(L.b200pdlp_form_layout_eval(h, g, world, ordered_max, _p(x, _dp), _p(y, _dp), _p(ax, _dp), _p(part, _dp),
                                               _p(st, _dp)), "b200pdlp_form_layout_eval")
            parts.append(part[:n].copy())
            stats.append(st)
            aty[:n] += part[:n]
        cbeg = np.zeros(n + 1, dtype=np.int32)
        cidx = np.zeros(max(nnz, 1), dtype=np.int32)
        cval = np.zeros(max(nnz, 1))
        _check(L.b200pdlp_form_get_csc(h, _p(cbeg, _ip), _p(cidx, _ip), _p(cval, _dp)), "form_get_csc")
        return dict(n=n, m=m, nnz=nnz, x=x[:n], y=y[:m], ax=ax[:m], aty=aty[:n], parts=parts, stats=stats,
                    cbeg=cbeg, cidx=cidx[:nnz], cval=cval[:nnz])
    finally:
        L.b200pdlp_form_destroy(h)


def solve_logical_shards(lp: HighsLp, world: int, device: int = -1, **params) -> list:
    """SURVEY.md 8(e): the multi-GPU code path with `world` logical shards inside this process (normally all on one
    device): one problem per rank, buffers wired to each other with b200pdlp_p2p_link_local, one host thread per rank
    (ctypes releases the GIL during the solve).  Returns the per-rank result dicts (identical by construction)."""
    import threading
    probs = [Problem(lp, rank=g, world=world, device=device, **params) for g in range(world)]
    try:
        arr = (C.c_void_p * world)(*[q._h for q in probs])
        _check(lib().b200pdlp_p2p_link_local(arr, world), "b200pdlp_p2p_link_local")
        out, err = [None] * world, [None] * world

        def run(g):
            try:
                out[g] = probs[g].solve(device=device, **params)
            except Exception as e:   # noqa: BLE001 -- reported to the caller below
                err[g] = e

        threads = [threading.Thread(target=run, args=(g,), daemon=True) for g in range(world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        for e in err:
            if e is not None:
                raise e
        return out
    finally:
        for q in probs:
            try:
                q.p2p_release()
            except Exception:
                pass
        for q in probs:
            q.close()


def device_count() -> int:
    return int(lib().b200pdlp_device_count())
