"""The HiPDLP kernel-level entry points and the per-block trace, without a GPU: exported symbols, no CPU fallback, argument
rejections, the trace layout, and the HiPDLP oracle's order switch (hip_set_sum_block) at its default of 0, which must leave
the oracle pinned to the reference's goldens.  The kernels themselves are tested on the GPU in test_gpu_hipdlp_kernels.py."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

NEW_SYMBOLS = ("b200pdlp_hipdlp_problem_create", "b200pdlp_hipdlp_step", "b200pdlp_hipdlp_check",
               "b200pdlp_hipdlp_problem_power_method")
# engine trace column -> HiPDLP oracle trace column (oracle/hipdlp_oracle.h: 10..13 are the post-restart fixed-point sums,
# which the engine's trace leaves out)
ORACLE_TRACE_COLS = list(range(10)) + list(range(14, 20))
ERR_ARG, ERR_CUDA = -1, -2


def _define(path, name):
    m = re.search(rf"#define\s+{name}\s+(\d+)", open(os.path.join(ROOT, path)).read())
    assert m, (path, name)
    return int(m.group(1))


def test_new_symbols_exported(engine_lib):
    from highs_b200 import engine
    for nm in NEW_SYMBOLS:
        assert hasattr(engine_lib, nm), nm
        assert nm in engine.ABI_SYMBOLS, nm


def test_trace_layout():
    """16 engine columns = the oracle's columns 0-9 and 14-19 (iterations, nine sums, restart, weight, steps, fpe, converged)"""
    from highs_b200 import engine
    assert _define("include/b200pdlp.h", "B200PDLP_HIP_TRACE_COLS") == engine.HIP_TRACE_COLS == len(ORACLE_TRACE_COLS) == 16
    assert _define("oracle/hipdlp_oracle.h", "HIP_TRACE_COLS") == 20 == ORACLE_TRACE_COLS[-1] + 1
    assert "trace_cap" in engine.solve_hipdlp.__code__.co_varnames


def test_no_cpu_fallback(engine_lib):
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(engine.EngineError, match="no CUDA device"):
        engine.HipProblem(synthetic_lp(50, 40, 3, 1))
    with pytest.raises(engine.EngineError, match="no CUDA device"):
        engine.HipProblem(synthetic_lp(5000, 4000, 3, 1), ordered_max=-1)


def test_argument_rejections(engine_lib):
    """NULL problems, arrays and parameters: B200PDLP_ERR_ARG before any device is looked for, naming the entry point"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    L = engine.lib()
    L.b200pdlp_hipdlp_problem_create.argtypes = [C.POINTER(engine.CLp), C.POINTER(engine.CHipdlpParams), C.POINTER(C.c_void_p)]
    L.b200pdlp_hipdlp_step.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_int32, C.c_int32, C.c_int32] + [engine._dp] * 10
    L.b200pdlp_hipdlp_check.argtypes = [C.c_void_p, C.c_int32] + [engine._dp] * 13
    L.b200pdlp_hipdlp_problem_power_method.argtypes = [C.c_void_p, engine._dp]
    lp = synthetic_lp(50, 40, 3, 1)
    clp, keep = engine.make_clp(lp)
    prm = engine._hipdlp_params({})
    h = C.c_void_p()
    assert L.b200pdlp_hipdlp_problem_create(None, C.byref(prm), C.byref(h)) == ERR_ARG
    assert L.b200pdlp_hipdlp_problem_create(C.byref(clp), None, C.byref(h)) == ERR_ARG
    assert L.b200pdlp_hipdlp_problem_create(C.byref(clp), C.byref(prm), None) == ERR_ARG
    assert not h.value
    v = np.zeros(64)
    pv = engine._p(v, engine._dp)
    assert L.b200pdlp_hipdlp_step(None, 1.0, 1.0, 0, 1, 1, *([pv] * 10)) == ERR_ARG
    assert "b200pdlp_hipdlp_step" in L.b200pdlp_last_error().decode()
    assert L.b200pdlp_hipdlp_step(None, 1.0, 1.0, 0, 1, 1, *([pv] * 9 + [None])) == ERR_ARG
    assert L.b200pdlp_hipdlp_check(None, 1, *([pv] * 13)) == ERR_ARG
    assert "b200pdlp_hipdlp_check" in L.b200pdlp_last_error().decode()
    # a major check needs rx, ry and hslack
    assert L.b200pdlp_hipdlp_check(None, 1, pv, pv, pv, pv, None, pv, pv, *([pv] * 6)) == ERR_ARG
    assert L.b200pdlp_hipdlp_problem_power_method(None, pv) == ERR_ARG
    assert "b200pdlp_hipdlp_problem_power_method" in L.b200pdlp_last_error().decode()
    lam = C.c_double(-1.0)
    assert L.b200pdlp_hipdlp_problem_power_method(None, C.byref(lam)) == ERR_ARG and lam.value == -1.0


def test_sum_block_zero_reproduces_goldens(oracle):
    """hip_set_sum_block(k) changes the oracle's summation order; after resetting it to 0 the oracle is the reference again"""
    from highs_b200.lp import read_b2lp
    cases = [c for c in json.load(open(os.path.join(GOLDEN, "hipdlp", "golden.json")))
             if c["name"] in ("afiro", "adlittle", "e226")]
    assert len(cases) >= 10
    acted = 0
    try:
        for case in cases:
            lp = read_b2lp(os.path.join(GOLDEN, "instances", case["name"] + ".b2lp"))
            kw = dict(max_iterations=case["options"].get("pdlp_iteration_limit", 2147483647),
                      tolerance=case["options"].get("kkt_tolerance", 1e-7),
                      step_size_strategy=case["options"].get("pdlp_step_size_strategy", 3),
                      scaling_mode=case["options"].get("pdlp_scaling_mode", 5),
                      ruiz_iterations=case["options"].get("pdlp_ruiz_iterations", 10))
            oracle.hipdlp_set_sum_block(7)
            moved = oracle.hipdlp_solve(lp, **kw)
            oracle.hipdlp_set_sum_block(0)
            res = oracle.hipdlp_solve(lp, **kw)
            gold = dict(np.load(os.path.join(GOLDEN, "hipdlp", case["file"])))
            assert res["iters"] == case["pdlp_iteration_count"], case["file"]
            for k in ("col_value", "col_dual", "row_value", "row_dual"):
                assert np.array_equal(res[k], gold[k]), (case["file"], k)
            acted += any(moved[k] != res[k] for k in ("op_norm_sq", "pfeas", "dfeas", "iters"))
    finally:
        oracle.hipdlp_set_sum_block(0)
    # the switch does act: a block of 7 changes the rounding of every dot product longer than 7
    assert acted >= len(cases) // 2, (acted, len(cases))
