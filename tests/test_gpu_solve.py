"""GPU parity of whole solves (through the C ABI) against the reference's goldens and the oracle.

Bar (BASELINE.json north_star): objectives and KKT residuals within 1e-6 relative of HiGHS's CPU
pdlp on identical HighsLp input.  The element-wise arithmetic of the CUDA path is bit-identical to
the reference's; only the order of the long reductions differs, so on the small goldens the
trajectories coincide: identical iteration counts and objectives to ~1e-9 relative.
"""
import numpy as np
import pytest

from conftest import (case_id, golden_lp, golden_solution, load_golden, options_to_params,
                      term_to_model_status)

pytestmark = pytest.mark.gpu

CASES = load_golden()
REL_TOL = 1e-6   # north_star tolerance


def _rel(a, b):
    return abs(a - b) / (1.0 + abs(b))


@pytest.mark.parametrize("case", [c for c in CASES if c["warm_from"] is None], ids=case_id)
def test_golden_solve(engine_lib, oracle, case):
    from highs_b200 import engine
    lp = golden_lp(case)
    params = options_to_params(case["options"])
    res = engine.solve(lp, **params)
    status = term_to_model_status(res["term_code"], res["iters"], params.get("iter_limit", 2147483647))
    if oracle.ref_available():
        # what Highs::run() reports after lpKktCheck for OUR solution (Highs.cpp:1990)
        kkt = oracle.reference_kkt(lp, res, status, case["options"])
        assert kkt["model_status_code"] == case["model_status_code"], (kkt["model_status"], case["model_status"])
        for fld in ("max_primal_infeasibility", "max_dual_infeasibility", "primal_dual_objective_error",
                    "max_complementarity_violation", "max_primal_residual_error", "max_dual_residual_error"):
            # residuals are O(tol) quantities: compare on the scale the reference itself uses (1 + |ref|)
            assert abs(kkt[fld] - case[fld]) <= REL_TOL * (1.0 + abs(case[fld])) + 1e-9, (fld, kkt[fld], case[fld])
    else:
        expect = case["model_status_code"]
        if case["model_status_code"] == 10 and status == 9:
            expect = 9   # kUnboundedOrInfeasible -> kUnbounded happens in lpKktCheck (HighsSolution.cpp:1074-1077)
        assert status == expect
    if max(lp.num_col_, lp.num_row_) <= 2048:   # ordered-reduction regime: trajectory reproduces exactly
        assert res["iters"] == case["pdlp_iteration_count"], (res["iters"], case["pdlp_iteration_count"])
    if case["model_status_code"] in (7, 14):
        obj = lp.objectiveValue(res["col_value"])
        assert _rel(obj, case["objective_function_value"]) <= REL_TOL
        gold = golden_solution(case)
        if gold is not None:
            scale = 1.0 + np.abs(gold["col_value"]).max()
            assert np.abs(res["col_value"] - gold["col_value"]).max() <= 1e-6 * scale
            assert np.abs(res["row_dual"] - gold["row_dual"]).max() <= 1e-6 * (1.0 + np.abs(gold["row_dual"]).max())


def test_hot_start(engine_lib, oracle):
    """check/TestPdlp.cpp:260-285: re-running from the previous HighsSolution."""
    from highs_b200 import engine
    case = [c for c in CASES if c["warm_from"]][0]
    lp = golden_lp(case)
    first = dict(np.load(__import__("os").path.join(__import__("conftest").GOLDEN, case["warm_from"])))
    res = engine.solve(lp, warm=(first["col_value"], first["row_value"], first["row_dual"]),
                       **options_to_params(case["options"]))
    assert res["term_name"] == "OPTIMAL"
    assert res["iters"] == case["pdlp_iteration_count"]
    assert _rel(lp.objectiveValue(res["col_value"]), case["objective_function_value"]) <= REL_TOL


@pytest.mark.parametrize("flags", [dict(scaling=0), dict(adaptive_step=0), dict(restart=0), dict(scaling=0, restart=0)])
def test_feature_switches_vs_oracle(engine_lib, oracle, flags):
    """pdlp_features_off paths (HConst.h:417-422) are not reachable through Highs options in 1.15.1,
    so they are pinned against the oracle restatement."""
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    import os
    from conftest import GOLDEN
    lp = read_b2lp(os.path.join(GOLDEN, "afiro.b2lp"))
    kw = dict(tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4, iter_limit=20000, **flags)
    res, orc = engine.solve(lp, **kw), oracle.solve(lp, **kw)
    assert res["term_code"] == orc["term_code"]
    assert res["iters"] == orc["iters"]
    assert _rel(lp.objectiveValue(res["col_value"]), lp.objectiveValue(orc["col_value"])) <= REL_TOL


def test_wrapper_interface(engine_lib):
    """solveLpCupdlp mirror: same struct contract as CupdlpWrapper.cpp:30-278."""
    from highs_b200 import pdlp
    from highs_b200.lp import read_b2lp
    import os
    from conftest import GOLDEN
    lp = read_b2lp(os.path.join(GOLDEN, "avgas.b2lp"))
    opt, sol, info, basis = pdlp.HighsOptions(), pdlp.HighsSolution(), pdlp.HighsInfo(), pdlp.HighsBasis(valid=True)
    st, ms = pdlp.solveLpCupdlp(opt, pdlp.HighsTimer(), lp, basis, sol, info)
    assert st == pdlp.HighsStatus.kOk and ms == pdlp.HighsModelStatus.kOptimal
    assert info.pdlp_iteration_count == 200 and sol.value_valid and sol.dual_valid and not basis.valid
    assert abs(lp.objectiveValue(sol.col_value) - (-7.7499999699309976)) < 1e-8
    # second call hot-starts from the incumbent (value_valid && dual_valid) and stops at once
    st, ms = pdlp.solveLpCupdlp(opt, pdlp.HighsTimer(), lp, basis, sol, info)
    assert ms == pdlp.HighsModelStatus.kOptimal and info.pdlp_iteration_count == 0
    opt.pdlp_iteration_limit = 80
    sol = pdlp.HighsSolution()
    st, ms = pdlp.solveLpCupdlp(opt, pdlp.HighsTimer(), lp, basis, sol, info)
    assert ms == pdlp.HighsModelStatus.kIterationLimit and info.pdlp_iteration_count == 79


def test_s2_properties(engine_lib):
    """Config S2 (m=n=100k, nnz=1M): size-independent properties of a solve to kkt 1e-4:
    KKT conditions of the returned point recomputed independently in numpy."""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(100000, 100000, 10, seed=12345)
    res = engine.solve(lp, tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4, iter_limit=200000)
    assert res["term_name"] == "OPTIMAL"
    A = lp.a_matrix_.to_scipy()
    x, y = res["col_value"], res["row_dual"]
    assert np.allclose(A @ x, res["row_value"], rtol=0, atol=1e-9 * (1 + np.abs(res["row_value"]).max()))
    rc = lp.col_cost_ - A.T @ y
    # x >= 0 without upper bounds: col_dual is the part of the reduced cost the bound can carry
    assert np.allclose(np.maximum(rc, 0), res["col_dual"], rtol=0, atol=1e-9 * (1 + np.abs(rc).max()))
    pinf = np.linalg.norm(np.minimum(A @ x - lp.row_lower_, 0))
    dinf = np.linalg.norm(np.minimum(rc, 0)) + np.linalg.norm(np.minimum(y, 0))
    assert x.min() >= 0
    assert pinf <= 1e-4 * (1 + np.linalg.norm(lp.row_lower_)) * 10
    assert dinf <= 1e-4 * (1 + np.linalg.norm(lp.col_cost_)) * 10
    pobj, dobj = lp.col_cost_ @ x, lp.row_lower_ @ y
    assert abs(pobj - dobj) <= 1e-3 * (1 + abs(pobj) + abs(dobj))


@pytest.mark.parametrize("name,kw", [
    ("avgas", {}), ("afiro", {}), ("adlittle", {}), ("boxed_row", {}), ("restart_lp", {}),
    ("distillation", dict(tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4)), ("sctest", {}), ("chip", {}),
    ("e226", dict(tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4)),
    ("afiro", dict(adaptive_step=0, tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4)),
    ("afiro", dict(scaling=0, tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4)),
])
def test_trajectory_bit_exact(engine_lib, oracle, name, kw):
    """Ordered-reduction mode (problems up to ordered_max rows/cols): every check iteration's
    objectives, residuals, step sizes and restart decisions equal the oracle's (and therefore the
    reference's) BIT FOR BIT, and so does the returned HighsSolution."""
    import os
    from conftest import GOLDEN
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    lp = read_b2lp(os.path.join(GOLDEN, name + ".b2lp"))
    res = engine.solve(lp, trace_cap=4096, **kw)
    orc = oracle.solve(lp, trace_cap=4096, **kw)
    assert res["iters"] == orc["iters"] and res["term_code"] == orc["term_code"]
    k = min(len(res["trace"]), len(orc["trace"]))
    assert k > 0 and len(res["trace"]) == len(orc["trace"])
    assert np.array_equal(res["trace"][:, :15], orc["trace"][:, :15]), \
        np.argwhere(res["trace"][:, :15] != orc["trace"][:, :15])[:5]
    for key in ("col_value", "col_dual", "row_value", "row_dual"):
        assert np.array_equal(res[key], orc[key]), key


def test_tree_vs_ordered_reductions_agree(engine_lib):
    """The production (tree) reductions against the ordered ones on the same LP: same optimum to the
    solver tolerance (trajectories may differ: the step rule divides by a cancelling sum)."""
    import os
    from conftest import GOLDEN
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    lp = read_b2lp(os.path.join(GOLDEN, "adlittle.b2lp"))
    a = engine.solve(lp, ordered_max=-1)
    b = engine.solve(lp)
    assert a["term_name"] == b["term_name"] == "OPTIMAL"
    assert _rel(lp.objectiveValue(a["col_value"]), lp.objectiveValue(b["col_value"])) <= REL_TOL


def _ragged_lp(seed):
    """empty columns and rows, fixed / free / boxed columns, EQ / ranged / free / LEQ / GEQ rows, maximise, offset"""
    import scipy.sparse as sp
    from highs_b200.lp import HighsLp, HighsSparseMatrix
    rng = np.random.default_rng(seed)
    m, n = 60, 50
    A = sp.random(m, n, density=0.12, random_state=seed, data_rvs=rng.standard_normal).tolil()
    A[:, [3, 17]] = 0          # empty columns
    A[[5, 40], :] = 0          # empty rows
    A = A.tocsc()
    A.eliminate_zeros()
    x0 = rng.random(n)
    ax = A @ x0
    kind = rng.integers(0, 5, size=m)
    rl = np.where(kind == 0, ax, np.where(kind == 1, ax - 0.5, np.where(kind == 2, -np.inf, np.where(kind == 3, ax - 1, -np.inf))))
    ru = np.where(kind == 0, ax, np.where(kind == 1, np.inf, np.where(kind == 2, ax + 0.5, np.where(kind == 3, ax + 1, np.inf))))
    rl[5], ru[5] = -1.0, 1.0   # empty ranged row (feasible)
    rl[40], ru[40] = -np.inf, np.inf
    lo = np.where(rng.random(n) < 0.7, 0.0, -np.inf)
    up = np.where(rng.random(n) < 0.4, 2.0, np.inf)
    lo[7] = up[7] = 0.5        # fixed column
    lo[3], up[3] = 0.0, 1.0
    c = rng.standard_normal(n)
    c[np.isinf(lo) & np.isinf(up)] = 0.0     # keep free columns bounded through zero cost
    return HighsLp(n, m, c, lo, up, rl, ru, HighsSparseMatrix(n, m, A.indptr, A.indices, A.data), -1 if seed % 2 else 1, 1.25)


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_ragged_lp_bit_exact(engine_lib, oracle, seed):
    from highs_b200 import engine
    lp = _ragged_lp(seed)
    kw = dict(tol_primal=1e-5, tol_dual=1e-5, tol_gap=1e-5, iter_limit=40000)
    res, orc = engine.solve(lp, trace_cap=2048, **kw), oracle.solve(lp, trace_cap=2048, **kw)
    assert res["term_code"] == orc["term_code"] and res["iters"] == orc["iters"]
    assert np.array_equal(res["trace"][:, :15], orc["trace"][:, :15])
    for key in ("col_value", "col_dual", "row_value", "row_dual"):
        assert np.array_equal(res[key], orc[key]), key


def test_time_limit(engine_lib):
    """D_TIME_LIM: the solve stops at the first check after the limit with kTimeLimit (CupdlpWrapper.cpp:233-236)"""
    from highs_b200 import pdlp
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(100000, 100000, 10, seed=3)
    opt = pdlp.HighsOptions(time_limit=1e-3)
    sol, info, basis = pdlp.HighsSolution(), pdlp.HighsInfo(), pdlp.HighsBasis()
    st, ms = pdlp.solveLpCupdlp(opt, pdlp.HighsTimer(), lp, basis, sol, info)
    assert st == pdlp.HighsStatus.kOk and ms == pdlp.HighsModelStatus.kTimeLimit
    assert 0 < info.pdlp_iteration_count < 100000 and sol.value_valid


def test_dense_column_s5_mini(engine_lib, oracle):
    """config S5 in miniature (one 50%-dense column: long-row segments in A^T): converges to the oracle's optimum"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(6000, 6000, 6, seed=2, dense_col_nnz=3000)
    kw = dict(tol_primal=1e-6, tol_dual=1e-6, tol_gap=1e-6, iter_limit=200000)
    res, orc = engine.solve(lp, **kw), oracle.solve(lp, **kw)
    assert res["term_name"] == orc["term_name"] == "OPTIMAL"
    assert _rel(lp.objectiveValue(res["col_value"]), lp.objectiveValue(orc["col_value"])) <= 1e-5


def _converged_parity(golden, tol):
    """SURVEY.md 8(d): config S2 (100k x 100k, 1M nonzeros; tree-mode reductions) solved to kkt_tolerance 1e-4 / 1e-6 against
    the UNMODIFIED reference's run on the same LP (tests/golden/s2_converged.json, written by make_s2_golden.py from
    oracle/_ref).  What "the same result" means for two converged PDLP runs whose long sums are added in different orders is
    MEASURED, not assumed: profiles/r02_s2_order_sensitivity.json holds the oracle (which reproduces the reference's 1240 /
    17 880 iterations and its objective to 13 digits with the reference's sequential sums) re-run with nothing changed but the
    grouping of those sums -- the iteration count then spreads over 1040 .. 1240 (1e-4) and 15 960 .. 26 360 (1e-6), the
    objective over 1.5 / 3.7 times t (1 + 2 |ref|) (the gap tolerance brackets the optimum only up to the primal infeasibility
    that the feasibility tolerance still allows).  Hence (SURVEY.md 8(c), "Reading"):
      * same status (Optimal from the reference's own lpKktCheck rules, evaluated on OUR solution by the device KKT check);
      * objective within 6 t (1 + 2 |ref|);
      * iteration count within a factor 2 either way;
      * the reference's KKT measures on the same side of the tolerance and at most one order of magnitude above its values."""
    import json
    import os
    from conftest import GOLDEN
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    path = os.path.join(GOLDEN, golden)
    if not os.path.exists(path):
        pytest.skip(f"tests/golden/{golden} missing (python tests/golden/make_s2_golden.py / make_s3_golden.py)")
    g = json.load(open(path))
    w, ref = g["workload"], g["runs"][tol]
    lp = synthetic_lp(w["m"], w["n"], w["nnz_per_col"], w["seed"])
    assert lp.a_matrix_.numNz() == w["nnz"]
    t = float(tol)
    res = engine.solve(lp, tol_primal=t, tol_dual=t, tol_gap=t, iter_limit=2_000_000)
    assert res["term_code"] == 0 and ref["model_status"] == "Optimal"
    assert max(res["form_cols"], res["form_rows"]) > 4096          # tree mode
    obj = lp.objectiveValue(res["col_value"])
    assert abs(obj - ref["objective_function_value"]) <= 6 * t * (1 + 2 * abs(ref["objective_function_value"]))
    assert 0.5 * ref["pdlp_iteration_count"] <= res["iters"] <= 2.0 * ref["pdlp_iteration_count"], (res["iters"], ref["pdlp_iteration_count"])
    kkt = engine.kkt_check(lp, res, kkt_tolerance=t, model_status=7)
    assert kkt["model_status"] == ref["model_status_code"] == 7
    floor = 1e-3 * t      # below a thousandth of the tolerance a measure is "zero" for both (e.g. the 1e-15 residual of A x - row_value)
    for k in ("max_primal_infeasibility", "max_dual_infeasibility", "max_relative_primal_infeasibility",
              "max_relative_dual_infeasibility", "max_primal_residual_error", "max_dual_residual_error",
              "max_relative_primal_residual_error", "max_relative_dual_residual_error",
              "primal_dual_objective_error", "max_complementarity_violation"):
        a, b = kkt[k], ref[k]
        assert a <= 10 * b + floor, (k, a, b)      # (a violation measure smaller than the reference's is no disagreement)



@pytest.mark.parametrize("tol", ["0.0001", "1e-06"])
def test_s2_converged_parity_with_the_reference(engine_lib, tol):
    _converged_parity("s2_converged.json", tol)


def test_s2_tight_tolerance_objective_to_1e_6(engine_lib):
    """SURVEY.md 8(d) verbatim: "tight-tolerance (1e-8) converged run on S2 for the 1e-6 parity check".  The unmodified reference
    needs 362 800 iterations / 51 minutes of CPU for it (tests/golden/s2_converged.json, run "1e-08"); the engine a few seconds.
    Both objectives then sit within ~1e-8 (1 + |p| + |d|) of the optimum: they must agree to 1e-6 (1 + |ref|), the north star's
    criterion, and the reference's KKT measures of OUR solution must pass at kkt_tolerance = 1e-8."""
    import json
    import os
    from conftest import GOLDEN
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    g = json.load(open(os.path.join(GOLDEN, "s2_converged.json")))
    if "1e-08" not in g["runs"]:
        pytest.skip("no 1e-8 run in tests/golden/s2_converged.json")
    w, ref = g["workload"], g["runs"]["1e-08"]
    lp = synthetic_lp(w["m"], w["n"], w["nnz_per_col"], w["seed"])
    res = engine.solve(lp, tol_primal=1e-8, tol_dual=1e-8, tol_gap=1e-8, iter_limit=5_000_000)
    assert res["term_code"] == 0 and ref["model_status"] == "Optimal"
    obj = lp.objectiveValue(res["col_value"])
    assert abs(obj - ref["objective_function_value"]) <= 1e-6 * (1 + abs(ref["objective_function_value"])), (obj, ref["objective_function_value"])
    assert 0.4 * ref["pdlp_iteration_count"] <= res["iters"] <= 2.5 * ref["pdlp_iteration_count"], (res["iters"], ref["pdlp_iteration_count"])
    kkt = engine.kkt_check(lp, res, kkt_tolerance=1e-8, model_status=7)
    assert kkt["model_status"] == ref["model_status_code"] == 7


def test_s3_converged_parity_with_the_reference(engine_lib):
    """The same comparison at the headline size (S3: 1M x 1M, 8M nonzeros), kkt_tolerance 1e-4: the reference needs minutes for
    it (tests/golden/s3_converged.json, make_s3_golden.py), the engine a fraction of a second."""
    _converged_parity("s3_converged.json", "0.0001")


@pytest.mark.parametrize("warm", [False, True], ids=["cold", "hot_start"])
def test_light_check_matches_the_spmv_check(engine_lib, oracle, monkeypatch, warm):
    """Dense-check phase (iterations 0-9 are all check iterations, cupdlp_solver.c:953-962): the passes carry A xSum and A'ySum
    and the checks are two vector sweeps (engine.cu `h_light`, pdhg_kernels.cu check_light_*).  Against the same solve with
    every check multiplying the average iterate by A and A' (B200PDLP_LIGHT_CHECK=0) and against the oracle: same check
    rows to rounding (A (sum w x) vs sum w (A x): a reassociation, like any tree-mode sum), same iteration counts.
    Columns with lower > 0 make proj(0) != 0 (xSum's start value); the hot start makes x0 != proj(0)."""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(7000, 6000, 6, seed=21)
    lp.col_lower_[::7] = 0.25                      # proj(0) = 0.25 there
    lp.col_upper_[::5] = 3.0
    w = None
    if warm:
        first = engine.solve(lp, ordered_max=-1, iter_limit=300)
        w = (first["col_value"], first["row_value"], first["row_dual"])
    kw = dict(ordered_max=-1, iter_limit=60, trace_cap=256, warm=w)
    monkeypatch.setenv("B200PDLP_LIGHT_CHECK", "0")
    a = engine.solve(lp, **kw)
    monkeypatch.setenv("B200PDLP_LIGHT_CHECK", "1")
    b = engine.solve(lp, **kw)
    assert a["iters"] == b["iters"] and a["term_code"] == b["term_code"]
    ta, tb = a["trace"], b["trace"]
    assert len(ta) == len(tb) >= 11 and np.array_equal(ta[:, 0], tb[:, 0])
    # the light phase launches two sweeps where the other launches an averaging kernel and two SpMV
    assert b["kernel_launches"] < a["kernel_launches"]
    scale = 1.0 + np.abs(ta[:, 1:9]).max(axis=0)
    assert (np.abs(ta[:, 1:9] - tb[:, 1:9]) <= 1e-9 * scale).all(), np.abs(ta[:, 1:9] - tb[:, 1:9]).max(axis=0)
    for k in ("col_value", "row_dual"):
        assert np.abs(a[k] - b[k]).max() <= 1e-9 * (1 + np.abs(a[k]).max())
    orc = oracle.solve(lp, iter_limit=60, trace_cap=256, warm=w)
    to = orc["trace"]
    assert len(to) == len(tb) and np.array_equal(to[:, 0], tb[:, 0])
    assert (np.abs(to[:11, 1:9] - tb[:11, 1:9]) <= 1e-7 * scale).all()
