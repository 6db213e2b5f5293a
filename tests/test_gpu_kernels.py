"""GPU parity of the SpMV kernels against the oracle's scatter SpMV (bit-exact)."""
import numpy as np
import pytest

from conftest import golden_lp, load_golden

pytestmark = pytest.mark.gpu


def _oracle_spmv(ob, lp, x, y):
    import ctypes as C
    L = ob.lib()
    clp, keep = ob._mk_lp(lp)
    f = ob.OrcForm()
    L.orc_formulate(C.byref(clp), C.byref(f))
    L.orc_scale(C.byref(f), 1)
    L.orc_build_csr(C.byref(f))
    ax, aty = np.zeros(max(f.m, 1)), np.zeros(max(f.n, 1))
    dp = C.POINTER(C.c_double)
    L.orc_ax(C.byref(f), x.ctypes.data_as(dp), ax.ctypes.data_as(dp))
    L.orc_aty(C.byref(f), y.ctypes.data_as(dp), aty.ctypes.data_as(dp))
    out = ax[: f.m].copy(), aty[: f.n].copy()
    L.orc_form_free(C.byref(f))
    return out


def _check(engine, ob, lp, seed=0):
    prob = engine.Problem(lp)
    rng = np.random.default_rng(seed)
    x, y = rng.standard_normal(prob.n), rng.standard_normal(prob.m)
    ax_o, aty_o = _oracle_spmv(ob, lp, x, y)
    ax, aty = prob.spmv_ax(x), prob.spmv_aty(y)
    prob.close()
    return ax, ax_o, aty, aty_o


@pytest.mark.parametrize("name", ["avgas", "afiro", "adlittle", "boxed_row", "restart_lp", "e226", "stair"])
def test_spmv_bit_exact_goldens(engine_lib, oracle, name):
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    import os
    from conftest import GOLDEN
    lp = read_b2lp(os.path.join(GOLDEN, name + ".b2lp"))
    ax, ax_o, aty, aty_o = _check(engine, oracle, lp)
    assert np.array_equal(ax, ax_o)
    assert np.array_equal(aty, aty_o)


@pytest.mark.parametrize("m,n,k", [(5000, 4000, 7), (100000, 100000, 10), (20000, 300, 3), (300, 20000, 2)])
def test_spmv_bit_exact_synthetic(engine_lib, oracle, m, n, k):
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(m, n, k, seed=5)
    ax, ax_o, aty, aty_o = _check(engine, oracle, lp)
    assert np.array_equal(ax, ax_o)
    assert np.array_equal(aty, aty_o)


def test_spmv_long_rows(engine_lib, oracle):
    """One 50%-dense column (config S5 in miniature): the A^T row of 10 000 nonzeros is split into
    segment blocks; their tree-summed partials are not in the oracle's sequential order, so the long
    row is compared to 1e-13 relative, everything else bit-exactly."""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(20000, 20000, 6, seed=9, dense_col_nnz=10000)
    ax, ax_o, aty, aty_o = _check(engine, oracle, lp)
    assert np.array_equal(ax, ax_o)
    assert np.array_equal(aty[1:], aty_o[1:])
    assert abs(aty[0] - aty_o[0]) <= 1e-13 * max(1.0, np.abs(aty_o).max())


# ---- fused hot-path kernels through their C-ABI entry points (SURVEY.md 8(b): _primal_step, _dual_step, _residuals)
def _form(ob, lp):
    return ob.formulate_and_scale(lp)


@pytest.mark.parametrize("m,n,k", [(3000, 2500, 6), (60000, 50000, 8)])
def test_primal_and_dual_step_kernels(engine_lib, oracle, m, n, k):
    """K1 / K2 against PDHG_primalGradientStep / PDHG_dualGradientStep (cupdlp_step.c:16-69) evaluated in the reference's
    CPU operation order on the oracle's scaled form: element-wise results bit for bit, the two norms to rounding"""
    import scipy.sparse as sp
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(m, n, k, seed=17)
    lp.col_upper_[::7] = 1.5    # some finite upper bounds
    f = _form(oracle, lp)
    prob = engine.Problem(lp)
    rng = np.random.default_rng(2)
    x, aty = rng.standard_normal(prob.n), rng.standard_normal(prob.n)
    y, ax = rng.standard_normal(prob.m), rng.standard_normal(prob.m)
    tau, sigma = 0.37, 0.81
    xn, dx2 = prob.primal_step(x, aty, tau)
    v = x + (-tau) * f["cost"]
    v = v + tau * aty
    v = np.minimum(v, f["upper"])
    v = np.maximum(v, f["lower"])
    assert np.array_equal(xn, v)
    assert abs(dx2 - np.sum((x - v) ** 2)) <= 1e-12 * (1 + dx2)
    yn, axn, dy2 = prob.dual_step(xn, y, ax, sigma)
    ax_o, _ = _oracle_spmv(oracle, lp, xn, y)   # the reference's scatter order
    assert np.array_equal(axn, ax_o)
    w = y + sigma * f["rhs"]
    w = w + (-2.0 * sigma) * ax_o
    w = w + sigma * ax
    w[f["neq"]:] = np.maximum(w[f["neq"]:], 0.0)
    assert np.array_equal(yn, w)
    assert abs(dy2 - np.sum((y - w) ** 2)) <= 1e-12 * (1 + dy2)
    prob.close()


def _residual_lp(kind, m, n, seed=23):
    """banded LP (2..10 entries per row within 1000 of the diagonal: the tiled pass shape is chosen for it, no row is long).
    geq: A x >= b, x >= 0.  mixed: boxed rows first (each becomes an equality row with a slack column), then equality rows,
    then LEQ and GEQ rows mixed; columns with a lower bound only, boxed, free, upper-only and fixed; maximised, with an
    offset"""
    from highs_b200.lp import HighsLp, HighsSparseMatrix, kHighsInf
    rng = np.random.default_rng(seed)
    ln = rng.integers(2, 11, size=m)
    rows = np.repeat(np.arange(m, dtype=np.int64), ln)
    cols = rows * n // m + rng.integers(-1000, 1001, size=rows.size)
    keep = (cols >= 0) & (cols < n)   # (not clipped: that would pile entries into long first and last columns)
    key = np.unique(cols[keep] * m + rows[keep])
    c, r = key // m, key % m
    start = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(c, minlength=n), out=start[1:])
    val = rng.standard_normal(key.size)
    cost = rng.standard_normal(n)
    lo, up = np.zeros(n), np.full(n, kHighsInf)
    b = rng.standard_normal(m)
    rl, ru = b.copy(), np.full(m, kHighsInf)
    sense, offset = 1, 0.0
    if kind == "mixed":
        t = np.arange(n) % 5
        lo[t == 1], up[t == 1] = -1.0, 2.0                      # boxed
        lo[t == 2] = -kHighsInf                                  # free
        lo[t == 3], up[t == 3] = -kHighsInf, 1.5                 # upper only
        lo[t == 4] = up[t == 4] = 0.75                           # fixed
        boxed, eq = np.arange(64), np.arange(64, 6000)
        ru[boxed] = b[boxed] + 1.0
        ru[eq] = b[eq]
        leq = np.flatnonzero((np.arange(m) >= 6000) & (rng.random(m) < 0.5))
        rl[leq], ru[leq] = -kHighsInf, b[leq]
        sense, offset = -1, 2.5
    return HighsLp(n, m, cost, lo, up, rl, ru, HighsSparseMatrix(n, m, start.astype(np.int32), r.astype(np.int32), val),
                   sense, offset, f"residual_{kind}")


def _residuals_reference(f, sense, offset, x, y):
    """numpy restatement of PDHG_Compute_Residuals, _Primal_Infeasibility, _Dual_Infeasibility and _Infeas_Residuals
    (cupdlp_solver.c) for the iterate (x, y) on the scaled standard form; returns {output: (value, tolerance)}"""
    import math
    import scipy.sparse as sp
    A = sp.csr_matrix((f["rval"], f["ridx"], f["rbeg"]), shape=(f["m"], f["n"]))
    ax, aty = A @ x, A.T @ y
    ineq = np.arange(f["m"]) >= f["neq"]
    c, lo, up, b, cs, rs = f["cost"], f["lower"], f["upper"], f["rhs"], f["col_scale"], f["row_scale"]
    hl, hu = lo > -np.inf, up < np.inf
    dot = lambda u, v: math.fsum(u * v)
    mag = lambda u, v: math.fsum(np.abs(u * v))
    # primal feasibility: objective, |[A x - b]_eq, min(A x - b, 0)_ineq rowScale|
    pobj = dot(c, x) * sense + offset
    r = ax - b
    r[ineq] = np.minimum(r[ineq], 0.0)
    pfeas = np.linalg.norm(r * rs)
    # dual feasibility: slacks of the reduced costs where the bound exists, dual objective, |rc - s+ + s-| colScale
    rc = c - aty
    spos, sneg = np.where(hl, np.maximum(rc, 0.0), 0.0), np.where(hu, -np.minimum(rc, 0.0), 0.0)
    lf, uf = np.where(hl, lo, 0.0), np.where(hu, up, 0.0)
    dobj = (math.fsum(np.concatenate([b * y, spos * lf, -(sneg * uf)]))) * sense + offset
    dfeas = np.linalg.norm((rc - spos + sneg) * cs)
    gap = pobj - dobj
    relgap = abs(pobj - dobj) / (1.0 + abs(pobj) + abs(dobj))
    # primal infeasibility: the dual ray (y, s+, s-) scaled to unit length
    dscale = math.sqrt(dot(y, y) + dot(spos, spos) + dot(sneg, sneg))
    dscale = 1.0 if dscale < 1e-8 else dscale
    pinf_obj = (dobj - offset) / sense / dscale
    pinf_res = np.linalg.norm((aty / dscale + spos / dscale - sneg / dscale) * cs)
    # dual infeasibility: the primal ray x scaled to unit length
    pscale = np.linalg.norm(x)
    pscale = 1.0 if pscale < 1e-8 else pscale
    dinf_obj = (pobj - offset) / sense / pscale
    ray = x / pscale
    k = ax / pscale
    k[ineq] = np.minimum(k[ineq], 0.0)
    lb = np.where(hl, np.minimum(ray, 0.0), 0.0) / cs
    ub = np.where(hu, np.maximum(ray, 0.0), 0.0) / cs
    dinf_res = math.sqrt(dot(k * rs, k * rs) + dot(lb, lb) + dot(ub, ub))
    # tolerances: 1e-11 of the magnitudes that enter each value (the objectives cancel)
    pm = mag(c, x) + abs(offset)
    dm = mag(b, y) + mag(spos, lf) + mag(sneg, uf) + abs(offset)
    tol = lambda v: 1e-11 * (1.0 + abs(v))
    return {"pobj": (pobj, 1e-11 * (1 + pm)), "dobj": (dobj, 1e-11 * (1 + dm)), "pfeas": (pfeas, tol(pfeas)),
            "dfeas": (dfeas, tol(dfeas)), "gap": (gap, 1e-11 * (1 + pm + dm)),
            "relgap": (relgap, 1e-11 * (1 + pm + dm) / (1.0 + abs(pobj) + abs(dobj))),
            "pinf_obj": (pinf_obj, 1e-11 * (1 + dm) / dscale), "pinf_res": (pinf_res, tol(pinf_res)),
            "dinf_obj": (dinf_obj, 1e-11 * (1 + pm) / pscale), "dinf_res": (dinf_res, tol(dinf_res))}


def test_residual_kernels(engine_lib, oracle, monkeypatch, capfd):
    """all ten check-iteration outputs of b200pdlp_residuals -- objectives, feasibilities, gaps and the four infeasibility
    quantities that decide INFEASIBLE / UNBOUNDED -- against numpy on the oracle's scaled form, for three LPs: a random one
    with x >= 0 and GEQ rows at a nonnegative iterate, and two banded ones (GEQ rows only; every kind of row and column
    bound) under every pass shape.  The banded LPs have no long rows, so A x and A'y of the iterate are the same bits in
    every shape, and so are the ten values."""
    from test_gpu_spmv_shapes import PASS_SHAPES, ROWS_PER_CTA, TILE_ROWS, assert_shape, forced_problem, sm_count
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    sms = sm_count()
    m = max(11 * TILE_ROWS, -(-(2 * ROWS_PER_CTA * sms + 4096) // TILE_ROWS) * TILE_ROWS)
    cases = [("random", synthetic_lp(40000, 30000, 7, seed=23), ("default",)),   # (too few rows for a persistent grid)
             ("geq", _residual_lp("geq", m, m - 2112), PASS_SHAPES),
             ("mixed", _residual_lp("mixed", m, m - 2112), PASS_SHAPES)]
    for kind, lp, arms in cases:
        f = _form(oracle, lp)
        if kind == "mixed":
            assert f["n"] == lp.num_col_ + 64 and f["neq"] == 6000
        rng = np.random.default_rng(4)
        x, y = rng.standard_normal(f["n"]), rng.standard_normal(f["m"])
        if kind == "random":
            x = np.abs(x)
            y[f["neq"]:] = np.abs(y[f["neq"]:])
        ref = _residuals_reference(f, lp.sense_, lp.offset_, x, y)
        outs = {}
        for arm in arms:
            prob, shapes = forced_problem(engine, lp, arm, monkeypatch, capfd)
            try:
                assert_shape(arm, shapes, {"A": f["m"], "A'": f["n"]}, sms)
                outs[arm] = got = prob.residuals(x, y)
            finally:
                prob.close()
            for k, (v, tol) in ref.items():
                assert abs(got[k] - v) <= tol, (kind, arm, k, got[k], v)
        for arm, got in outs.items():
            assert got == outs["default"], (kind, arm, {k: (v, outs["default"][k]) for k, v in got.items()
                                                        if v != outs["default"][k]})
