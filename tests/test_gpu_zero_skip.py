"""The zero-skip shape of the PDHG pass SpMVs returns the bits of the shape it stands in for.

On one GPU in tree mode the engine runs K2 (A x' + dual step) and K3 (A'y' + interaction) with spmv_sell_zskip_kernel
wherever the matrix is not tiled: it gathers only the inputs whose bit in the nonzero bitmap is 1 and writes the same block
partial sums as the shape chosen otherwise.  B200PDLP_ZERO_SKIP=0 (read when a problem is created) turns the choice off.
Every case below runs both arms and asks for equal arrays, np.array_equal, not for a tolerance.
"""
import os
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_ZS_RE = re.compile(r"zero-skip pass SpMVs: A (\d+) CTAs  A' (\d+) CTAs")


def planted_lp(A, seed, name):
    """min c.x  s.t.  A x >= b, x >= 0 on the scipy matrix A, with a planted optimal pair (as highs_b200.lp.synthetic_lp)"""
    from highs_b200.lp import HighsLp, HighsSparseMatrix, kHighsInf
    A = A.tocsc()
    A.sort_indices()
    m, n = A.shape
    rng = np.random.default_rng(seed)
    xs = np.where(rng.random(n) < 0.5, 0.0, rng.random(n))
    ys = np.where(rng.random(m) < 0.5, 0.0, rng.random(m))
    b = A @ xs - np.where(ys > 0, 0.0, rng.random(m))
    c = A.T @ ys + np.where(xs > 0, 0.0, rng.random(n))
    return HighsLp(n, m, c, np.zeros(n), np.full(n, kHighsInf), b, np.full(m, kHighsInf),
                   HighsSparseMatrix(n, m, A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(np.float64)),
                   1, 0.0, name)


def s3_like(n=200_000):
    from highs_b200.lp import synthetic_lp
    return synthetic_lp(n, n, 8, seed=7)


def s5_like(n=200_000):
    """S5's dense column (a long row of A') and, transposed, a dense row (a long row of A)"""
    from highs_b200.lp import synthetic_lp
    a = synthetic_lp(n, n, 8, seed=9, dense_col_nnz=20_000).a_matrix_.to_scipy()
    import scipy.sparse as sp
    return planted_lp(sp.hstack([a, a.T[:, : n // 2]]), 10, "s5_like_both_long")


def create(engine, lp, arm, monkeypatch, capfd):
    """engine.Problem(lp) in tree mode with the zero-skip shape on (arm 1) or off (arm 0); checks which one the engine took"""
    monkeypatch.setenv("B200PDLP_ZERO_SKIP", str(arm))
    monkeypatch.setenv("B200PDLP_TIMING", "1")
    capfd.readouterr()
    prob = engine.Problem(lp, ordered_max=-1)
    found = _ZS_RE.findall(capfd.readouterr().err)
    monkeypatch.delenv("B200PDLP_ZERO_SKIP")
    monkeypatch.delenv("B200PDLP_TIMING")
    assert found, "the engine printed no zero-skip line"
    a, at = (int(v) for v in found[-1])
    assert (a > 0 and at > 0) if arm else (a == 0 and at == 0), (arm, a, at)
    return prob


def zeros_input(rng, k):
    """a vector with exact +0.0, -0.0, subnormals and dense runs of zeros"""
    v = rng.standard_normal(k)
    v[rng.random(k) < 0.4] = 0.0
    v[rng.random(k) < 0.1] = -0.0
    v[rng.random(k) < 0.02] = 5e-324
    v[rng.random(k) < 0.02] = -2.2e-310
    for s in rng.integers(0, k, size=20):
        v[s:s + 4096] = 0.0
    v[: min(k, 3000)] = 0.0
    return v


@pytest.mark.parametrize("transposed", [False, True], ids=["A_x", "AT_y"])
def test_pass_spmv_bits(engine_lib, monkeypatch, capfd, transposed):
    """K2 on inputs full of zeros of every kind: A x' and y' (and |dy|^2) equal in both arms.  A'y runs through the same
    kernel as the A x of the transposed LP."""
    from highs_b200 import engine
    lp = s5_like(60_000)
    if transposed:
        lp = planted_lp(lp.a_matrix_.to_scipy().T, 3, "transposed")
    out = []
    for arm in (0, 1):
        prob = create(engine, lp, arm, monkeypatch, capfd)
        r = np.random.default_rng(5)
        x, y, ax = zeros_input(r, prob.n), zeros_input(r, prob.m), r.standard_normal(prob.m)
        out.append(prob.dual_step(x, y, ax, 0.37))
        prob.close()
    (y0, ax0, d0), (y1, ax1, d1) = out
    assert np.array_equal(ax0, ax1) and np.array_equal(y0, y1)
    assert np.array_equal(np.signbit(ax0), np.signbit(ax1))
    assert d0 == d1


@pytest.mark.parametrize("case", ["s3_like", "s5_like", "golden_greenbea"])
def test_solve_bits(engine_lib, monkeypatch, capfd, case):
    """every output of a 300-iteration solve is the same in both arms"""
    from highs_b200 import engine
    if case == "s3_like":
        lp = s3_like()
    elif case == "s5_like":
        lp = s5_like()
    else:
        from highs_b200.lp import read_b2lp
        lp = read_b2lp(os.path.join(ROOT, "tests", "golden", "instances", "greenbea.b2lp"))
    res = []
    for arm in (0, 1):
        prob = create(engine, lp, arm, monkeypatch, capfd)
        res.append(prob.solve(iter_limit=300))
        prob.close()
    a, b = res
    for k in ("col_value", "col_dual", "row_value", "row_dual"):
        assert np.array_equal(a[k], b[k]), k
    for k in ("iters", "restarts", "term_name"):
        assert a[k] == b[k], (k, a[k], b[k])
