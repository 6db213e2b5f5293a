"""Child process of tests/test_gpu_hipdlp_batch.py (own process: a faulting kernel must not poison the CUDA context of the
test session).  Runs one named case of b200pdlp_solve_hipdlp_batch against b200pdlp_solve_hipdlp on each member alone (and,
for the oracle cases, against the HiPDLP oracle).  "Identical" = byte equality of the ints (status, iterate, iterations,
passes, restarts, form dimensions), the six residual scalars and the four HighsSolution vectors.
usage: python tests/hipdlp_batch_child.py CASE   -> one JSON line {check: "ok" | error text}"""
import glob
import json
import os
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from highs_b200 import engine  # noqa: E402
from highs_b200.lp import HighsLp, HighsSparseMatrix, read_b2lp  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
FILES = sorted(glob.glob(os.path.join(GOLDEN, "instances", "*.b2lp")))
# the option sets of tests/hipdlp_child.py
VARIANTS = [dict(iter_limit=800), dict(iter_limit=4000, tolerance=1e-4), dict(iter_limit=400, step_size_strategy=0),
            dict(iter_limit=400, scaling_mode=7, ruiz_iterations=3), dict(iter_limit=1200, tolerance=1e-3, scaling_mode=0)]
ORACLE_ALL_VARIANTS = ("afiro", "adlittle", "sctest", "e226", "25fv47")   # the others: variants 0 and 1 (as hipdlp_child.py)
INTS = ("term_code", "term_iterate", "iters", "passes", "restarts", "form_cols", "form_rows", "form_nnz", "form_neq")
SCALARS = ("primal_obj", "dual_obj", "primal_feas", "dual_feas", "gap", "rel_gap")
VECTORS = ("col_value", "col_dual", "row_value", "row_dual")


def _bits(v):
    return np.ascontiguousarray(v, dtype=np.float64).view(np.uint64)


def assert_same(a, b, what):
    for k in INTS:
        assert a[k] == b[k], (what, k, a[k], b[k])
    for k in SCALARS:
        assert _bits(a[k]) == _bits(b[k]), (what, k, a[k], b[k])
    for k in VECTORS:
        assert np.array_equal(_bits(a[k]), _bits(b[k])), (what, k)


def instances(ordered_max=4096):
    """every instance file whose HiPDLP standard form is an ordered-mode problem"""
    out = []
    for p in FILES:
        lp = read_b2lp(p)
        f = engine.host_form_hipdlp(lp)
        if max(f["n"], f["m"]) <= ordered_max:
            out.append((os.path.basename(p)[:-5], lp))
    return out


def golden(name):
    return read_b2lp(os.path.join(GOLDEN, name + ".b2lp"))


def small_set():
    return [(nm, golden(nm)) for nm in ("afiro", "avgas", "distillation", "boxed_row", "blending")]


def batch_vs_single(named, **kw):
    """one batch of every LP of `named` against each solved alone; returns the batch's results"""
    got = engine.solve_hipdlp_batch([lp for _, lp in named], **kw)
    assert len(got) == len(named)
    rounds = got[0]["kernel_launches"] if got else 0
    for (nm, lp), g in zip(named, got):
        assert_same(g, engine.solve_hipdlp(lp, **kw), nm)
        assert g["kernel_launches"] == rounds and g["solve_seconds"] == got[0]["solve_seconds"], nm
    return got


# ---- synthetic LPs
def lp_from_dense(cost, A, col_lower, col_upper, row_lower, row_upper):
    import scipy.sparse as sp
    m, n = A.shape
    a = sp.csc_matrix(A)
    a.sort_indices()
    mat = HighsSparseMatrix(n, m, a.indptr, a.indices, a.data)
    return HighsLp(n, m, cost, col_lower, col_upper, row_lower, row_upper, mat)


def mixed_lp(seed, m=60, n=80):
    """rows: equality, <=, >=, ranged, free, 1e25-bounded (a slack column for HiPDLP); columns: fixed, free, boxed, >= 0"""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((m, n)) * (rng.random((m, n)) < 0.08)
    for i in range(m):   # no empty rows
        A[i, rng.integers(n)] = 1.0 + rng.random()
    xs = rng.random(n)
    kind = np.arange(n) % 4
    lo = np.where(kind == 0, 0.5, np.where(kind == 1, -np.inf, 0.0))
    up = np.where(kind == 0, 0.5, np.where(kind == 1, np.inf, np.where(kind == 2, 2.0, np.inf)))
    xs = np.clip(xs, np.where(np.isfinite(lo), lo, -10), np.where(np.isfinite(up), up, 10))
    b = A @ xs
    rk = np.arange(m) % 7
    rl = np.select([rk == 0, rk == 1, rk == 2, rk == 3, rk == 4, rk == 5], [b, -np.inf, b - 0.5, b - 1.0, -np.inf, b - 0.1],
                   -1e25)
    ru = np.select([rk == 0, rk == 1, rk == 2, rk == 3, rk == 4, rk == 5], [b, b + 0.5, np.inf, b + 1.0, np.inf, 1e25],
                   b + 0.1)
    y = rng.standard_normal(m)
    cost = A.T @ y * 0.1 + rng.random(n)
    return lp_from_dense(cost, A, lo, up, rl, ru)


def no_rows_lp():
    rng = np.random.default_rng(5)
    n = 30
    return lp_from_dense(rng.standard_normal(n), np.zeros((0, n)), np.zeros(n), np.ones(n), np.zeros(0), np.zeros(0))


def zero_optimal_lp():
    """x = 0, y = 0 (the initial point) is optimal: the member converges at the iteration-0 check"""
    rng = np.random.default_rng(9)
    m, n = 6, 9
    A = rng.standard_normal((m, n))
    return lp_from_dense(1.0 + rng.random(n), A, np.zeros(n), np.full(n, np.inf), np.full(m, -1.0), np.full(m, np.inf))


# ---- cases
def case_instances(vi):
    def run():
        inst = instances()
        assert len(inst) > 40, len(inst)
        batch_vs_single(inst, **VARIANTS[vi])
    return run


def case_oracle(vi):
    def run():
        from oracle import binding as ob
        prm = VARIANTS[vi]
        inst = [(nm, lp) for nm, lp in instances() if vi < 2 or nm in ORACLE_ALL_VARIANTS]
        assert inst
        got = engine.solve_hipdlp_batch([lp for _, lp in inst], **prm)
        okw = dict(max_iterations=prm.get("iter_limit"), tolerance=prm.get("tolerance", 1e-7),
                   scaling_mode=prm.get("scaling_mode", 5), ruiz_iterations=prm.get("ruiz_iterations", 10),
                   step_size_strategy=prm.get("step_size_strategy", 3))
        for (nm, lp), g in zip(inst, got):
            ref = ob.hipdlp_solve(lp, **okw)
            assert g["iters"] == ref["iters"], (nm, "iterations", g["iters"], ref["iters"])
            assert (g["term_code"] == 0) == (ref["term_code"] == 0), (nm, "termination")
            for k in VECTORS:
                assert np.array_equal(_bits(g[k]), _bits(ref[k])), (nm, k)
    return run


def case_limits():
    for lim in (0, 1, 40, 41, 80):
        got = batch_vs_single(small_set(), iter_limit=lim, tolerance=1e-9)
        blocks = -(-lim // 40) if lim > 0 else 0   # a run stops at the first block end at or past the limit
        for g in got:
            assert g["term_name"] == "OPTIMAL" or (g["iters"] == 40 * blocks and g["term_iterate"] == 0), (lim, g["iters"])
        assert got[0]["kernel_launches"] == 1 + blocks, (lim, got[0]["kernel_launches"])


def case_time_limit_zero():
    got = batch_vs_single(small_set(), time_limit=0.0)
    for g in got:
        assert g["iters"] == 0 and g["term_name"] == "TIMELIMIT_OR_ITERLIMIT" and g["term_iterate"] == 2
        assert g["kernel_launches"] == 1


def case_converged_at_zero():
    named = [("distillation", golden("distillation")), ("zero_optimal", zero_optimal_lp()), ("adlittle", golden("adlittle"))]
    got = batch_vs_single(named, iter_limit=4000)
    assert got[1]["iters"] == 0 and got[1]["term_name"] == "OPTIMAL", (got[1]["iters"], got[1]["term_name"])
    assert got[0]["iters"] >= 200 and got[2]["iters"] >= 200, (got[0]["iters"], got[2]["iters"])


def case_synthetic():
    named = [(f"mixed{s}", mixed_lp(s)) for s in (1, 2, 3)] + [("no_rows", no_rows_lp()), ("zero_optimal", zero_optimal_lp())]
    got = batch_vs_single(named, iter_limit=2000, tolerance=1e-6)
    assert got[3]["form_rows"] == 0
    f = engine.host_form_hipdlp(named[0][1])
    assert f["n"] > named[0][1].num_col_   # the ranged, free and 1e25 rows have slack columns


def case_switches():
    for kw in (dict(scaling_mode=0), dict(scaling_mode=7), dict(ruiz_iterations=3), dict(step_size_strategy=0)):
        batch_vs_single(small_set() + [("mixed1", mixed_lp(1))], iter_limit=2000, tolerance=1e-5, **kw)


def case_position():
    """2001 members (more CTAs than are resident at once): afiro first, in the middle and last, the instances repeated
    around them; every copy equals its LP solved alone"""
    kw = dict(iter_limit=200)
    inst = instances()
    afiro = golden("afiro")
    names, lps = [], []
    k = 0
    while len(lps) < 2001:
        if len(lps) in (0, 1000, 2000):
            names.append("afiro"); lps.append(afiro)
        else:
            nm, lp = inst[k % len(inst)]
            names.append(nm); lps.append(lp)
            k += 1
    got = engine.solve_hipdlp_batch(lps, **kw)
    alone = {nm: engine.solve_hipdlp(lp, **kw) for nm, lp in [("afiro", afiro)] + inst}
    for i, (nm, g) in enumerate(zip(names, got)):
        assert_same(g, alone[nm], f"{nm} at {i}")


def case_twice():
    lp = golden("adlittle")
    got = batch_vs_single([("adlittle", lp), ("afiro", golden("afiro")), ("adlittle", lp)])
    assert_same(got[0], got[2], "the same LP twice")


def case_largest():
    inst = instances()
    sizes = [(engine.host_form_hipdlp(lp)["nnz"], nm, lp) for nm, lp in inst]
    _, nm, big = max(sizes, key=lambda t: t[0])
    afiro = golden("afiro")
    for named in ([(nm, big), ("afiro", afiro)], [("afiro", afiro), (nm, big)]):
        batch_vs_single(named, iter_limit=2000)


CASES = {f"instances{v}": case_instances(v) for v in range(len(VARIANTS))}
CASES.update({f"oracle{v}": case_oracle(v) for v in range(len(VARIANTS))})
CASES.update(limits=case_limits, time_limit_zero=case_time_limit_zero, converged_at_zero=case_converged_at_zero,
             synthetic=case_synthetic, switches=case_switches, position=case_position, twice=case_twice, largest=case_largest)


def main():
    name = sys.argv[1]
    try:
        CASES[name]()
        out = {name: "ok"}
    except Exception as e:   # noqa: BLE001
        traceback.print_exc()
        out = {name: f"{type(e).__name__}: {e}"[:600]}
    print(json.dumps(out))
    return 0 if out[name] == "ok" else 1


if __name__ == "__main__":
    sys.exit(main())
