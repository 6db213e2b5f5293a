"""Child process of tests/test_gpu_hipdlp_batch_mixed.py (own process: a faulting kernel must not poison the CUDA context of
the test session).  Runs one named case of b200pdlp_solve_hipdlp_batch_mixed against b200pdlp_solve_hipdlp on each tree
member alone (and against b200pdlp_solve_hipdlp_batch for the ordered members).  "Identical" = byte equality of the ints,
the six residual scalars, the four HighsSolution vectors and the trace rows.
usage: python tests/hipdlp_batch_mixed_child.py CASE   -> one JSON line {case: "ok" | error text}"""
import json
import os
import re
import sys
import tempfile
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

from highs_b200 import engine  # noqa: E402
from highs_b200.lp import HighsLp, HighsSparseMatrix  # noqa: E402
from hipdlp_batch_child import (VARIANTS, _bits, assert_same, golden, instances, mixed_lp, no_rows_lp,  # noqa: E402
                                small_set, zero_optimal_lp)

TRACE = 256   # trace rows kept per member: more than any case's blocks


def assert_same_trace(a, b, what):
    assert_same(a, b, what)
    assert a["trace"].shape == b["trace"].shape, (what, "trace rows", a["trace"].shape, b["trace"].shape)
    assert np.array_equal(_bits(a["trace"]), _bits(b["trace"])), (what, "trace")


def mixed_vs_single(named, **kw):
    """one mixed batch of every LP of `named` against each solved alone by solve_hipdlp; returns the batch's results"""
    got = engine.solve_hipdlp_batch_mixed([lp for _, lp in named], trace_cap=TRACE, **kw)
    assert len(got) == len(named)
    for (nm, lp), g in zip(named, got):
        assert_same_trace(g, engine.solve_hipdlp(lp, trace_cap=TRACE, **kw), nm)
        assert g["kernel_launches"] == got[0]["kernel_launches"] and g["solve_seconds"] == got[0]["solve_seconds"], nm
    return got


# ---- mid-size synthetic members (tree mode at the default ordered_max)
def midsize_lp(seed, m, n, per_col=4, long_rows=(), long_cols=(), empty=True, descending=False):
    """mixed_lp's row kinds (equality, <=, >=, ranged, free, 1e25-bounded) and column kinds (fixed, free, boxed, >= 0) at
    size: `long_rows` / `long_cols` give rows / columns of that many nonzeros, `empty` leaves the last row (a free row) and
    the last column (cost >= 0, x >= 0) without entries, `descending` stores column 1's entries in descending row order"""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    nr = n - (1 if empty else 0)
    rows = [rng.choice(m - (1 if empty else 0), size=per_col, replace=False) for _ in range(nr)]
    cols = [np.full(per_col, j) for j in range(nr)]
    for k, ln in enumerate(long_rows):   # row k: ln entries
        cols.append(rng.choice(nr, size=ln, replace=False)); rows.append(np.full(ln, k))
    for k, ln in enumerate(long_cols):   # column k: ln entries
        rows.append(rng.choice(m - (1 if empty else 0), size=ln, replace=False)); cols.append(np.full(ln, k))
    r, c = np.concatenate(rows), np.concatenate(cols)
    A = sp.csc_matrix((rng.standard_normal(r.size), (r, c)), shape=(m, n))
    A.sum_duplicates()
    A.sort_indices()
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
    if empty:
        rl[-1], ru[-1] = -np.inf, np.inf
    cost = A.T @ rng.standard_normal(m) * 0.1 + rng.random(n)
    if empty:
        lo[-1], up[-1], cost[-1] = 0.0, np.inf, 1.0
    start, index, value = A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.copy()
    if descending:
        s0, s1 = start[1], start[2]
        index[s0:s1], value[s0:s1] = index[s0:s1][::-1].copy(), value[s0:s1][::-1].copy()
    return HighsLp(n, m, cost, lo, up, rl, ru, HighsSparseMatrix(n, m, start, index, value))


def easy_lp(seed, n):
    """A = I + a sparse perturbation, equality rows, boxed columns: well conditioned, converges in a few blocks"""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    A = (sp.identity(n, format="csc") + sp.random(n, n, density=2.0 / n, random_state=seed, format="csc") * 0.1).tocsc()
    A.sort_indices()
    xs = rng.random(n)
    b = A @ xs
    return HighsLp(n, n, rng.standard_normal(n), np.zeros(n), np.ones(n), b, b,
                   HighsSparseMatrix(n, n, A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.copy()))


def midsize_set():
    return [("rows_long", midsize_lp(1, 6000, 5000, long_rows=(700, 1500, 2048, 2049, 4900))),
            ("cols_long", midsize_lp(2, 5000, 7000, long_cols=(600, 2048, 3000, 4500), descending=True)),
            ("both_long", midsize_lp(3, 20000, 18000, long_rows=(9000,), long_cols=(513, 2600))),
            ("wide", midsize_lp(4, 8000, 40000, per_col=3, long_rows=(4100, 20000))),
            ("tall", midsize_lp(5, 120000, 90000, per_col=3, empty=True, descending=True)),
            ("easy", easy_lp(6, 8000))]


# ---- cases
def case_instances_tree(vi):
    def run():
        inst = instances()
        assert len(inst) > 40, len(inst)
        mixed_vs_single(inst, ordered_max=-1, **VARIANTS[vi])
    return run


def case_midsize():
    named = midsize_set()
    for nm, lp in named:
        f = engine.host_form_hipdlp(lp)
        assert 5000 <= max(f["n"], f["m"]) <= 200000, (nm, f["n"], f["m"])
    got = mixed_vs_single(named, iter_limit=3000, tolerance=1e-4)
    assert any(g["restarts"] > 0 for g in got), [g["restarts"] for g in got]
    assert any(g["term_name"] == "OPTIMAL" for g in got), [g["term_name"] for g in got]


def case_mixed():
    """ordered and tree members interleaved: the tree members equal their single solves, the ordered members the plain batch"""
    small = small_set() + [("mixed1", mixed_lp(1)), ("no_rows", no_rows_lp())]
    mid = midsize_set()[:3]
    named = [small[0], mid[0], small[1], small[2], mid[1], small[3], mid[2], small[4], small[5], small[6]]
    kw = dict(iter_limit=2000, tolerance=1e-5)
    got = engine.solve_hipdlp_batch_mixed([lp for _, lp in named], trace_cap=TRACE, **kw)
    ordered = [i for i, (nm, _) in enumerate(named) if nm not in dict(mid)]
    plain = engine.solve_hipdlp_batch([named[i][1] for i in ordered], **kw)
    for i, p in zip(ordered, plain):
        assert_same(got[i], p, named[i][0])
        assert_same_trace(got[i], engine.solve_hipdlp(named[i][1], trace_cap=TRACE, **kw), named[i][0])
    for i, (nm, lp) in enumerate(named):
        if i not in ordered:
            assert_same_trace(got[i], engine.solve_hipdlp(lp, trace_cap=TRACE, **kw), nm)


def _timed_mixed(lps, **kw):
    """solve_hipdlp_batch_mixed with B200PDLP_TIMING=1; returns the results and the cluster size its timing line names"""
    os.environ["B200PDLP_TIMING"] = "1"
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            got = engine.solve_hipdlp_batch_mixed(lps, trace_cap=TRACE, **kw)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["B200PDLP_TIMING"]
        f.seek(0)
        text = f.read()
    m = re.search(r"tree members (\d+), cluster of C = (\d+) CTAs", text)
    assert m, text[-2000:]
    assert int(m.group(1)) == sum(1 for lp in lps), (m.group(1), len(lps))
    return got, int(m.group(2))


def case_clusters():
    named = midsize_set()[:4] + [("mixed2", mixed_lp(2))]
    kw = dict(iter_limit=1200, tolerance=1e-6, ordered_max=-1)
    runs = {}
    for c in ("1", "2", "4", "8"):
        os.environ["B200PDLP_BATCH_CLUSTER"] = c
        try:
            runs[c] = engine.solve_hipdlp_batch_mixed([lp for _, lp in named], trace_cap=TRACE, **kw)
        finally:
            del os.environ["B200PDLP_BATCH_CLUSTER"]
    for c in ("2", "4", "8"):
        for (nm, _), a, b in zip(named, runs["1"], runs[c]):
            assert_same_trace(a, b, f"{nm} C=1 vs C={c}")
    # the default choice: a few members take C > 1; more copies than clusters of 2 fit on the GPU take C = 1
    got, c = _timed_mixed([lp for _, lp in named], **kw)
    assert c > 1, c
    for (nm, lp), g in zip(named, got):
        assert_same_trace(g, engine.solve_hipdlp(lp, trace_cap=TRACE, **kw), nm)
    afiro, adl = golden("afiro"), golden("adlittle")
    many = [afiro if i % 2 else adl for i in range(1200)]
    kw = dict(iter_limit=200, ordered_max=-1)
    got, c = _timed_mixed(many, **kw)
    assert c == 1, c
    alone = {id(afiro): engine.solve_hipdlp(afiro, trace_cap=TRACE, **kw), id(adl): engine.solve_hipdlp(adl, trace_cap=TRACE, **kw)}
    for i, (lp, g) in enumerate(zip(many, got)):
        assert_same_trace(g, alone[id(lp)], f"copy {i}")


def case_limits():
    named = small_set() + [("mixed3", mixed_lp(3)), ("no_rows", no_rows_lp()), ("zero_optimal", zero_optimal_lp())]
    for lim in (0, 1, 40, 41, 80):
        got = mixed_vs_single(named, iter_limit=lim, tolerance=1e-9, ordered_max=-1)
        assert got[0]["kernel_launches"] == 1 + (-(-lim // 40) if lim > 0 else 0), (lim, got[0]["kernel_launches"])
    got = mixed_vs_single(named, time_limit=0.0, ordered_max=-1)
    assert all(g["term_iterate"] == 2 or g["term_name"] == "OPTIMAL" for g in got)
    got = mixed_vs_single(named, iter_limit=2000, ordered_max=-1)
    assert got[-1]["iters"] == 0 and got[-1]["term_name"] == "OPTIMAL", (got[-1]["iters"], got[-1]["term_name"])
    assert got[-2]["form_rows"] == 0
    for kw in (dict(step_size_strategy=0), dict(scaling_mode=0)):
        mixed_vs_single(named + midsize_set()[:1], iter_limit=1000, tolerance=1e-5, ordered_max=-1, **kw)


def case_host_prologue():
    named = midsize_set()[:3] + [("mixed1", mixed_lp(1)), ("afiro", golden("afiro"))]
    kw = dict(iter_limit=1000, tolerance=1e-5, ordered_max=-1)
    got = engine.solve_hipdlp_batch_mixed([lp for _, lp in named], trace_cap=TRACE, **kw)
    for (nm, lp), g in zip(named, got):
        assert_same_trace(g, engine.solve_hipdlp(lp, trace_cap=TRACE, device_prep=-1, **kw), nm)


def case_twice():
    named = midsize_set()[:2] + [("afiro", golden("afiro"))]
    kw = dict(iter_limit=800, ordered_max=-1)
    a = engine.solve_hipdlp_batch_mixed([lp for _, lp in named], trace_cap=TRACE, **kw)
    b = mixed_vs_single(named, **kw)
    for (nm, _), x, y in zip(named, a, b):
        assert_same_trace(x, y, nm)


CASES = {f"instances_tree{v}": case_instances_tree(v) for v in range(len(VARIANTS))}
CASES.update(midsize=case_midsize, mixed=case_mixed, clusters=case_clusters, limits=case_limits,
             host_prologue=case_host_prologue, twice=case_twice)


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
