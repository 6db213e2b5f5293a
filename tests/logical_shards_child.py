"""Child process of tests/test_gpu_logical_shards.py: the multi-GPU code path (row blocks + column shards, the fused
peer-memory kernels, flag barriers, device-side step rule, speculative check, NCCL-free solution assembly) with G
LOGICAL shards on ONE device -- SURVEY.md 8(e): "the same code path must run with G logical shards on 1 device".
Run in its own process so that a stuck barrier can be killed by PID without taking the test session along.
usage: python tests/logical_shards_child.py <world> <case>      prints one JSON line and exits 0 on success"""
import json
import os
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # one hardware queue per logical rank's stream
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from highs_b200 import engine  # noqa: E402
from highs_b200.lp import read_b2lp, synthetic_lp  # noqa: E402


def long_rows_lp():
    """two row blocks of 9000 rows, each with one row of 3 segments (6000 and 4500 entries): DualEpilogueMg and
    CheckRowEpilogue write the long rows' terms"""
    import scipy.sparse as sp
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_zero_skip import planted_lp
    a = [synthetic_lp(7000, 9000, 5, seed=s, dense_col_nnz=k).a_matrix_.to_scipy() for s, k in ((5, 6000), (6, 4500))]
    return planted_lp(sp.vstack([a[0].T, a[1].T]), 19, "long_rows")


def main():
    world, case = int(sys.argv[1]), sys.argv[2]
    tol = 1e-5
    if case == "synthetic":
        lp = synthetic_lp(6000, 5000, 6, seed=11)
    elif case == "dense":
        lp = synthetic_lp(9000, 7000, 5, seed=5, dense_col_nnz=4000)     # long rows of A' on every rank
    elif case == "long_rows":
        lp = long_rows_lp()
    else:
        lp = read_b2lp(os.path.join(ROOT, "tests", "golden", case + ".b2lp"))
        tol = 1e-7
    prm = dict(iter_limit=400000, tol_primal=tol, tol_dual=tol, tol_gap=tol)
    # the ORACLE (CPU restatement pinned to the reference) is what the shards must agree with; the single-GPU engine is
    # reported beside it
    from oracle import binding as ob
    ref = ob.solve(lp, **prm)
    one = engine.solve(lp, ordered_max=-1, **prm)
    rerun_fails = []
    if len(sys.argv) > 3 and sys.argv[3] == "c_entry":
        # the same thing through the one-call C entry point the HiGHS shim uses for B200PDLP_GPUS > 1, all ranks on device 0
        r = engine.solve_multi(lp, world, devices=[0] * world, **prm)
        res = [r, r]
    else:
        res = engine.solve_logical_shards(lp, world, **prm)
    if case == "long_rows":
        # a second solve returns the same bits on every rank: the long rows' terms have fixed slots
        again = engine.solve_logical_shards(lp, world, **prm)
        for g, (r, q) in enumerate(zip(res, again)):
            for k in ("col_value", "col_dual", "row_value", "row_dual"):
                if not np.array_equal(r[k], q[k]):
                    rerun_fails.append(f"rank {g} {k}: the second solve differs")
            if (r["iters"], r["term_code"]) != (q["iters"], q["term_code"]):
                rerun_fails.append(f"rank {g}: iters/term {q['iters']}/{q['term_code']} in the second solve vs {r['iters']}/{r['term_code']}")
    o_ref = lp.objectiveValue(ref["col_value"])
    out = dict(world=world, case=case, ref_iters=ref["iters"], ref_term=ref["term_code"], ref_obj=o_ref,
               one_gpu_iters=one["iters"], one_gpu_obj=lp.objectiveValue(one["col_value"]),
               iters=[r["iters"] for r in res], term=[r["term_code"] for r in res],
               obj=[lp.objectiveValue(r["col_value"]) for r in res])
    fails = list(rerun_fails)
    for g, r in enumerate(res[1:], start=1):   # every rank takes the same decisions and returns the same (complete) solution
        for k in ("col_value", "col_dual", "row_value", "row_dual"):
            if not np.array_equal(r[k], res[0][k]):
                bad = np.flatnonzero(r[k] != res[0][k])
                fails.append(f"rank {g} {k}: {bad.size} of {r[k].size} entries differ from rank 0 (first at {int(bad[0])}, last at {int(bad[-1])})")
        if not (r["iters"] == res[0]["iters"] and r["term_code"] == res[0]["term_code"]):
            fails.append(f"rank {g}: iters/term {r['iters']}/{r['term_code']} vs rank 0 {res[0]['iters']}/{res[0]['term_code']}")
    out["ranks_identical"] = not fails
    r0 = res[0]
    if not (r0["term_code"] == ref["term_code"] == 0):
        fails.append(f"term {r0['term_code']} vs oracle {ref['term_code']}")
    # both runs stop at relative gap < tol: they bracket the optimum to ~tol (1 + |p| + |d|) each
    if not abs(out["obj"][0] - o_ref) <= 3 * tol * (1 + 2 * abs(o_ref)):
        fails.append(f"objective {out['obj'][0]} vs oracle {o_ref}")
    # (converged iteration counts spread by tens of percent under a mere regrouping of the long sums: measured on the oracle
    #  itself, profiles/r02_s2_order_sensitivity.json)
    if not 0.5 * ref["iters"] - 80 <= r0["iters"] <= 2.0 * ref["iters"] + 80:
        fails.append(f"iterations {r0['iters']} vs oracle {ref['iters']}")
    # the assembled solution in the ORIGINAL space: row_value must be A x
    A = lp.a_matrix_.to_scipy()
    ax = A @ r0["col_value"]
    err = float(np.abs(ax - r0["row_value"]).max())
    out["row_value_err"] = err
    if not np.allclose(ax, r0["row_value"], rtol=1e-8, atol=1e-7 * (1 + np.abs(r0["row_value"]).max())):
        bad = np.flatnonzero(np.abs(ax - r0["row_value"]) > 1e-7 * (1 + np.abs(r0["row_value"]).max()) + 1e-8 * np.abs(r0["row_value"]))
        fails.append(f"row_value != A col_value: max err {err}, {bad.size} rows (first {int(bad[0])}, last {int(bad[-1])})")
    out["restarts"] = [r.get("restarts") for r in res]
    out["term_iterate"] = [r.get("term_iterate") for r in res]
    out["fails"] = fails
    ok = not fails
    out["ok"] = bool(ok)
    print(json.dumps(out))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
