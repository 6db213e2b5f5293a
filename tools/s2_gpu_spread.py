"""GPU side of tools/s2_order_sensitivity.py: S2 solved to `tol` by the engine under settings that only regroup floating-point
sums (grid shapes of the SpMV kernels, light vs SpMV checks) -- the spread of the iteration count.
    python tools/s2_gpu_spread.py <tol> [<tol> ...]      (one JSON line per run)"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from highs_b200 import engine  # noqa: E402
from highs_b200.lp import synthetic_lp  # noqa: E402

lp = synthetic_lp(100_000, 100_000, 10, 12345)
SETTINGS = [
    ("default", {}),
    ("at_grid_0", {"B200PDLP_SPMV_AT_CTAS_PER_SM": "0"}),
    ("at_grid_2", {"B200PDLP_SPMV_AT_CTAS_PER_SM": "2"}),
    ("a_grid_3", {"B200PDLP_SPMV_A_CTAS_PER_SM": "3"}),
    ("spmv_checks", {"B200PDLP_LIGHT_CHECK": "0"}),
    ("host_prologue", {"B200PDLP_DEVICE_PREP": "0"}),
]
for tol in [float(a) for a in sys.argv[1:]]:
    for name, env in SETTINGS:
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            r = engine.solve(lp, tol_primal=tol, tol_dual=tol, tol_gap=tol, iter_limit=2_000_000)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        print(json.dumps(dict(tol=tol, setting=name, iters=r["iters"], restarts=r["restarts"], term=r["term_name"],
                              objective=lp.objectiveValue(r["col_value"]), solve_seconds=r["solve_seconds"])), flush=True)
