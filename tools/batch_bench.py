"""Batched solve against a loop of single solves: b200pdlp_solve_batch (one CTA per LP) vs b200pdlp_solve per LP.

Workload: every ordered-mode instance of tests/golden/instances (standard form max(n, m) <= 4096), replicated R times, at the
default tolerances and at kkt_tolerance 1e-4, each bounded by --iter-limit PDHG iterations (some instances need 10^5
iterations at the default tolerances; the bound keeps the loop arm to minutes).  After one warm-up of each arm, the arms run
in alternating order --repeats times; the two must return identical bits.  Prints one JSON line: per workload the best
time of each arm, LPs/s, summed PDHG iterations/s, the batch's rounds, its host time per round beside its kernel time per
round, and the speed-up, with the card's name and power limit read in the same run.
--solver hipdlp: the same measurement for the HiPDLP mode, b200pdlp_solve_hipdlp_batch against a loop of
b200pdlp_solve_hipdlp, on the instances whose HiPDLP standard form is ordered, at the default tolerance and at 1e-4.
    python tools/batch_bench.py [--solver pdlp|hipdlp] [--replicas 8] [--iter-limit 500] [--repeats 2]
"""
import argparse
import glob
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from highs_b200 import engine  # noqa: E402
from highs_b200.lp import read_b2lp  # noqa: E402

INTS = ("term_code", "term_iterate", "iters", "passes", "restarts")
FLOATS = ("primal_obj", "dual_obj", "primal_feas", "dual_feas", "gap", "rel_gap")
VECTORS = ("col_value", "col_dual", "row_value", "row_dual")


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                      text=True, timeout=30).strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return dict(card=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # (the measurement itself still needs the GPU: engine calls fail without one)
        return dict(card=f"unknown ({e})", power_limit="unknown", max_sm_clock="unknown")


def identical(a, b):
    if any(a[k] != b[k] for k in INTS):
        return False
    if any(np.float64(a[k]).view(np.uint64) != np.float64(b[k]).view(np.uint64) for k in FLOATS):
        return False
    return all(np.array_equal(a[k].view(np.uint64), b[k].view(np.uint64)) for k in VECTORS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=8)
    ap.add_argument("--iter-limit", type=int, default=500)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--solver", choices=("pdlp", "hipdlp"), default="pdlp")
    a = ap.parse_args()
    hip = a.solver == "hipdlp"
    if engine.device_count() == 0:
        sys.exit("batch_bench.py needs a CUDA device")
    lps = []
    for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "instances", "*.b2lp"))):
        lp = read_b2lp(p)
        f = engine.host_form_hipdlp(lp) if hip else engine.host_form(lp, 1)
        if max(f["n"], f["m"]) <= 4096:
            lps.append(lp)
    work = lps * a.replicas
    result = dict(card(), **({"solver": "hipdlp"} if hip else {}), instances=len(lps), replicas=a.replicas, members=len(work),
                  iter_limit=a.iter_limit, repeats=a.repeats, workloads=[])
    for name, tol in (("default", None), ("kkt1e-4", 1e-4)):
        kw = dict(iter_limit=a.iter_limit)
        if tol:
            kw.update(dict(tolerance=tol) if hip else dict(tol_primal=tol, tol_dual=tol, tol_gap=tol))
        solve_batch, solve = (engine.solve_hipdlp_batch, engine.solve_hipdlp) if hip else (engine.solve_batch, engine.solve)

        def run_batch():
            t = time.perf_counter()
            r = solve_batch(work, **kw)
            return time.perf_counter() - t, r

        def run_loop():
            t = time.perf_counter()
            r = [solve(lp, **kw) for lp in work]
            return time.perf_counter() - t, r

        run_batch(); run_loop()   # warm-up (module loads, allocation caches)
        tb, tl, same = [], [], True
        for rep in range(a.repeats):
            for arm in ((run_batch, run_loop) if rep % 2 == 0 else (run_loop, run_batch)):
                t, r = arm()
                if arm is run_batch:
                    tb.append(t); rb = r
                else:
                    tl.append(t); rl = r
            same = same and all(identical(x, y) for x, y in zip(rb, rl))
        iters = sum(r["iters"] for r in rb)
        rounds = rb[0]["kernel_launches"]
        loop_s = rb[0]["solve_seconds"]
        kernel_ms = rb[0]["iter_device_ms"]
        result["workloads"].append(dict(
            name=name, identical_bits=same, pdhg_iterations=iters,
            batch_s=[round(t, 4) for t in tb], loop_s=[round(t, 4) for t in tl],
            batch_lps_per_s=round(len(work) / min(tb), 2), loop_lps_per_s=round(len(work) / min(tl), 2),
            batch_iters_per_s=round(iters / min(tb), 1), loop_iters_per_s=round(iters / min(tl), 1),
            rounds=rounds, batch_setup_ms=round(1e3 * rb[0]["setup_seconds"], 2),
            kernel_ms_per_round=round(kernel_ms / max(rounds, 1), 4),
            host_ms_per_round=round((1e3 * loop_s - kernel_ms) / max(rounds, 1), 4),
            speedup=round(min(tl) / min(tb), 3)))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
