#!/usr/bin/env python3
"""tools/hipdlp_batch_mixed_bench.py -- mid-size HiPDLP LPs solved by b200pdlp_solve_hipdlp_batch_mixed (one thread-block
cluster per LP) against a loop of b200pdlp_solve_hipdlp over the same LPs.

    python tools/hipdlp_batch_mixed_bench.py [--out DIR] [--counts 4,300] [--m 30000] [--n 30000] [--per-col 5] [--iters 400]

Members: synthetic_lp(m, n, per_col, seed) for seeds 1..count (~ per_col * n nonzeros each), a fixed iteration limit and a
tolerance no member reaches, so that every arm runs the same number of Halpern steps.  For every count: the loop of single
solves, the default batch (the host picks C), and the batch with C forced to 1, 2, 4 and 8 (B200PDLP_BATCH_CLUSTER).  Every
member of every batch is compared byte for byte with the loop's result in the same run.  Times are wall clocks around whole
calls (each call ends in a device synchronisation), after one warm-up call of each arm on two members.  Prints one JSON
document (and writes DIR/hipdlp_batch_mixed.json) with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

INTS = ("term_code", "term_iterate", "iters", "passes", "restarts", "form_cols", "form_rows", "form_nnz", "form_neq")
SCALARS = ("primal_obj", "dual_obj", "primal_feas", "dual_feas", "gap", "rel_gap")
VECTORS = ("col_value", "col_dual", "row_value", "row_dual")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             check=True).stdout.strip().splitlines()
        return [dict(zip(q.split(","), (v.strip() for v in line.split(",")))) for line in out]
    except (OSError, subprocess.CalledProcessError) as e:
        return {"error": str(e)}


def same(a, b):
    bits = lambda v: np.ascontiguousarray(v, dtype=np.float64).view(np.uint64)  # noqa: E731
    return (all(a[k] == b[k] for k in INTS) and all(bits(a[k]) == bits(b[k]) for k in SCALARS) and
            all(np.array_equal(bits(a[k]), bits(b[k])) for k in VECTORS))


def batch(lps, cluster, kw):
    if cluster:
        os.environ["B200PDLP_BATCH_CLUSTER"] = str(cluster)
    try:
        t0 = time.perf_counter()
        got = engine.solve_hipdlp_batch_mixed(lps, **kw)
        return time.perf_counter() - t0, got
    finally:
        os.environ.pop("B200PDLP_BATCH_CLUSTER", None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--counts", default="4,300")
    ap.add_argument("--m", type=int, default=30000)
    ap.add_argument("--n", type=int, default=30000)
    ap.add_argument("--per-col", type=int, default=5)
    ap.add_argument("--iters", type=int, default=400)
    a = ap.parse_args()
    from highs_b200.lp import synthetic_lp
    kw = dict(iter_limit=a.iters, tolerance=1e-12)
    counts = [int(c) for c in a.counts.split(",")]
    lps = [synthetic_lp(a.m, a.n, a.per_col, seed) for seed in range(1, max(counts) + 1)]
    arms = [None, 1, 2, 4, 8]
    for c in arms:   # warm-up: module loads, pinned and device caches
        batch(lps[:2], c, kw)
    engine.solve_hipdlp(lps[0], **kw)
    rows = []
    for count in counts:
        sub = lps[:count]
        t0 = time.perf_counter()
        alone = [engine.solve_hipdlp(lp, **kw) for lp in sub]
        t_loop = time.perf_counter() - t0
        row = {"count": count, "loop_s": t_loop, "iters": alone[0]["iters"], "nnz": alone[0]["form_nnz"]}
        for c in arms:
            t, got = batch(sub, c, kw)
            name = f"C{c}" if c else "default"
            row[f"{name}_s"] = t
            row[f"{name}_round_device_ms"] = got[0]["iter_device_ms"]
            row[f"{name}_identical"] = all(same(g, s) for g, s in zip(got, alone))
            row[f"{name}_speedup_vs_loop"] = t_loop / t
        rows.append(row)
        print(json.dumps(row), flush=True)
    doc = {"card": card(), "m": a.m, "n": a.n, "per_col": a.per_col, "iter_limit": a.iters, "rows": rows}
    print(json.dumps(doc))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "hipdlp_batch_mixed.json"), "w") as f:
            json.dump(doc, f, indent=1)
    return 0 if all(r[k] for r in rows for k in r if k.endswith("_identical")) else 1


if __name__ == "__main__":
    from highs_b200 import engine
    sys.exit(main())
