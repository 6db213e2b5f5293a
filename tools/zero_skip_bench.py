#!/usr/bin/env python3
"""tools/zero_skip_bench.py -- how many of the pass SpMVs' gathers read an exact zero, and what skipping them buys.

    python tools/zero_skip_bench.py --out DIR [--zeros S3,S2,...] [--ab S3,...] [--runs 3]

--zeros: for each workload, solves from the same initial point to 200, 700, 1200, 1700 and 2200 iterations and counts the
exact zeros of the returned current iterate (col_value = x, row_dual = y at the iteration limit; unscaling keeps a zero a
zero).  `gathers_skipped` weights every zero by the entries of its column (A x gathers x) or of its row (A'y gathers y), so
it is the share of the pass's gathers that read a zero.

--ab: bench.py --no-cpu-baseline on each workload with the zero-skip shape off (B200PDLP_ZERO_SKIP=0) and on, in
alternating order, `--runs` times per arm, with --dump-outputs: records `value`, the per-kernel times, the SM clocks, and a
hash of every dumped array, so that the arms can be compared bit for bit.

Writes one JSON file, DIR/zero_skip.json, with the card's name, power limit and clocks read in the same run.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

ARRAYS = ("col_value", "col_dual", "row_value", "row_dual")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             check=True).stdout.strip().splitlines()
        return [dict(zip(q.split(","), (v.strip() for v in line.split(",")))) for line in out]
    except (OSError, subprocess.CalledProcessError) as e:
        return {"error": str(e)}


def zero_counts(workloads, limits):
    import bench
    from highs_b200 import engine
    out = {}
    for w in workloads:
        lp = bench.make_lp(w)
        a = lp.a_matrix_
        start = np.asarray(a.start_, dtype=np.int64)
        col_nnz = np.diff(start)
        row_nnz = np.bincount(np.asarray(a.index_, dtype=np.int64), minlength=lp.num_row_)
        nnz = int(start[-1])
        prob = engine.Problem(lp)
        rows = []
        for k in limits:
            r = prob.solve(iter_limit=k + 1)
            zx = np.asarray(r["col_value"]) == 0.0
            zy = np.asarray(r["row_dual"]) == 0.0
            rows.append({"iter": int(r["iters"]), "x_zero": float(zx.mean()), "y_zero": float(zy.mean()),
                         "ax_gathers_skipped": float(col_nnz[zx].sum() / nnz),
                         "aty_gathers_skipped": float(row_nnz[zy].sum() / nnz)})
            print(w, json.dumps(rows[-1]), flush=True)
        prob.close()
        out[w] = rows
    return out


def bench_run(workload, arm, steps, warmup):
    env = dict(os.environ)
    if arm is not None:
        env["B200PDLP_ZERO_SKIP"] = str(arm)
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--no-cpu-baseline", "--workload", workload,
               "--steps", str(steps), "--warmup", str(warmup), "--dump-outputs", td]
        p = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
        if p.returncode != 0:
            return {"workload": workload, "arm": arm, "error": p.stderr[-2000:]}
        line = json.loads(p.stdout.strip().splitlines()[-1])
        hashes = {k: hashlib.sha256(np.load(os.path.join(td, k + ".npy")).tobytes()).hexdigest()[:16] for k in ARRAYS}
    roof = line.get("roofline") or {}
    clk = (line.get("clocks") or {}).get("timed_region") or {}
    return {"workload": workload, "arm": arm, "value": line["value"], "per_kernel_us": roof.get("per_kernel_us"),
            "restarts": line.get("restarts"), "sm_clock": clk, "hashes": hashes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--zeros", default="", help="workloads whose zero fractions to count, comma-separated")
    ap.add_argument("--ab", default="", help="workloads to time with the zero-skip shape off and on, comma-separated")
    ap.add_argument("--arms", default="0,1", help="B200PDLP_ZERO_SKIP values, alternated; 'none' leaves it unset")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    res = {"card_before": card()}
    if args.zeros:
        res["zeros"] = zero_counts(args.zeros.split(","), (200, 700, 1200, 1700, 2200))
    if args.ab:
        arms = [None if a == "none" else int(a) for a in args.arms.split(",")]
        runs = []
        for w in args.ab.split(","):
            for i in range(args.runs):
                for arm in (arms if i % 2 == 0 else arms[::-1]):
                    runs.append(bench_run(w, arm, args.steps, args.warmup))
                    print(json.dumps(runs[-1]), flush=True)
        res["runs"] = runs
        summary = {}
        for w in args.ab.split(","):
            for arm in arms:
                rr = [r for r in runs if r["workload"] == w and r["arm"] == arm and "value" in r]
                if not rr:
                    continue
                vals = [r["value"] for r in rr]
                summary[f"{w}/{arm}"] = {"value_min": min(vals), "value_max": max(vals), "value_median": float(np.median(vals)),
                                         "hashes_agree": len({json.dumps(r["hashes"], sort_keys=True) for r in rr}) == 1,
                                         "hashes": rr[0]["hashes"]}
            hs = {json.dumps(summary[f"{w}/{a}"]["hashes"], sort_keys=True) for a in arms if f"{w}/{a}" in summary}
            summary[f"{w}/identical_across_arms"] = len(hs) == 1
        res["summary"] = summary
    res["card_after"] = card()
    with open(os.path.join(args.out, "zero_skip.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res.get("summary", {}), indent=1))


if __name__ == "__main__":
    main()
