#!/usr/bin/env python3
"""tools/solve_device_bench.py -- one S3-shaped LP (bench.py's generator and seed: 1M x 1M, 8M nonzeros) solved from host
arrays (b200pdlp_solve / b200pdlp_solve_hipdlp) and from the same arrays in GPU memory (b200pdlp_solve_device /
b200pdlp_solve_hipdlp_device), both modes, at a fixed iteration limit.

    python tools/solve_device_bench.py [--out DIR] [--workload S3] [--iters 200] [--repeats 3]

The host arm's input arrays and result vectors are page-locked (b200pdlp_host_register), so its copies run at PCIe speed: the
comparison is with the best a host-array caller can do.  The device arm's LP is uploaded once, before any clock; its outputs
stay on the device (the call returns when they are complete).  The arms alternate, host then device, `repeats` times per mode
after one warm-up call of each.  Every call is compared byte for byte with the first host call of its mode.  Reported per arm:
setup_seconds (the result field: sizing, prologue and initial point) and the wall clock of the whole call, each call's and the
median.  Prints one JSON document (and writes DIR/solve_device.json) with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bench  # noqa: E402
from hipdlp_batch_mixed_bench import card, same  # noqa: E402
from highs_b200 import engine  # noqa: E402


def host(d):
    return {k: (v.cpu().numpy() if hasattr(v, "is_cuda") else v) for k, v in d.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--workload", default="S3", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    lp = bench.make_lp(args.workload)
    dlp = engine.lp_to_device(lp, 0)
    torch.cuda.synchronize()
    n, m = lp.num_col_, lp.num_row_
    outs = tuple(np.zeros(k) for k in (n, n, m, m))
    pinned = engine.pin_arrays(engine.lp_arrays(lp) + list(outs))
    # a tolerance no run reaches: every call runs the same iterations
    modes = {
        "pdlp": (lambda: engine.solve(lp, out_arrays=outs, iter_limit=args.iters, tol_primal=1e-15, tol_dual=1e-15, tol_gap=1e-15),
                 lambda: engine.solve_device(dlp, iter_limit=args.iters, tol_primal=1e-15, tol_dual=1e-15, tol_gap=1e-15)),
        "hipdlp": (lambda: engine.solve_hipdlp(lp, out_arrays=outs, iter_limit=args.iters, tolerance=1e-15),
                   lambda: engine.solve_hipdlp_device(dlp, iter_limit=args.iters, tolerance=1e-15)),
    }
    report = {"workload": args.workload, "n": n, "m": m, "nnz": int(lp.a_matrix_.start_[-1]), "iters": args.iters,
              "repeats": args.repeats, "host_arrays_pinned": len(pinned), "card": card(), "modes": {}}
    try:
        for mode, (solve_host, solve_dev) in modes.items():
            ref = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in solve_host().items()}   # warm-up + reference
            solve_dev()
            arms = {"host": {"setup_seconds": [], "call_seconds": []}, "device": {"setup_seconds": [], "call_seconds": []}}
            identical = True
            for _ in range(args.repeats):
                for arm, fn in (("host", solve_host), ("device", solve_dev)):
                    t0 = time.perf_counter()
                    got = fn()
                    if arm == "device":
                        torch.cuda.synchronize()
                    wall = time.perf_counter() - t0
                    arms[arm]["setup_seconds"].append(got["setup_seconds"])
                    arms[arm]["call_seconds"].append(wall)
                    identical &= same(host(got), ref)
            for a in arms.values():
                a["median_setup_seconds"] = statistics.median(a["setup_seconds"])
                a["median_call_seconds"] = statistics.median(a["call_seconds"])
            arms["identical_bits"] = bool(identical)
            arms["iters_run"] = ref["iters"]
            report["modes"][mode] = arms
    finally:
        engine.unpin_arrays(pinned)
    report["card_after"] = card()
    text = json.dumps(report, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "solve_device.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
