"""Setup and postsolve time of the HiPDLP mode (b200pdlp_solve_hipdlp), device prologue against host prologue.

For each workload (bench.py's S3, S3B, S3D by default) the LP's arrays are page-locked (b200pdlp_host_register), then
solve_hipdlp runs with the default device-resident prologue and with device_prep=-1 (host threads), a warm-up call first
and `--reps` timed calls each.  One JSON line per (workload, prologue):
  setup_seconds      everything before the iteration loop (the engine's own clock)
  postsolve_seconds  wall - setup - solve: the download and the un-scaling / un-permuting / row_value = A x
  shapes             the `SpMV shapes:` line B200PDLP_TIMING prints (the device prologue path only)
  value / e2e        iterations and end-to-end wall time of the call
usage: python tools/hipdlp_setup_bench.py [--workloads S3,S3B,S3D] [--iters 400] [--reps 3]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def one(workload, iters, reps, device_prep):
    import numpy as np
    from bench import make_lp
    from highs_b200 import engine
    lp = make_lp(workload)
    pinned = engine.pin_arrays(engine.lp_arrays(lp))
    try:
        rows = []
        for r in range(reps + 1):   # the first call warms the block cache and the CUDA context
            t0 = time.perf_counter()
            res = engine.solve_hipdlp(lp, iter_limit=iters, device_prep=device_prep)
            wall = time.perf_counter() - t0
            if r:
                rows.append((res["setup_seconds"], wall - res["setup_seconds"] - res["solve_seconds"], wall, res["iters"]))
        a = np.array([x[:3] for x in rows])
        med = np.median(a, axis=0)
        return dict(workload=workload, prologue="device" if device_prep == 0 else "host", setup_seconds=float(med[0]),
                    postsolve_seconds=float(med[1]), value=int(rows[-1][3]), e2e=float(med[2]), reps=reps)
    finally:
        engine.unpin_arrays(pinned)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="S3,S3B,S3D")
    ap.add_argument("--iters", type=int, default=400)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--child", default=None)
    args = ap.parse_args()
    if args.child:   # one (workload, prologue) per process, so that B200PDLP_TIMING's lines belong to it
        wl, dp = args.child.split(":")
        print(json.dumps(one(wl, args.iters, args.reps, int(dp))), flush=True)
        return 0
    import torch
    gpu = torch.cuda.get_device_name(0)
    for wl in args.workloads.split(","):
        for dp in (0, -1):
            env = dict(os.environ, B200PDLP_TIMING="1")
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", f"{wl}:{dp}", "--iters", str(args.iters),
                                "--reps", str(args.reps)], capture_output=True, text=True, env=env, cwd=ROOT)
            lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            if r.returncode != 0 or not lines:
                print(json.dumps(dict(workload=wl, device_prep=dp, error=r.stderr[-1500:])))
                continue
            out = json.loads(lines[-1])
            m = re.findall(r"SpMV shapes: (.+)", r.stderr)
            out["shapes"] = m[-1].strip() if m else "one slice per warp (host prologue: no shape choice)"
            norms = re.findall(r"ordered \|c\|\^2, \|b\|\^2 .*?([\d.]+) ms", r.stderr)
            if norms:
                out["ordered_norms_ms"] = float(norms[-1])
            out["gpu"] = gpu
            print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
