"""Iteration rate and setup time of the HiPDLP mode on one GPU and on several ranks (b200pdlp_solve_hipdlp_multi).

For each workload (bench.py's S3, S3B, S3D by default) the LP's arrays are page-locked (b200pdlp_host_register) and every
arm runs a fixed number of iterations (no tolerance is reached at 1e-12): one warm-up call, then `--reps` timed calls, and
the median is reported.  Arms:
  one_gpu            solve_hipdlp, default (device prologue, engine-chosen SpMV shapes)
  one_gpu_host_prep  solve_hipdlp(device_prep=-1): host prologue, one slice per warp -- what the shards reproduce bit for bit
  shards_G           G logical shards on device 0 (a correctness vehicle: G ranks share one GPU, so expect it slower), device
                     prologue (one per device, every rank's blocks built there)
  shards_G_host_prep the same with device_prep=-1: the host prologue and host-built blocks, same layouts, same bits
  gpus_G             G physical GPUs, where the box has them
One JSON line per (workload, arm): us_per_step = loop_device_ms / iterations (checks included), setup_seconds (the engine's
clock: everything before the loop), the GPU's name and power limit.  The arms run in alternating order: forward for the
first workload, reversed for the second, and so on, so that no arm always runs first.
usage: python tools/hipdlp_shards_bench.py [--workloads S3,S3B,S3D] [--iters 800] [--reps 3] [--world 2]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run_arm(workload, arm, iters, reps, world):
    import numpy as np
    from bench import make_lp
    from highs_b200 import engine
    lp = make_lp(workload)
    pinned = engine.pin_arrays(engine.lp_arrays(lp))
    prm = dict(iter_limit=iters, tolerance=1e-12)
    if arm == "one_gpu":
        call = lambda: engine.solve_hipdlp(lp, **prm)   # noqa: E731
    elif arm == "one_gpu_host_prep":
        call = lambda: engine.solve_hipdlp(lp, device_prep=-1, **prm)   # noqa: E731
    elif arm.startswith("shards_") and arm.endswith("_host_prep"):
        call = lambda: engine.solve_hipdlp_multi(lp, world, devices=[0] * world, device_prep=-1, **prm)   # noqa: E731
    elif arm.startswith("shards_"):
        call = lambda: engine.solve_hipdlp_multi(lp, world, devices=[0] * world, **prm)   # noqa: E731
    else:
        call = lambda: engine.solve_hipdlp_multi(lp, world, devices=list(range(world)), **prm)   # noqa: E731
    try:
        rows = []
        for r in range(reps + 1):   # the first call warms the block cache and the CUDA context
            res = call()
            if r:
                rows.append((1e3 * res["loop_device_ms"] / max(res["iters"], 1), res["setup_seconds"], res["solve_seconds"]))
        a = np.array(rows)
        med = np.median(a, axis=0)
        return dict(workload=workload, arm=arm, iters=int(res["iters"]), us_per_step=float(med[0]), setup_seconds=float(med[1]),
                    solve_seconds=float(med[2]), reps=reps, us_per_step_range=[float(a[:, 0].min()), float(a[:, 0].max())],
                    setup_seconds_range=[float(a[:, 1].min()), float(a[:, 1].max())])
    finally:
        engine.unpin_arrays(pinned)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="S3,S3B,S3D")
    ap.add_argument("--iters", type=int, default=800)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--world", type=int, default=2)
    ap.add_argument("--child", default=None)
    args = ap.parse_args()
    if args.child:   # one (workload, arm) per process
        wl, arm = args.child.split(":")
        print(json.dumps(run_arm(wl, arm, args.iters, args.reps, args.world)), flush=True)
        return 0
    from highs_b200 import engine
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    gpu = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    arms = ["one_gpu", "one_gpu_host_prep", f"shards_{args.world}", f"shards_{args.world}_host_prep"]
    if engine.device_count() >= args.world:
        arms.append(f"gpus_{args.world}")
    for i, wl in enumerate(args.workloads.split(",")):
        for arm in (arms if i % 2 == 0 else arms[::-1]):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", f"{wl}:{arm}", "--iters", str(args.iters),
                                "--reps", str(args.reps), "--world", str(args.world)], capture_output=True, text=True, cwd=ROOT)
            lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            out = json.loads(lines[-1]) if r.returncode == 0 and lines else dict(workload=wl, arm=arm, error=r.stderr[-1500:])
            out["gpu"] = gpu
            print(json.dumps(out), flush=True)
    if engine.device_count() < args.world:
        print(json.dumps(dict(note=f"gpus_{args.world} not run: {engine.device_count()} device(s) visible")), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
