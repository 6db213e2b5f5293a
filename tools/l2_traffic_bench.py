#!/usr/bin/env python3
"""tools/l2_traffic_bench.py -- time and traffic of the PDHG pass kernels, K1, K2 and K3, on the one-GPU PDLP solve.

    python tools/l2_traffic_bench.py --out DIR [--workloads S3,S3B,S5] [--roots .,OTHER_TREE] [--rounds 3]

For each workload: a warm-up solve, a timed solve of --steps iterations, then engine.Problem.bench_pass (CUDA events
around each kernel of the pass, in the pass sequence, on the iterate the solve returned).  Per kernel it reports

  us               time per launch;
  bytes            the algorithmic bytes of bench.py (matrix, epilogue vectors, each once);
  gathers          the gathers the zero-skip shape issues on the returned iterate: every entry of A whose column has a
                   nonzero in x (K2 gathers x'), every entry of A' whose row has a nonzero in y (K3 gathers y');
  gather_sectors   32 bytes per gather: on random columns (S3, S5) every gather is its own sector, so this is the
                   traffic between L2 and the SMs that the gathers cause on top of `bytes`.

--roots alternates several source trees, each built in place (this one, and for instance a checkout of an earlier
commit): each round runs every tree once, in a subprocess of its own, in alternating order, so that the trees share the
card's state.  The card's name, power limit and SM clocks are read from NVML in every subprocess, around the timing.
Writes DIR/l2_traffic.json.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def nvml_card(index=0):
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        name = pynvml.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0,
                "sm_clock_mhz": pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM),
                "sm_clock_max_mhz": pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)}
    except Exception as e:   # noqa: BLE001
        return {"error": f"NVML unavailable: {e}"[:160]}


def measure(root, workloads, steps, warmup, reps):
    """one tree: imports highs_b200 from `root` (bench.py's workloads and byte model come from this tool's tree)"""
    sys.path.insert(0, ROOT)
    import bench
    sys.path.insert(0, root)
    for k in [k for k in sys.modules if k == "highs_b200" or k.startswith("highs_b200.")]:
        del sys.modules[k]
    import numpy as np
    from highs_b200 import engine
    if engine.device_count() == 0:
        raise SystemExit("l2_traffic_bench.py needs a CUDA device")
    out = {"root": os.path.abspath(root), "engine": os.path.abspath(engine.__file__), "card_before": nvml_card(),
           "workloads": {}}
    for w in workloads:
        lp = bench.make_lp(w)
        a = lp.a_matrix_
        start = np.asarray(a.start_, dtype=np.int64)
        col_nnz = np.diff(start)
        row_nnz = np.bincount(np.asarray(a.index_, dtype=np.int64), minlength=lp.num_row_)
        prob = engine.Problem(lp)
        prob.solve(iter_limit=warmup + 1)
        r = prob.solve(iter_limit=steps + 1)
        kms = prob.bench_pass(reps)
        B = bench.algorithmic_bytes(prob.n, prob.m, prob.nnz)
        g2 = int(col_nnz[np.asarray(r["col_value"]) != 0.0].sum())
        g3 = int(row_nnz[np.asarray(r["row_dual"]) != 0.0].sum())
        us = [1e3 * v / reps for v in kms]
        out["workloads"][w] = {
            "it_per_s": steps / (r["loop_device_ms"] / 1e3),
            "K1": {"us": us[0], "bytes": B["k1"], "gbs": B["k1"] / us[0] / 1e3},
            "K2": {"us": us[1], "bytes": B["k2"], "gbs": B["k2"] / us[1] / 1e3, "gathers": g2, "gather_sectors": g2},
            "K3": {"us": us[2], "bytes": B["k3"], "gbs": B["k3"] / us[2] / 1e3, "gathers": g3, "gather_sectors": g3},
        }
        for k in ("K2", "K3"):
            e = out["workloads"][w][k]
            e["gather_bytes"] = 32 * e["gather_sectors"]
            e["gbs_with_gathers"] = (e["bytes"] + e["gather_bytes"]) / e["us"] / 1e3
        prob.close()
    out["card_after"] = nvml_card()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--workloads", default="S3,S3B,S5")
    ap.add_argument("--roots", default=ROOT, help="source trees to alternate, comma-separated (each built in place)")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    workloads = args.workloads.split(",")
    if args.child:
        print(json.dumps(measure(args.child, workloads, args.steps, args.warmup, args.reps)))
        return
    roots = [os.path.abspath(r) for r in args.roots.split(",")]
    runs = []
    for i in range(args.rounds):
        for root in (roots if i % 2 == 0 else roots[::-1]):
            cmd = [sys.executable, os.path.abspath(__file__), "--child", root, "--workloads", args.workloads,
                   "--steps", str(args.steps), "--warmup", str(args.warmup), "--reps", str(args.reps)]
            p = subprocess.run(cmd, capture_output=True, text=True)
            if p.returncode != 0:
                runs.append({"root": root, "round": i, "error": p.stderr[-2000:]})
            else:
                runs.append(dict(json.loads(p.stdout.strip().splitlines()[-1]), round=i))
            r = runs[-1]
            for w, v in r.get("workloads", {}).items():
                print(f"round {i} {root} {w}: {v['it_per_s']:.0f} it/s  K1 {v['K1']['us']:.1f}  K2 {v['K2']['us']:.1f}  "
                      f"K3 {v['K3']['us']:.1f} us  gathers K2 {v['K2']['gathers']:,}  K3 {v['K3']['gathers']:,}  "
                      f"({r['card_before'].get('name')}, {r['card_before'].get('power_limit_w')} W, "
                      f"SM {r['card_before'].get('sm_clock_mhz')} MHz)", flush=True)
            if "error" in r:
                print(f"round {i} {root}: failed\n{r['error']}", flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "l2_traffic.json"), "w") as f:
            json.dump({"runs": runs}, f, indent=1)


if __name__ == "__main__":
    main()
