"""The batch on host arrays against the batch on LPs already in GPU memory: b200pdlp_solve_batch vs b200pdlp_solve_batch_device
(--solver hipdlp: b200pdlp_solve_hipdlp_batch vs b200pdlp_solve_hipdlp_batch_device).

Workload (as tools/batch_bench.py): every ordered-mode instance of tests/golden/instances (standard form max(n, m) <= 4096),
replicated R times, at the default tolerances and at kkt_tolerance 1e-4, each bounded by --iter-limit PDHG iterations.
With --solver hipdlp the instances are those whose HiPDLP standard form is ordered, and 1e-4 is HiPDLP's tolerance.
Three arms:
  host      solve_batch on host arrays (prologue and postsolve on host threads)
  device    solve_batch_device on LPs already resident on the GPU (prologue and postsolve on the device)
  upload    the raw LPs copied to the GPU, solve_batch_device, the four solution vectors copied back
After one warm-up of each arm, the arms run in alternating order --repeats times; all must return identical bits.  One more
call of the device arm with B200PDLP_TIMING=1 gives its laps (validation + sizing, device prologue, rounds, postsolve).
Prints one JSON line with the card's name, power limit and max SM clock read in the same run.
    python tools/batch_device_bench.py [--solver pdlp|hipdlp] [--replicas 8] [--iter-limit 500] [--repeats 2]
"""
import argparse
import glob
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from highs_b200 import engine  # noqa: E402
from highs_b200.lp import read_b2lp  # noqa: E402

INTS = ("term_code", "term_iterate", "iters", "passes", "restarts", "form_cols", "form_rows", "form_nnz", "form_neq")
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


def host_vectors(r):
    """a result dict with its vectors as numpy arrays (device arms return torch tensors)"""
    return dict(r, **{k: r[k] if isinstance(r[k], np.ndarray) else r[k].cpu().numpy() for k in VECTORS})


def identical(a, b):
    if any(a[k] != b[k] for k in INTS):
        return False
    if any(np.float64(a[k]).view(np.uint64) != np.float64(b[k]).view(np.uint64) for k in FLOATS):
        return False
    return all(np.array_equal(np.asarray(a[k]).view(np.uint64), np.asarray(b[k]).view(np.uint64)) for k in VECTORS)


def timing_laps(fn):
    """run fn() with B200PDLP_TIMING=1 and return the engine's "[b200pdlp batch device]" laps in ms (stderr captured at fd 2)"""
    os.environ["B200PDLP_TIMING"] = "1"
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+b") as f:
        os.dup2(f.fileno(), 2)
        try:
            fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["B200PDLP_TIMING"]
        f.seek(0)
        text = f.read().decode(errors="replace")
    laps = {}
    for m in re.finditer(r"\[b200pdlp batch device\]\s+(.+?)\s+([0-9.]+) ms", text):
        laps[m.group(1).strip()] = float(m.group(2))
    return laps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=8)
    ap.add_argument("--iter-limit", type=int, default=500)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--solver", choices=("pdlp", "hipdlp"), default="pdlp")
    a = ap.parse_args()
    hip = a.solver == "hipdlp"
    solve_host = engine.solve_hipdlp_batch if hip else engine.solve_batch
    solve_device = engine.solve_hipdlp_batch_device if hip else engine.solve_batch_device
    if engine.device_count() == 0:
        sys.exit("batch_device_bench.py needs a CUDA device")
    import torch
    lps = []
    for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "instances", "*.b2lp"))):
        lp = read_b2lp(p)
        f = engine.host_form_hipdlp(lp) if hip else engine.host_form(lp, 1)
        if max(f["n"], f["m"]) <= 4096:
            lps.append(lp)
    work = lps * a.replicas
    resident = [engine.lp_to_device(lp, 0) for lp in work]
    torch.cuda.synchronize()
    result = dict(card(), **(dict(solver="hipdlp") if hip else {}), instances=len(lps), replicas=a.replicas, members=len(work),
                  iter_limit=a.iter_limit, repeats=a.repeats, workloads=[])
    for name, tol in (("default", None), ("kkt1e-4", 1e-4)):
        kw = dict(iter_limit=a.iter_limit)
        if tol and hip:
            kw.update(tolerance=tol)
        elif tol:
            kw.update(tol_primal=tol, tol_dual=tol, tol_gap=tol)

        def run_host():
            t = time.perf_counter()
            r = solve_host(work, **kw)
            return time.perf_counter() - t, r

        def run_device():
            t = time.perf_counter()
            r = solve_device(resident, **kw)
            return time.perf_counter() - t, r

        def run_upload():
            t = time.perf_counter()
            r = solve_device([engine.lp_to_device(lp, 0) for lp in work], **kw)
            r = [host_vectors(x) for x in r]
            return time.perf_counter() - t, r

        arms = dict(host=run_host, device=run_device, upload=run_upload)
        for fn in arms.values():   # warm-up (module loads, allocation caches)
            fn()
        times = {k: [] for k in arms}
        same = True
        for rep in range(a.repeats):
            order = list(arms) if rep % 2 == 0 else list(arms)[::-1]
            got = {}
            for k in order:
                t, r = arms[k]()
                times[k].append(t)
                got[k] = r
            ref = got["host"]
            for k in ("device", "upload"):
                same = same and all(identical(host_vectors(x), y) for x, y in zip(got[k], ref))
        dev_result = solve_device(resident, **kw)
        laps = timing_laps(lambda: solve_device(resident, **kw))
        best = {k: min(v) for k, v in times.items()}
        result["workloads"].append(dict(
            name=name, identical_bits=same, pdhg_iterations=sum(r["iters"] for r in dev_result),
            rounds=dev_result[0]["kernel_launches"], **{f"{k}_s": [round(t, 4) for t in v] for k, v in times.items()},
            **{f"{k}_best_s": round(t, 4) for k, t in best.items()},
            device_setup_ms=round(1e3 * dev_result[0]["setup_seconds"], 2),
            device_laps_ms=laps, upload_beats_host=best["upload"] < best["host"],
            host_over_device=round(best["host"] / best["device"], 3), host_over_upload=round(best["host"] / best["upload"], 3)))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
