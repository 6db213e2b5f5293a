"""HiGHS's post-solve KKT assessment (lpKktCheck) of a whole batch of solutions: four ways to judge the same results.

Workload (as tools/batch_device_bench.py): every ordered-mode instance of tests/golden/instances (standard form
max(n, m) <= 4096), replicated R times, solved once by solve_batch_device with at most --iter-limit PDHG iterations.  Each
member's incoming model status is what the solver's termination maps to.  Four arms assess the results:
  host_loop      kkt_check(on_device=False) per member (the sequential host twin)
  device_loop    kkt_check per member (the single device check: its own stream, allocations and a dozen launches each)
  batch          kkt_check_batch on the host result dicts (one packed upload, one launch, one read-back)
  batch_device   kkt_check_batch_device on the CUDA-tensor results of solve_batch_device (nothing copied but descriptors)
The loops and batch take host vectors, copied from the device results once before timing.  After one warm-up of each arm,
the arms run in alternating order --repeats times.  Both batch arms must equal the host loop bit for bit (any NaN matching
any NaN).  One more call of each batch arm with B200PDLP_TIMING=1 gives its laps.  Prints one JSON line with the card's
name, power limit and max SM clock read in the same run.
    python tools/kkt_batch_bench.py [--replicas 8] [--iter-limit 500] [--repeats 3]
"""
import argparse
import glob
import json
import math
import os
import re
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from highs_b200 import engine  # noqa: E402
from highs_b200.lp import read_b2lp  # noqa: E402

VECTORS = ("col_value", "col_dual", "row_value", "row_dual")


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                      text=True, timeout=30).strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return dict(card=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # (the measurement itself still needs the GPU: engine calls fail without one)
        return dict(card=f"unknown ({e})", power_limit="unknown", max_sm_clock="unknown")


def model_status(term_code, iters, iter_limit):
    """cuPDLP termination -> HighsModelStatus code before lpKktCheck (CupdlpWrapper.cpp:220-251)"""
    return {0: 7, 1: 8, 2: 10, 3: 9}.get(term_code, 14 if iters >= iter_limit - 1 else 13)


def same_info(a, b):
    for k, w in b.items():
        g = a[k]
        if isinstance(w, float):
            if not ((math.isnan(g) and math.isnan(w)) or struct.pack("<d", g) == struct.pack("<d", w)):
                return False
        elif g != w:
            return False
    return True


def timing_laps(fn):
    """run fn() with B200PDLP_TIMING=1 and return the engine's "[b200pdlp kkt batch]" laps in ms (stderr captured at fd 2)"""
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
    return {m.group(1).strip(): float(m.group(2)) for m in re.finditer(r"\[b200pdlp kkt batch\]\s+(.+?)\s+([0-9.]+) ms", text)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replicas", type=int, default=8)
    ap.add_argument("--iter-limit", type=int, default=500)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if engine.device_count() == 0:
        sys.exit("kkt_batch_bench.py needs a CUDA device")
    import torch
    lps = []
    for p in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "instances", "*.b2lp"))):
        lp = read_b2lp(p)
        f = engine.host_form(lp, 1)
        if max(f["n"], f["m"]) <= 4096:
            lps.append(lp)
    work = lps * a.replicas
    resident = [engine.lp_to_device(lp, 0) for lp in work]
    res = engine.solve_batch_device(resident, iter_limit=a.iter_limit)
    torch.cuda.synchronize()
    statuses = [model_status(r["term_code"], r["iters"], a.iter_limit) for r in res]
    sols = [{k: r[k].cpu().numpy() for k in VECTORS} for r in res]

    def host_loop():
        return [engine.kkt_check(lp, s, model_status=st, on_device=False) for lp, s, st in zip(work, sols, statuses)]

    def device_loop():
        return [engine.kkt_check(lp, s, model_status=st) for lp, s, st in zip(work, sols, statuses)]

    def batch():
        return engine.kkt_check_batch(work, sols, model_status=statuses)

    def batch_device():
        return engine.kkt_check_batch_device(resident, res, model_status=statuses)

    arms = dict(host_loop=host_loop, device_loop=device_loop, batch=batch, batch_device=batch_device)
    for fn in arms.values():   # warm-up (module loads, allocation caches)
        fn()
    times = {k: [] for k in arms}
    identical = {"batch": True, "batch_device": True}
    for rep in range(a.repeats):
        order = list(arms) if rep % 2 == 0 else list(arms)[::-1]
        got = {}
        for k in order:
            t = time.perf_counter()
            got[k] = arms[k]()
            times[k].append(time.perf_counter() - t)
        for k in identical:
            identical[k] = identical[k] and len(got[k]) == len(work) and all(
                same_info(x, y) for x, y in zip(got[k], got["host_loop"]))
    best = {k: min(v) for k, v in times.items()}
    result = dict(card(), instances=len(lps), replicas=a.replicas, members=len(work), iter_limit=a.iter_limit,
                  repeats=a.repeats, identical=identical, **{f"{k}_s": [round(t, 5) for t in v] for k, v in times.items()},
                  **{f"{k}_best_s": round(t, 5) for k, t in best.items()},
                  **{f"{k}_range_s": round(max(v) - min(v), 5) for k, v in times.items()},
                  batch_laps_ms=timing_laps(batch), batch_device_laps_ms=timing_laps(batch_device),
                  device_loop_over_batch_device=round(best["device_loop"] / best["batch_device"], 1),
                  host_loop_over_batch_device=round(best["host_loop"] / best["batch_device"], 1))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
