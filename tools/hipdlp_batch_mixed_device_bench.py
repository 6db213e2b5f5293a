#!/usr/bin/env python3
"""tools/hipdlp_batch_mixed_device_bench.py -- mid-size HiPDLP LPs already in GPU memory solved by
b200pdlp_solve_hipdlp_batch_mixed_device (prologue and postsolve on the device), against b200pdlp_solve_hipdlp_batch_mixed on
host arrays and a loop of b200pdlp_solve_hipdlp over the same LPs.

    python tools/hipdlp_batch_mixed_device_bench.py [--out DIR] [--counts 4,300] [--m 30000] [--n 30000] [--per-col 5]
                                                    [--iters 400]

Members: hipdlp_batch_mixed_bench.py's -- synthetic_lp(m, n, per_col, seed) for seeds 1..count, a fixed iteration limit and a
tolerance (1e-12) no member reaches, so that every arm runs the same number of Halpern steps.  Arms per count: the loop of
single solves; the host-array batch and the device-array batch, each at the default cluster size C and at C = 8
(B200PDLP_BATCH_CLUSTER).  The device arm's LPs are uploaded before its clock starts; its outputs stay on the device (the
clock stops when the call returns, i.e. when they are complete).  Every member of every arm is compared byte for byte with the
loop's result in the same run.  Times are wall clocks around whole calls, after one warm-up call of each arm on two members.
One more device call with B200PDLP_TIMING=1 records its laps.  Prints one JSON document (and writes
DIR/hipdlp_batch_mixed_device.json) with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

from hipdlp_batch_mixed_bench import card, same  # noqa: E402


def timed(fn, cluster):
    if cluster:
        os.environ["B200PDLP_BATCH_CLUSTER"] = str(cluster)
    try:
        t0 = time.perf_counter()
        got = fn()
        return time.perf_counter() - t0, got
    finally:
        os.environ.pop("B200PDLP_BATCH_CLUSTER", None)


def host(d):
    return {k: (v.cpu().numpy() if hasattr(v, "is_cuda") else v) for k, v in d.items()}


def laps(dlps, kw):
    """the device arm's B200PDLP_TIMING=1 laps (ms by name) and its tree-member line"""
    os.environ["B200PDLP_TIMING"] = "1"
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            engine.solve_hipdlp_batch_mixed_device(dlps, **kw)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["B200PDLP_TIMING"]
        f.seek(0)
        text = f.read()
    out = {m.group(1).strip(): float(m.group(2)) for m in re.finditer(r"\[b200pdlp batch device\]\s+(.+?)\s+([\d.]+) ms", text)}
    m = re.search(r"tree members (\d+), cluster of C = (\d+)", text)
    if m:
        out["cluster"] = int(m.group(2))
    return out


def main():
    import torch  # noqa: F401  (the device arm's tensors)
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
    dlps_all = [engine.lp_to_device(lp, 0) for lp in lps]
    arms = {"host": lambda sub, dsub: engine.solve_hipdlp_batch_mixed(sub, **kw),
            "device": lambda sub, dsub: engine.solve_hipdlp_batch_mixed_device(dsub, **kw)}
    for c in (None, 8):   # warm-up: module loads, pinned and device caches
        for fn in arms.values():
            timed(lambda: fn(lps[:2], dlps_all[:2]), c)
    engine.solve_hipdlp(lps[0], **kw)
    rows = []
    for count in counts:
        sub, dsub = lps[:count], dlps_all[:count]
        t0 = time.perf_counter()
        alone = [engine.solve_hipdlp(lp, **kw) for lp in sub]
        t_loop = time.perf_counter() - t0
        row = {"count": count, "loop_s": t_loop, "iters": alone[0]["iters"], "nnz": alone[0]["form_nnz"]}
        for name, fn in arms.items():
            for c in (None, 8):
                t, got = timed(lambda: fn(sub, dsub), c)
                tag = f"{name}_{'C8' if c else 'default'}"
                row[f"{tag}_s"] = t
                row[f"{tag}_setup_s"] = got[0]["setup_seconds"]
                row[f"{tag}_round_device_ms"] = got[0]["iter_device_ms"]
                row[f"{tag}_identical"] = all(same(host(g), s) for g, s in zip(got, alone))
                row[f"{tag}_speedup_vs_loop"] = t_loop / t
        row["device_laps_ms"] = laps(dsub, kw)
        rows.append(row)
        print(json.dumps(row), flush=True)
    doc = {"card": card(), "m": a.m, "n": a.n, "per_col": a.per_col, "iter_limit": a.iters, "rows": rows}
    print(json.dumps(doc))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "hipdlp_batch_mixed_device.json"), "w") as f:
            json.dump(doc, f, indent=1)
    return 0 if all(r[k] for r in rows for k in r if k.endswith("_identical")) else 1


if __name__ == "__main__":
    from highs_b200 import engine
    sys.exit(main())
