"""The tree-mode PDLP solve runs one loop whatever it is asked to report.  On one GPU and on logical shards:
- log_level=2 returns the same bytes as log_level=0 (ints, scalars, the four vectors, the trace) and prints exactly one
  line per check, from the trace row the check kernels write;
- a trace_cap below the number of checks keeps the first rows, with and without the log;
- iter_limit <= 0 runs no loop: TIMELIMIT_OR_ITERLIMIT, no iteration, no restart, and the vectors of the start point's
  postsolve (tests/golden/solve_loop_iter_limit.npz, recorded on an H100 from the engine before the loops were merged).
The log comes from C printf, so every solve runs in a child process whose stdout holds nothing else."""
import collections
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
pytestmark = pytest.mark.gpu

INTS = ("value_valid", "dual_valid", "term_code", "term_iterate", "iters", "passes", "restarts", "kernel_launches",
        "form_cols", "form_rows", "form_nnz", "form_neq", "trace_len")
SCALARS = ("primal_obj", "dual_obj", "primal_feas", "dual_feas", "gap", "rel_gap")
VECTORS = ("col_value", "col_dual", "row_value", "row_dual")
# golden instances (name, tag of the options) that restart in tree mode, and the LP of the logical-shard cases
CASES = [("adlittle", "kkt1e-4"), ("restart_lp", "kkt1e-4"), ("e226", "kkt1e-4"), ("synth_2000x2000x8_s12345", "kkt1e-4")]
SHARDS_CASE = ("adlittle", "kkt1e-4")


def _lp_and_params(name, tag):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from conftest import golden_lp, load_golden, options_to_params
    case = next(c for c in load_golden() if c["name"] == name and c["tag"] == tag)
    return golden_lp(case), options_to_params(case["options"])


def child_main(spec, out_path):
    """one solve (world 1: engine.solve in tree mode; world > 1: that many logical shards); the results of every rank go to
    out_path, nothing but the engine's log to stdout"""
    sys.path.insert(0, ROOT)
    from highs_b200 import engine
    lp, prm = _lp_and_params(spec["name"], spec["tag"])
    prm.update(spec.get("params", {}))
    if spec["world"] == 1:
        ranks = [engine.solve(lp, ordered_max=-1, trace_cap=spec["trace_cap"], **prm)]
    else:
        ranks = engine.solve_logical_shards(lp, spec["world"], trace_cap=spec["trace_cap"], **prm)
    out = {}
    for g, r in enumerate(ranks):
        for k in INTS:
            out[f"{g}_{k}"] = np.int64(r[k])
        for k in SCALARS:
            out[f"{g}_{k}"] = np.float64(r[k])
        for k in VECTORS:
            out[f"{g}_{k}"] = r[k]
        out[f"{g}_trace"] = r.get("trace", np.zeros((0, 16)))
    np.savez(out_path, world=len(ranks), **out)
    return 0


def _solve(tmp_path, label, **spec):
    """runs child_main; returns (per-rank result dicts, iterations of the printed check lines)"""
    out = tmp_path / f"{label}.npz"
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200PDLP_")}
    try:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "child", json.dumps(spec), str(out)],
                           capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    except subprocess.TimeoutExpired:
        pytest.fail(f"{label}: the solve did not finish in 600 s (child killed)")
    assert r.returncode == 0, (label, r.stdout[-2000:], r.stderr[-3000:])
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("[b200pdlp] it ")]
    assert len(lines) == len(r.stdout.splitlines()), (label, "stdout holds more than the check lines", r.stdout[-2000:])
    z = np.load(out)
    ranks = [{k[len(f"{g}_"):]: z[k] for k in z.files if k.startswith(f"{g}_")} for g in range(int(z["world"]))]
    return ranks, [int(ln.split()[2]) for ln in lines]


def _assert_same_bytes(a, b, what):
    for k in INTS + SCALARS + VECTORS + ("trace",):
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), (what, k)


def _log_case(tmp_path, name, tag, world):
    """log_level=2 vs 0, whole trace: the same bytes on every rank, one printed line per check on every rank, and the
    printed iterations are the trace's"""
    base = dict(name=name, tag=tag, world=world, trace_cap=100000)
    quiet, printed_q = _solve(tmp_path, "quiet", **base)
    loud, printed = _solve(tmp_path, "log", params=dict(log_level=2), **base)
    assert printed_q == []
    for g in range(world):
        _assert_same_bytes(quiet[g], loud[g], f"rank {g}")
        assert int(loud[g]["restarts"]) > 0 and int(loud[g]["trace_len"]) > 1, "the case must restart"
    iters = [int(t) for t in loud[0]["trace"][:, 0]]
    assert collections.Counter(printed) == collections.Counter(iters * world), (len(printed), len(iters))
    if world == 1:
        assert printed == iters


@pytest.mark.parametrize("name,tag", CASES, ids=[c[0] for c in CASES])
def test_log_changes_no_bit_one_gpu(tmp_path, name, tag):
    """one GPU, tree mode: log_level=2 vs 0 with the whole trace"""
    _log_case(tmp_path, name, tag, 1)


def test_log_changes_no_bit_logical_shards(tmp_path):
    """2 logical shards: log_level=2 vs 0 on every rank; every rank prints its lines"""
    _log_case(tmp_path, *SHARDS_CASE, 2)


def test_truncated_trace_with_and_without_log(tmp_path):
    """trace_cap below the number of checks: the first trace_cap rows, the same with the log, which still prints every check"""
    name, tag = CASES[0]
    full, _ = _solve(tmp_path, "full", name=name, tag=tag, world=1, trace_cap=100000)
    checks = int(full[0]["trace_len"])
    cap = 5
    assert checks > 2 * cap
    quiet, _ = _solve(tmp_path, "quiet", name=name, tag=tag, world=1, trace_cap=cap)
    loud, printed = _solve(tmp_path, "log", name=name, tag=tag, world=1, trace_cap=cap, params=dict(log_level=2))
    _assert_same_bytes(quiet[0], loud[0], "trace_cap 5")
    assert int(loud[0]["trace_len"]) == cap
    assert loud[0]["trace"].tobytes() == full[0]["trace"][:cap].tobytes()
    assert printed == [int(t) for t in full[0]["trace"][:, 0]]


@pytest.mark.parametrize("world", [1, 2], ids=["one_gpu", "2_shards"])
@pytest.mark.parametrize("iter_limit", [0, -1])
def test_no_loop_below_one_iteration(tmp_path, iter_limit, world):
    """iter_limit <= 0: no check and no iteration; the vectors are what the engine returned before the loops were merged"""
    got, printed = _solve(tmp_path, "limit", name=SHARDS_CASE[0], tag=SHARDS_CASE[1], world=world, trace_cap=16,
                          params=dict(iter_limit=iter_limit, log_level=2))
    want = np.load(os.path.join(GOLDEN, "solve_loop_iter_limit.npz"))
    assert printed == []
    for g in range(world):
        key = f"w{world}_l{'m1' if iter_limit < 0 else iter_limit}_r{g}"
        r = got[g]
        assert int(r["term_code"]) == int(want[key + "_term_code"]) == 4   # B200PDLP_TIMELIMIT_OR_ITERLIMIT
        assert int(r["iters"]) == 0 and int(r["restarts"]) == 0 and int(r["trace_len"]) == 0
        for k in VECTORS:
            assert r[k].tobytes() == want[f"{key}_{k}"].tobytes(), (key, k)


if __name__ == "__main__" and len(sys.argv) >= 4 and sys.argv[1] == "child":
    sys.exit(child_main(json.loads(sys.argv[2]), sys.argv[3]))
