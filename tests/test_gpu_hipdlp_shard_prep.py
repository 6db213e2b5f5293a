"""The device prologue of the HiPDLP mode on several GPUs (DevicePrologue in block mode, b200pdlp_solve_hipdlp_multi with
device_prep = 0) against the host prologue it replaces there.

1. Layout parity: b200pdlp_debug_hipdlp_shard_prep_compare reports no mismatch -- the partition of the device rows and
   columns, every rank's A_g and A_g' (slices, column ids, values, long rows), the vectors in device order, the row upper
   bounds and both unscaled norms bit for bit -- on every instance fixture for 2, 3 and 4 ranks under four scaling options,
   and on LPs with long rows, every row class, shuffled columns, and fewer rows and columns than ranks.
2. Solve parity: solve_hipdlp_multi(device_prep=0), solve_hipdlp_multi(device_prep=-1) and solve_hipdlp(device_prep=-1)
   return the same iteration count, termination, term_iterate and four solution vectors byte for byte, iteration-limited and
   converged, on instances forced into tree mode (ordered_max=-1) and on synthetic LP families.
3. The device path really ran: with B200PDLP_TIMING=1 the setup lap names the sharded device prologue for device_prep=0 in
   tree mode, and not for device_prep=-1 or an ordered-mode instance.

Every case runs in a child process (this file with `child <case>`) with a hard timeout: a barrier that never completes
must not take the test session along."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

VECS = ("col_value", "col_dual", "row_value", "row_dual")
SCALINGS = [(5, 10), (7, 10), (0, 10), (5, 4)]   # (scaling_mode, ruiz_iterations)
LIMITED, CONVERGED = dict(iter_limit=400), dict(tolerance=1e-4, iter_limit=100_000)
HANDFUL = ("afiro", "adlittle", "sctest", "e226", "25fv47")
DEVICE_LAP, HOST_LAP = "HiPDLP shards: device prologue", "HiPDLP shards: host prologue"


# ----------------------------------------------------------------------------------------------------------- child side
def _tiny_lp():
    """2 rows, 3 columns: fewer rows and columns than 4 ranks"""
    from test_gpu_hipdlp_shards import _tiny_lp as tiny
    return tiny()


def _layout(out, key, lp, world, mode=5, ruiz=10):
    from highs_b200 import engine
    try:
        rep = engine.hipdlp_shard_prep_compare(lp, world, mode, ruiz)
        bad = {k: v for k, v in rep.items() if k != "ranks" and v != 0}
        for g, r in enumerate(rep["ranks"]):
            bad.update({f"r{g}.{k}": v for k, v in r.items() if v != 0})
        out[key] = "ok" if not bad else str(bad)[:300]
    except Exception as e:   # noqa: BLE001
        out[key] = f"{type(e).__name__}: {e}"[:300]


def _same(one, multi, what):
    assert multi["iters"] == one["iters"], (what, "iterations", multi["iters"], one["iters"])
    assert multi["term_code"] == one["term_code"], (what, "termination", multi["term_code"], one["term_code"])
    assert multi["term_iterate"] == one["term_iterate"], (what, "term_iterate", multi["term_iterate"], one["term_iterate"])
    for k in VECS:
        assert multi[k].tobytes() == one[k].tobytes(), (what, k, float(np.max(np.abs(multi[k] - one[k]))))


def _three_way(out, key, lp, worlds, prm, devices=None, expect=None):
    """solve_hipdlp_multi with either prologue against solve_hipdlp(device_prep=-1), byte for byte"""
    from highs_b200 import engine
    try:
        one = engine.solve_hipdlp(lp, device_prep=-1, **prm)
        if expect == "limited":
            assert one["term_code"] != 0, "converged within the iteration limit"
            assert not any(np.any(one[k]) for k in ("col_value", "row_dual")), "an iteration-limited run returns x = y = 0"
        elif expect == "converged":
            assert one["term_code"] == 0, ("did not converge", one["iters"])
        for g in worlds:
            dev = devices if devices is not None else [0] * g
            for dp in (0, -1):
                _same(one, engine.solve_hipdlp_multi(lp, g, devices=dev, device_prep=dp, **prm), f"G={g} device_prep={dp}")
        out[key] = "ok"
    except Exception as e:   # noqa: BLE001
        out[key] = f"{type(e).__name__}: {e}"[:300]


def _instances():
    from highs_b200.lp import read_b2lp
    for path in sorted(glob.glob(os.path.join(TESTS, "golden", "instances", "*.b2lp"))):
        yield os.path.basename(path)[:-5], read_b2lp(path)


def child_main(case):
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    from test_gpu_hipdlp_device_prep import long_rows_lp, mixed_rows_lp, shuffled_lp
    out = {}
    if case.startswith("layout:"):
        world = int(case.split(":")[1])
        for name, lp in _instances():
            for mode, ruiz in SCALINGS:
                _layout(out, f"{name}#{mode}/{ruiz}", lp, world, mode, ruiz)
    elif case == "layout_families":
        for name, lp in (("long_rows", long_rows_lp()), ("mixed_rows", mixed_rows_lp()), ("shuffled", shuffled_lp()),
                         ("tiny", _tiny_lp())):
            for world in (2, 3, 4):
                _layout(out, f"{name}#G{world}", lp, world)
    elif case == "solve_instances":
        lps = dict(_instances())
        for name in HANDFUL:
            for tag, prm in (("limited", LIMITED), ("tol1e-4", dict(tolerance=1e-4, iter_limit=4000))):
                _three_way(out, f"{name}#{tag}", lps[name], (2, 3, 4), dict(prm, ordered_max=-1))
    elif case == "solve_families":
        for name, lp, worlds in (("synthetic_12k_9k", synthetic_lp(12000, 9000, 6, 21), (2, 3)),
                                 ("mixed_rows_max_offset", mixed_rows_lp(), (2, 4)),
                                 ("s2_banded", synthetic_lp(100_000, 100_000, 10, 12345, band=2048), (2,)),
                                 ("long_rows", long_rows_lp(), (2,))):
            _three_way(out, f"{name}#limited", lp, worlds, LIMITED, expect="limited")
            _three_way(out, f"{name}#converged", lp, worlds, CONVERGED, expect="converged")
    elif case == "solve_edge":
        tiny = _tiny_lp()
        _three_way(out, "tiny#limited", tiny, (2, 3, 4), dict(iter_limit=40, ordered_max=-1))
        _three_way(out, "tiny#converged", tiny, (2, 3, 4), dict(CONVERGED, ordered_max=-1), expect="converged")
        lp = synthetic_lp(12000, 9000, 6, 21)
        _three_way(out, "time_limit_zero", lp, (2, 3), dict(time_limit=0.0))
        # a limit inside the run: every rank stops after the same block
        r = engine.solve_hipdlp_multi(lp, 3, devices=[0, 0, 0], device_prep=0, tolerance=1e-12, time_limit=0.3)
        ok = r["term_iterate"] == 2 and r["term_code"] != 0 and r["iters"] > 0 and r["iters"] % 40 == 0
        out["time_limit_mid_run"] = "ok" if ok else str((r["term_iterate"], r["term_code"], r["iters"]))
    elif case == "laps":   # the parent sets B200PDLP_TIMING=1 and reads the setup laps between the markers
        afiro = dict(_instances())["afiro"]
        lp = synthetic_lp(12000, 9000, 6, 21)
        for name, arg, prm in (("tree_device", lp, {}), ("tree_host", lp, dict(device_prep=-1)), ("ordered", afiro, {})):
            print(f"@@ {name}", file=sys.stderr, flush=True)
            engine.solve_hipdlp_multi(arg, 2, devices=[0, 0], iter_limit=40, **prm)
            out[name] = "ok"
        print("@@ end", file=sys.stderr, flush=True)
    elif case == "two_gpus":
        for name, lp in (("synthetic_12k_9k", synthetic_lp(12000, 9000, 6, 21)), ("mixed_rows", mixed_rows_lp())):
            _three_way(out, f"{name}#converged", lp, (2,), CONVERGED, devices=[0, 1], expect="converged")
    print(json.dumps(out), flush=True)
    return 0


# ----------------------------------------------------------------------------------------------------------- parent side
def _run_child(case, timeout=600, env_extra=None):
    env = {k: v for k, v in os.environ.items() if k not in ("B200PDLP_TIMING", "B200PDLP_DEVICE_PREP", "B200PDLP_GPUS")}
    env.update(env_extra or {})
    try:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "child", case], capture_output=True, text=True,
                           timeout=timeout, cwd=ROOT, env=env)
    except subprocess.TimeoutExpired:
        pytest.fail(f"child {case} did not finish in {timeout} s (killed)")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert lines and r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-3000:])
    out = json.loads(lines[-1])
    bad = {k: v for k, v in out.items() if v != "ok"}
    assert out and not bad, dict(list(bad.items())[:10])
    return out, r.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 4])
def test_layouts_match_host_on_instance_fixtures(world):
    out, _ = _run_child(f"layout:{world}")
    assert len(out) >= 74 * len(SCALINGS)


@pytest.mark.gpu
def test_layouts_match_host_on_lp_families():
    out, _ = _run_child("layout_families")
    assert len(out) == 12


@pytest.mark.gpu
def test_solve_matches_host_prologue_on_instances_in_tree_mode():
    out, _ = _run_child("solve_instances")
    assert len(out) == 2 * len(HANDFUL)


@pytest.mark.gpu
def test_solve_matches_host_prologue_on_lp_families():
    out, _ = _run_child("solve_families")
    assert len(out) == 8


@pytest.mark.gpu
def test_fewer_rows_than_ranks_and_time_limits():
    out, _ = _run_child("solve_edge")
    assert len(out) == 4


@pytest.mark.gpu
def test_setup_lap_names_the_prologue_that_ran():
    _, err = _run_child("laps", env_extra={"B200PDLP_TIMING": "1"})
    parts, name = {}, None
    for ln in err.splitlines():
        if ln.startswith("@@ "):
            name = ln[3:].strip()
            parts[name] = []
        elif name is not None:
            parts[name].append(ln)
    seg = {k: "\n".join(v) for k, v in parts.items()}
    assert DEVICE_LAP in seg["tree_device"] and HOST_LAP not in seg["tree_device"], seg["tree_device"][-1500:]
    assert DEVICE_LAP not in seg["tree_host"] and HOST_LAP in seg["tree_host"], seg["tree_host"][-1500:]
    assert DEVICE_LAP not in seg["ordered"] and HOST_LAP in seg["ordered"], seg["ordered"][-1500:]


@pytest.mark.gpu
def test_two_physical_gpus():
    from highs_b200 import engine
    if engine.device_count() < 2:
        pytest.skip("needs two GPUs")
    out, _ = _run_child("two_gpus")
    assert len(out) == 2


@pytest.mark.gpu
def test_through_the_shim_on_two_ranks_in_tree_mode(oracle, monkeypatch):
    """solver=hipdlp through the HiGHS shim with B200PDLP_GPUS=2 on an LP large enough for tree mode (so the shards take the
    device prologue): status and iteration count of the one-GPU drop-in.  (The shim clamps B200PDLP_GPUS to the number of
    devices, so on a box with one GPU both runs take the one-GPU solve.)"""
    from highs_b200.lp import synthetic_lp
    drv = os.path.join(os.path.dirname(oracle.DROPIN_DRIVER), "ref_driver_b200_hipdlp")
    if not os.path.exists(drv):
        pytest.skip("oracle/_ref/ref_driver_b200_hipdlp not built")
    lp = synthetic_lp(12000, 9000, 6, 21)
    opts = {"solver": "hipdlp", "presolve": "off", "pdlp_iteration_limit": 20000}
    for k in ("B200PDLP_GPUS", "B200PDLP_DEVICE_PREP", "B200PDLP_TIMING"):
        monkeypatch.delenv(k, raising=False)
    one = oracle.run_reference(lp=lp, options=opts, driver=drv, timeout=300)
    monkeypatch.setenv("B200PDLP_GPUS", "2")
    two = oracle.run_reference(lp=lp, options=opts, driver=drv, timeout=300)
    assert two["model_status_code"] == one["model_status_code"], (two["model_status"], one["model_status"])
    assert two["pdlp_iteration_count"] == one["pdlp_iteration_count"]


if __name__ == "__main__" and len(sys.argv) >= 3 and sys.argv[1] == "child":
    sys.exit(child_main(sys.argv[2]))
