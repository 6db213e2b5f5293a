"""The HiPDLP mode on several GPUs (b200pdlp_solve_hipdlp_multi) returns the one-GPU bits.

Rank g computes whole rows of A and whole rows of A' in the one-GPU entry order, and every check sum runs over full
vectors with the one-GPU kernels, so a G-rank solve must equal engine.solve_hipdlp(lp, device_prep=-1, **same params)
byte for byte: iteration count, term_code, term_iterate and all four solution vectors.  Most cases run G logical shards
on device 0 (the same kernels, barriers and peer stores as G GPUs); two physical GPUs run where a box has them.

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
LIMITED, CONVERGED = dict(iter_limit=400), dict(tolerance=1e-4, iter_limit=100_000)
HANDFUL = ("afiro", "adlittle", "sctest", "e226", "25fv47")


# ----------------------------------------------------------------------------------------------------------- child side
def _tiny_lp():
    """2 rows, 3 columns: fewer rows and columns than 4 ranks"""
    from highs_b200.lp import HighsLp, HighsSparseMatrix, kHighsInf
    n, m = 3, 2
    return HighsLp(n, m, np.array([1.0, 2.0, 1.5]), np.zeros(n), np.full(n, kHighsInf), np.array([1.0, 0.5]),
                   np.array([kHighsInf, 4.0]), HighsSparseMatrix(n, m, np.array([0, 2, 3, 4], dtype=np.int32),
                                                                  np.array([0, 1, 1, 0], dtype=np.int32),
                                                                  np.array([1.0, 2.0, 3.0, 1.0])), 1, 0.0, "tiny")


def _same(one, multi, what):
    assert multi["iters"] == one["iters"], (what, "iterations", multi["iters"], one["iters"])
    assert multi["term_code"] == one["term_code"], (what, "termination", multi["term_code"], one["term_code"])
    assert multi["term_iterate"] == one["term_iterate"], (what, "term_iterate", multi["term_iterate"], one["term_iterate"])
    for k in VECS:
        assert multi[k].tobytes() == one[k].tobytes(), (what, k, float(np.max(np.abs(multi[k] - one[k]))))


def _compare(out, key, lp, worlds, prm, devices=None, expect=None):
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
            multi = engine.solve_hipdlp_multi(lp, g, devices=dev, **prm)
            _same(one, multi, f"G={g}")
            # the sharded path ran: its steps launch two barriers and its checks two gathers more than one GPU's
            assert multi["iters"] == 0 or multi["kernel_launches"] > one["kernel_launches"], (multi["kernel_launches"], one["kernel_launches"])
        print(f"{key}: iters {one['iters']} term {one['term_code']} launches {one['kernel_launches']} (one GPU)", file=sys.stderr)
        out[key] = "ok"
    except Exception as e:   # noqa: BLE001
        out[key] = f"{type(e).__name__}: {e}"[:300]


def _families():
    from highs_b200.lp import synthetic_lp
    from test_gpu_hipdlp_device_prep import long_rows_lp, mixed_rows_lp
    return {"synthetic_12k_9k": (synthetic_lp(12000, 9000, 6, 21), (2, 3, 4)),
            "mixed_rows_max_offset": (mixed_rows_lp(), (2, 3, 4)),
            "s2_banded": (synthetic_lp(100_000, 100_000, 10, 12345, band=2048), (2,)),
            "long_rows": (long_rows_lp(), (2, 4))}


def child_main(case):
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    out = {}
    if case == "instances":
        for path in sorted(glob.glob(os.path.join(TESTS, "golden", "instances", "*.b2lp"))):
            name = os.path.basename(path)[:-5]
            lp = read_b2lp(path)
            if lp.a_matrix_.numNz() > 200000:
                continue
            worlds = (2, 3, 4) if name in HANDFUL else (2,)
            for tag, prm in (("limited", LIMITED), ("tol1e-4", dict(tolerance=1e-4, iter_limit=4000))):
                _compare(out, f"{name}#{tag}", lp, worlds, prm)
    elif case == "families":
        for name, (lp, worlds) in _families().items():
            _compare(out, f"{name}#limited", lp, worlds, LIMITED, expect="limited")
            _compare(out, f"{name}#converged", lp, worlds, CONVERGED, expect="converged")
    elif case == "few_rows":
        lp = _tiny_lp()
        _compare(out, "tiny#limited", lp, (2, 3, 4), dict(iter_limit=40))
        _compare(out, "tiny#converged", lp, (2, 3, 4), CONVERGED, expect="converged")
    elif case == "time_limit":
        from highs_b200.lp import synthetic_lp
        lp = synthetic_lp(12000, 9000, 6, 21)
        # time_limit = 0: before the first block, as on one GPU
        _compare(out, "zero", lp, (2, 3), dict(time_limit=0.0))
        r = engine.solve_hipdlp_multi(lp, 3, devices=[0, 0, 0], time_limit=0.0)
        out["zero_term_iterate"] = "ok" if (r["term_iterate"], r["iters"]) == (2, 0) else str((r["term_iterate"], r["iters"]))
        # a limit inside the run: every rank stops after the same block (otherwise a barrier would never complete)
        r = engine.solve_hipdlp_multi(lp, 3, devices=[0, 0, 0], tolerance=1e-12, time_limit=0.3)
        ok = r["term_iterate"] == 2 and r["term_code"] != 0 and r["iters"] > 0 and r["iters"] % 40 == 0
        out["mid_run"] = "ok" if ok else str((r["term_iterate"], r["term_code"], r["iters"]))
    elif case == "api":
        from highs_b200.lp import synthetic_lp
        lp = synthetic_lp(3000, 2500, 6, 11)
        try:   # ngpus = 1 is the one-GPU solve itself, whatever the prologue
            one = engine.solve_hipdlp(lp, **CONVERGED)
            _same(one, engine.solve_hipdlp_multi(lp, 1, **CONVERGED), "G=1")
            out["ngpus_1"] = "ok"
        except Exception as e:   # noqa: BLE001
            out["ngpus_1"] = f"{type(e).__name__}: {e}"[:300]
        try:
            engine.solve_hipdlp_multi(lp, 17, devices=[0] * 17)
            out["ngpus_17"] = "no error"
        except engine.EngineError as e:
            out["ngpus_17"] = "ok" if "(-1)" in str(e) else str(e)[:300]
    elif case == "two_gpus":
        from highs_b200.lp import synthetic_lp
        from test_gpu_hipdlp_device_prep import mixed_rows_lp
        for name, lp in (("synthetic_12k_9k", synthetic_lp(12000, 9000, 6, 21)), ("mixed_rows", mixed_rows_lp())):
            _compare(out, f"{name}#converged", lp, (2,), CONVERGED, devices=[0, 1], expect="converged")
    print(json.dumps(out), flush=True)
    return 0


# ----------------------------------------------------------------------------------------------------------- parent side
def _run_child(case, timeout=600):
    try:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "child", case], capture_output=True, text=True,
                           timeout=timeout, cwd=ROOT)
    except subprocess.TimeoutExpired:
        pytest.fail(f"child {case} did not finish in {timeout} s (killed)")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert lines and r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-3000:])
    out = json.loads(lines[-1])
    bad = {k: v for k, v in out.items() if v != "ok"}
    assert out and not bad, dict(list(bad.items())[:10])
    return out


@pytest.mark.gpu
def test_instance_fixtures_match_one_gpu():
    out = _run_child("instances")
    assert len(out) >= 2 * 60


@pytest.mark.gpu
def test_synthetic_families_match_one_gpu():
    assert len(_run_child("families")) == 8


@pytest.mark.gpu
def test_fewer_rows_and_columns_than_ranks():
    assert len(_run_child("few_rows")) == 2


@pytest.mark.gpu
def test_time_limit_stops_every_rank_at_the_same_block():
    assert len(_run_child("time_limit")) == 3


@pytest.mark.gpu
def test_one_rank_and_too_many_ranks():
    assert len(_run_child("api")) == 2


@pytest.mark.gpu
def test_two_physical_gpus():
    from highs_b200 import engine
    if engine.device_count() < 2:
        pytest.skip("needs two GPUs")
    assert len(_run_child("two_gpus")) == 2


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["afiro", "adlittle"])
def test_through_the_shim_on_two_ranks(oracle, name, monkeypatch):
    """solver=hipdlp through the HiGHS shim with B200PDLP_GPUS=2: status and iteration count of the one-GPU drop-in"""
    from highs_b200.lp import read_b2lp
    drv = os.path.join(os.path.dirname(oracle.DROPIN_DRIVER), "ref_driver_b200_hipdlp")
    if not os.path.exists(drv):
        pytest.skip("oracle/_ref/ref_driver_b200_hipdlp not built")
    lp = read_b2lp(os.path.join(TESTS, "golden", "instances", name + ".b2lp"))
    opts = {"solver": "hipdlp", "presolve": "off", "pdlp_iteration_limit": 8000}
    one = oracle.run_reference(lp=lp, options=opts, driver=drv)
    monkeypatch.setenv("B200PDLP_GPUS", "2")
    two = oracle.run_reference(lp=lp, options=opts, driver=drv)
    assert two["model_status_code"] == one["model_status_code"], (two["model_status"], one["model_status"])
    assert two["pdlp_iteration_count"] == one["pdlp_iteration_count"]


if __name__ == "__main__" and len(sys.argv) >= 3 and sys.argv[1] == "child":
    sys.exit(child_main(sys.argv[2]))
