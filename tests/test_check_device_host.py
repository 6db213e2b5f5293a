"""The device check's entry point (b200pdlp_check_device) and the decision rules of test_gpu_check_device.py, without a GPU:
the export, argument rejections that write nothing, no CPU fallback, the ctypes mirrors of b200pdlp_check_in / _out against
the header, and the numpy restart and termination rules replayed over the oracle's trace, which they must reproduce bit for
bit before they judge the device."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT, golden_lp, load_golden, options_to_params

ERR_ARG, ERR_CUDA = -1, -2


def test_symbol_exported(engine_lib):
    from highs_b200 import engine
    assert hasattr(engine_lib, "b200pdlp_check_device")
    assert "b200pdlp_check_device" in engine.ABI_SYMBOLS


def test_structs_match_header():
    """sizeof and every field offset of b200pdlp_check_in / b200pdlp_check_out from a C compile of the header"""
    from highs_b200 import engine
    fields = {"b200pdlp_check_in": engine.CCheckIn, "b200pdlp_check_out": engine.CCheckOut}
    body = "".join(f'printf("{s} %zu\\n", sizeof({s}));' + "".join(
        f'printf("{s}.{k} %zu\\n", offsetof({s}, {k}));' for k, _ in cls._fields_) for s, cls in fields.items())
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write('#include <stdio.h>\n#include <stddef.h>\n#include "b200pdlp.h"\nint main(){' + body + "return 0;}\n")
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = dict(ln.split() for ln in subprocess.check_output([exe], text=True).splitlines())
    for s, cls in fields.items():
        assert int(got[s]) == C.sizeof(cls), s
        for k, _ in cls._fields_:
            assert int(got[f"{s}.{k}"]) == getattr(cls, k).offset, (s, k)


def test_argument_rejections_write_nothing(engine_lib):
    from highs_b200 import engine
    L = engine.lib()
    cin, cout = engine.CCheckIn(interval=40), engine.CCheckOut()
    C.memset(C.byref(cout), 0x5A, C.sizeof(cout))
    before = bytes(cout)
    vs = [np.full(8, 7.0) for _ in engine.CHECK_VECTORS]
    ptrs = [engine._p(v, engine._dp) for v in vs]
    assert L.b200pdlp_check_device(None, C.byref(cin), *ptrs, C.byref(cout)) == ERR_ARG
    assert "b200pdlp_check_device" in L.b200pdlp_last_error().decode()
    cin.light = 1
    for k in (8, 9):   # a light check needs axsum and atysum
        p = list(ptrs)
        p[k] = None
        assert L.b200pdlp_check_device(None, C.byref(cin), *p, C.byref(cout)) == ERR_ARG
    assert L.b200pdlp_check_device(None, C.byref(cin), *ptrs, None) == ERR_ARG
    assert L.b200pdlp_check_device(None, None, *ptrs, C.byref(cout)) == ERR_ARG
    assert bytes(cout) == before and all((v == 7.0).all() for v in vs)


def test_no_cpu_fallback(engine_lib):
    """no device: a tree-mode problem -- the only kind the entry point takes -- cannot be created (B200PDLP_ERR_CUDA)"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(engine.EngineError, match=r"\(-2\)"):
        engine.Problem(synthetic_lp(5000, 4000, 3, 1), ordered_max=-1)


# ---------------------------------------------------------------------------------------------- oracle trace replay
REPLAY = ["restart_lp", "adlittle", "distillation", "infeasible", "unbounded"]


def _residual_row(t, first):
    """trace columns first .. first + 3 -> the residuals the rules read (gap = pobj - dobj, as the check forms it)"""
    pobj, dobj, pf, df = t[first:first + 4]
    return dict(pobj=pobj, dobj=dobj, pfeas=pf, dfeas=df, gap=pobj - dobj,
                relgap=abs(pobj - dobj) / (1.0 + abs(pobj) + abs(dobj)))


@pytest.mark.parametrize("name", REPLAY)
def test_rules_replay_the_oracle_trace(oracle, name):
    """each check row of the oracle's trace through the numpy rules: the restart column (12) bit for bit, given columns
    1-8, beta (column 11 of the row before) and the memo the rules carry; termination where the oracle stopped and nowhere
    else; sigma = tau beta on every restart row.  A row that restarted to the average shows the average's residuals in
    columns 1-4 (the reference re-evaluates the copied iterate), so there the current iterate's score is unknown and the
    row is checked with the average as the candidate."""
    from test_gpu_check_device import decide, score
    cases = [c for c in load_golden() if c["name"] == name]
    assert cases
    restarts_seen = 0
    for case in cases:
        lp = golden_lp(case)
        prm = options_to_params(case["options"])
        f = oracle.formulate_and_scale(lp)
        res = oracle.solve(lp, trace_cap=100000, **prm)
        tr = res["trace"]
        assert len(tr) >= 2 and res["term_code"] == {7: 0, 9: 3, 10: 3, 14: 4}[case["model_status_code"]]
        tol_p = prm.get("tol_primal", 1e-7) * (1.0 + f["norm_rhs"])
        tol_d = prm.get("tol_dual", 1e-7) * (1.0 + f["norm_cost"])
        tol_gap = prm.get("tol_gap", 1e-7)
        restart_on = prm.get("restart", 1)
        memo = dict(pf_lr=0.0, df_lr=0.0, gap_lr=0.0, pf_lc=0.0, df_lc=0.0, gap_lc=0.0, last_restart_iter=0)
        beta = tr[0, 11]
        inf_big = 1e300
        for i, t in enumerate(tr):
            L, A = _residual_row(t, 1), _residual_row(t, 5)
            for Q in (L, A):   # the infeasibility quantities are not in the trace: values that never decide
                Q.update(pinf_obj=-1.0, pinf_res=inf_big, dinf_obj=1.0, dinf_res=inf_big)
            sc = dict(tol_p=tol_p, tol_d=tol_d, tol_gap=tol_gap, time_flag=0, iter=int(t[0]),
                      iter_limit=prm.get("iter_limit", 2147483647), restart_on=restart_on, beta=beta)
            last = i == len(tr) - 1
            choice = int(t[12])
            if choice == 1:
                # the candidate was the average (mu_avg <= mu_cur): give the current iterate a score that cannot win
                L = dict(A, pfeas=A["pfeas"] * 4 + 1.0, dfeas=A["dfeas"] * 4 + 1.0, gap=abs(A["gap"]) * 4 + 1.0)
            term, ti, got, memo2, branch = decide((L, A), sc, memo)
            if last and res["term_code"] == 0:
                assert term == 0 and ti == res["term_iterate"], (case["tag"], i, branch)
                continue
            if last and res["term_code"] != 0:
                assert term < 0 or (term == 4 and res["term_code"] == 4), (case["tag"], i, branch)
                continue
            assert term < 0, (case["tag"], i, "the rules stop early", branch)
            assert got == choice, (case["tag"], i, int(t[0]), got, choice, branch)
            memo = memo2
            if choice:
                restarts_seen += 1
                R = A if choice == 1 else L
                memo.update(pf_lr=R["pfeas"], df_lr=R["dfeas"], gap_lr=R["gap"], last_restart_iter=int(t[0]))
                assert t[10] == t[9] * t[11], (case["tag"], i, "sigma != tau beta")
            beta = t[11]
    if name not in ("unbounded",):
        assert restarts_seen > 0, name
