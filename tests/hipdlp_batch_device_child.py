"""Child process of tests/test_gpu_hipdlp_batch_device.py (own process: a faulting kernel must not poison the CUDA context of
the test session).  Runs one named case of b200pdlp_solve_hipdlp_batch_device against b200pdlp_solve_hipdlp_batch on the same
LPs from host arrays.  "Identical" = byte equality of the ints (status, iterate, iterations, passes, restarts, form
dimensions), the six residual scalars and the four HighsSolution vectors; no input tensor may change.
usage: python tests/hipdlp_batch_device_child.py CASE   -> one JSON line {CASE: "ok" | error text}"""
import ctypes as C
import json
import os
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

from highs_b200 import engine  # noqa: E402
from highs_b200.lp import HighsLp, HighsSparseMatrix, synthetic_lp  # noqa: E402
from hipdlp_batch_child import (INTS, SCALARS, VARIANTS, VECTORS, golden, instances, lp_from_dense, mixed_lp,  # noqa: E402
                                no_rows_lp, small_set, zero_optimal_lp)


def _bits(v):
    return np.ascontiguousarray(v, dtype=np.float64).view(np.uint64)


def _host(t):
    return t.cpu().numpy()


def assert_same(dev, host, what):
    for k in INTS:
        assert dev[k] == host[k], (what, k, dev[k], host[k])
    for k in SCALARS:
        assert _bits(dev[k]) == _bits(host[k]), (what, k, dev[k], host[k])
    for k in VECTORS:
        assert np.array_equal(_bits(_host(dev[k])), _bits(host[k])), (what, k)


def _snapshot(dlps):
    return [{k: _host(v).tobytes() for k, v in d.items() if hasattr(v, "is_cuda")} for d in dlps]


def _assert_unchanged(dlps, snap):
    for i, (d, s) in enumerate(zip(dlps, snap)):
        for k, b in s.items():
            assert _host(d[k]).tobytes() == b, (i, k)


def device_vs_host(named, **kw):
    """solve_hipdlp_batch_device on device copies of the LPs of `named` against solve_hipdlp_batch on the host arrays"""
    lps = [lp for _, lp in named]
    dlps = [engine.lp_to_device(lp, 0) for lp in lps]
    snap = _snapshot(dlps)
    got = engine.solve_hipdlp_batch_device(dlps, **kw)
    want = engine.solve_hipdlp_batch(lps, **kw)
    assert len(got) == len(named)
    for (nm, _), g, w in zip(named, got, want):
        assert_same(g, w, nm)
    _assert_unchanged(dlps, snap)
    return got


# ---- synthetic members
def edge_lps():
    """every row class (FREE rows and rows bounded at +-1e25 among them), columns stored unsorted with repeated rows of
    different values, empty rows and columns, an LP without rows, a maximisation with an offset"""
    inf = np.inf
    af = golden("afiro")
    a = af.a_matrix_
    # afiro with a ranged, a free and a 1e25-bounded empty row appended and two empty columns in front
    start = np.concatenate([[0, 0], a.start_]).astype(np.int32)
    empty = HighsLp(af.num_col_ + 2, af.num_row_ + 3, np.concatenate([[1.0, -1.0], af.col_cost_]),
                    np.concatenate([[0.0, -1.0], af.col_lower_]), np.concatenate([[1.0, 2.0], af.col_upper_]),
                    np.concatenate([af.row_lower_, [-1.0, -inf, -1e25]]), np.concatenate([af.row_upper_, [1.0, inf, 1e25]]),
                    HighsSparseMatrix(af.num_col_ + 2, af.num_row_ + 3, start, a.index_.copy(), a.value_.copy()))
    maxi = golden("afiro")
    maxi.col_cost_ = -maxi.col_cost_
    maxi.sense_, maxi.offset_ = -1, 3.5
    # columns stored in descending row order, and every third column with one of its rows repeated at another value
    rev = mixed_lp(4)
    a = rev.a_matrix_
    idx, val, st = [], [], [0]
    for j in range(rev.num_col_):
        s, e = a.start_[j], a.start_[j + 1]
        ci, cv = list(a.index_[s:e][::-1]), list(a.value_[s:e][::-1])
        if j % 3 == 0 and ci:
            ci.insert(1 % (len(ci) + 1), ci[0])
            cv.insert(1 % (len(cv) + 1), -0.5 * cv[0] + 0.25)
        idx += ci
        val += cv
        st.append(len(idx))
    rev.a_matrix_ = HighsSparseMatrix(rev.num_col_, rev.num_row_, np.asarray(st, dtype=np.int32),
                                      np.asarray(idx, dtype=np.int32), np.asarray(val, dtype=np.float64))
    named = [("empty_rows_cols", empty), ("maximise_offset", maxi), ("unsorted_repeated", rev), ("no_rows", no_rows_lp())]
    named += [(f"mixed{s}", mixed_lp(s)) for s in (1, 2, 3)]
    return named


# ---- cases
def case_instances(vi):
    def run():
        inst = instances()
        assert len(inst) > 40, len(inst)
        device_vs_host(inst, **VARIANTS[vi])
    return run


def case_limits():
    named = small_set() + edge_lps()
    for lim in (0, 1, 40, 41, 80):
        device_vs_host(named, iter_limit=lim, tolerance=1e-9)
    got = device_vs_host(named, time_limit=0.0)
    assert all(g["iters"] == 0 and g["term_iterate"] == 2 for g in got)


def case_synthetic():
    named = edge_lps()
    got = device_vs_host(named, iter_limit=2000, tolerance=1e-6)
    assert got[3]["form_rows"] == 0
    f = engine.host_form_hipdlp(named[0][1])
    assert f["n"] >= named[0][1].num_col_ + 3   # the appended ranged, free and 1e25 rows have slack columns


def case_scaling():
    named = small_set() + edge_lps()
    for mode in (0, 1, 2, 4, 5, 7):
        for ruiz in (0, 3, 10):
            for strategy in (0, 3):
                device_vs_host(named, iter_limit=200, tolerance=1e-5, scaling_mode=mode, ruiz_iterations=ruiz,
                               step_size_strategy=strategy)


def case_converged_at_zero():
    named = [("distillation", golden("distillation")), ("zero_optimal", zero_optimal_lp()), ("adlittle", golden("adlittle"))]
    got = device_vs_host(named, iter_limit=4000)
    assert got[1]["iters"] == 0 and got[1]["term_name"] == "OPTIMAL", (got[1]["iters"], got[1]["term_name"])
    assert got[0]["iters"] >= 200 and got[2]["iters"] >= 200, (got[0]["iters"], got[2]["iters"])


def case_replicated_576():
    inst = instances()
    named = (inst * 8)[:576]
    while len(named) < 576:
        named.append(inst[0])
    device_vs_host(named, iter_limit=100)


def case_prep_compare():
    named = instances() + edge_lps()
    for mode in (0, 1, 2, 4, 5, 7):
        for ruiz in ((0, 10) if mode & 1 else (10,)):
            reps = engine.hipdlp_batch_prep_compare([lp for _, lp in named], scaling_mode=mode, ruiz_iterations=ruiz)
            bad = {nm: {k: v for k, v in r.items() if v != 0} for (nm, _), r in zip(named, reps) if any(v != 0 for v in r.values())}
            assert not bad, (mode, ruiz, bad)


# ---- errors: ERR_ARG naming the member, nothing written
def _raw_call(dlps, **params):
    """b200pdlp_solve_hipdlp_batch_device through the C ABI with NaN-filled device outputs and sentinel result fields"""
    import torch
    L = engine.lib()
    L.b200pdlp_solve_hipdlp_batch_device.argtypes = [C.c_int32, C.POINTER(engine.CLp), C.POINTER(engine.CHipdlpParams),
                                                     C.POINTER(engine.CResult)]
    count = len(dlps)
    clps, cres, outs = (engine.CLp * count)(), (engine.CResult * count)(), []
    for i, d in enumerate(dlps):
        clps[i] = d if isinstance(d, engine.CLp) else engine.make_clp_device(d)
        n, m = clps[i].num_col, clps[i].num_row
        v = [torch.full((k,), float("nan"), dtype=torch.float64, device="cuda") for k in (n, n, m, m)]
        cres[i].col_value, cres[i].col_dual, cres[i].row_value, cres[i].row_dual = (C.cast(C.c_void_p(t.data_ptr()), engine._dp) for t in v)
        cres[i].term_code, cres[i].iters, cres[i].setup_seconds = -7, -7, -7.0
        outs.append(v)
    prm = engine._hipdlp_params(params)
    rc = L.b200pdlp_solve_hipdlp_batch_device(count, clps, C.byref(prm), cres)
    for i in range(count):
        assert cres[i].term_code == -7 and cres[i].iters == -7 and cres[i].setup_seconds == -7.0, i
        assert all(bool(t.isnan().all()) for t in outs[i]), i
    return rc, L.b200pdlp_last_error().decode()


def case_errors():
    lps = [golden(nm) for nm in ("afiro", "avgas", "adlittle", "blending")]
    dlps = [engine.lp_to_device(lp, 0) for lp in lps]
    snap = _snapshot(dlps)
    # a host pointer in member 2
    clp2 = engine.make_clp_device(dlps[2])
    clp2.col_cost = engine._p(lps[2].col_cost_, engine._dp)
    rc, msg = _raw_call(dlps[:2] + [clp2] + dlps[3:])
    assert rc == -1 and "member 2: col_cost is not device memory" in msg, msg
    # malformed a_index (member 1) and a_start (member 3): the lower one is named
    bad_index = dict(dlps[1])
    bad_index["a_index"] = bad_index["a_index"].clone()
    bad_index["a_index"][5] = lps[1].num_row_
    decreasing = dict(dlps[3])
    decreasing["a_start"] = decreasing["a_start"].clone()
    decreasing["a_start"][1] = decreasing["a_start"][2] + 1
    rc, msg = _raw_call([dlps[0], bad_index, dlps[2], decreasing])
    assert rc == -1 and "member 1: " in msg and "a_index entry outside" in msg, msg
    rc, msg = _raw_call([dlps[0], dlps[1], dlps[2], decreasing])
    assert rc == -1 and "member 3: " in msg and "non-decreasing" in msg, msg
    # 100 rows bounded at 1e25 on one side: ranged rows with a slack each for HiPDLP (4100 columns), >= rows for the 1e20 rule
    big = synthetic_lp(100, 4000, 3, 1)
    big.row_upper_ = np.full(100, 1e25)
    assert engine.host_form(big, 1)["n"] == 4000 and engine.host_form_hipdlp(big)["n"] == 4100
    dbig = engine.lp_to_device(big, 0)
    rc, msg = _raw_call([dlps[0], dbig, dlps[2]])
    assert rc == -1 and "member 1: standard form 100 x 4100 exceeds ordered_max = 4096" in msg, msg
    _assert_unchanged(dlps, snap)
    _assert_unchanged([bad_index, decreasing, dbig], _snapshot([bad_index, decreasing, dbig]))


CASES = {f"instances{v}": case_instances(v) for v in range(len(VARIANTS))}
CASES.update(limits=case_limits, synthetic=case_synthetic, scaling=case_scaling, converged_at_zero=case_converged_at_zero,
             replicated_576=case_replicated_576, prep_compare=case_prep_compare, errors=case_errors)


def main():
    name = sys.argv[1]
    try:
        CASES[name]()
        out = {name: "ok"}
    except Exception as e:   # noqa: BLE001
        traceback.print_exc()
        out = {name: f"{type(e).__name__}: {e}"[:600]}
    print(json.dumps(out))
    return 0 if out[name] == "ok" else 1


if __name__ == "__main__":
    sys.exit(main())
