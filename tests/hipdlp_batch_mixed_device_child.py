"""Child process of tests/test_gpu_hipdlp_batch_mixed_device.py (own process: a faulting kernel must not poison the CUDA
context of the test session).  Runs one named case of b200pdlp_solve_hipdlp_batch_mixed_device against
b200pdlp_solve_hipdlp_batch_mixed on host copies of the same LPs and against b200pdlp_solve_hipdlp on each tree member alone.
"Identical" = byte equality as in tests/hipdlp_batch_mixed_child.py: the ints, the six residual scalars, the four
HighsSolution vectors and the trace rows; no input tensor may change.
usage: python tests/hipdlp_batch_mixed_device_child.py CASE   -> one JSON line {CASE: "ok" | error text}"""
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
from hipdlp_batch_child import (VARIANTS, _bits, assert_same, golden, instances, mixed_lp, no_rows_lp, small_set,  # noqa: E402
                                zero_optimal_lp)
from hipdlp_batch_mixed_child import TRACE, midsize_lp, midsize_set  # noqa: E402


def _host(d):
    """a result of the device call with its tensors copied to the host"""
    return {k: (v.cpu().numpy() if hasattr(v, "is_cuda") else v) for k, v in d.items()}


def assert_same_trace(a, b, what):
    assert_same(a, b, what)
    assert a["trace"].shape == b["trace"].shape, (what, "trace rows", a["trace"].shape, b["trace"].shape)
    assert np.array_equal(_bits(a["trace"]), _bits(b["trace"])), (what, "trace")


def _snapshot(dlps):
    return [{k: v.cpu().numpy().tobytes() for k, v in d.items() if hasattr(v, "is_cuda")} for d in dlps]


def _assert_unchanged(dlps, snap):
    for i, (d, s) in enumerate(zip(dlps, snap)):
        for k, b in s.items():
            assert d[k].cpu().numpy().tobytes() == b, (i, k)


def device_vs_host(named, single=True, **kw):
    """solve_hipdlp_batch_mixed_device on device copies of the LPs of `named` against solve_hipdlp_batch_mixed on the host
    arrays and (single) against solve_hipdlp on each member alone; returns the device results (host copies)"""
    lps = [lp for _, lp in named]
    dlps = [engine.lp_to_device(lp, 0) for lp in lps]
    snap = _snapshot(dlps)
    got = [_host(g) for g in engine.solve_hipdlp_batch_mixed_device(dlps, trace_cap=TRACE, **kw)]
    _assert_unchanged(dlps, snap)
    want = engine.solve_hipdlp_batch_mixed(lps, trace_cap=TRACE, **kw)
    assert len(got) == len(named)
    for (nm, lp), g, w in zip(named, got, want):
        assert_same_trace(g, w, nm)
        assert g["kernel_launches"] == got[0]["kernel_launches"] and g["solve_seconds"] == got[0]["solve_seconds"], nm
    if single:
        for (nm, lp), g in zip(named, got):
            assert_same_trace(g, engine.solve_hipdlp(lp, trace_cap=TRACE, **kw), nm)
    return got


# ---- synthetic members for the prologue comparison
def _csc_lp(n, m, cols, rl, ru, seed=0):
    """an LP from columns given as (rows, values) lists, stored in the given order"""
    rng = np.random.default_rng(seed)
    start, idx, val = [0], [], []
    for r, v in cols:
        idx += list(r); val += list(v); start.append(len(idx))
    return HighsLp(n, m, rng.standard_normal(n), np.zeros(n), np.full(n, 4.0), np.asarray(rl, dtype=float),
                   np.asarray(ru, dtype=float),
                   HighsSparseMatrix(n, m, np.asarray(start, dtype=np.int32), np.asarray(idx, dtype=np.int32),
                                     np.asarray(val, dtype=np.float64)))


def edge_tree_lps():
    rng = np.random.default_rng(11)
    named = []
    # equality rows of exactly 512, 513, 2048 and 2049 entries (the long-row threshold and the segment size), in rows and
    # (through the transpose) in columns
    import scipy.sparse as sp
    m, n = 3000, 2600
    r, c = [rng.integers(4, m, size=2 * n)], [np.repeat(np.arange(n), 2)]
    for k, ln in enumerate((512, 513, 2048, 2049)):
        r.append(np.full(ln, k)); c.append(rng.choice(n, size=ln, replace=False))
    r, c = np.concatenate(r), np.concatenate(c)
    A = sp.csc_matrix((rng.standard_normal(r.size), (r, c)), shape=(m, n))
    A.sum_duplicates(); A.sort_indices()
    named.append(("row_lengths", _csc_lp(n, m, [(A.indices[A.indptr[j]:A.indptr[j + 1]], A.data[A.indptr[j]:A.indptr[j + 1]])
                                                for j in range(n)], np.zeros(m), np.zeros(m), 3)))
    named.append(("col_lengths", _csc_lp(m, n, [(A.T.tocsc().indices[s0:s1], A.T.tocsc().data[s0:s1])
                                                for s0, s1 in zip(A.T.tocsc().indptr[:-1], A.T.tocsc().indptr[1:])],
                                         np.full(n, -1.0), np.full(n, np.inf), 4)))
    # more than one sort window on both sides of neq: 20000 rows, half equalities, many rows of equal length
    m, n = 20000, 18000
    cols = []
    for j in range(n):
        r = np.sort(rng.choice(m, size=2, replace=False))
        cols.append((r, rng.standard_normal(2)))
    rl = np.where(np.arange(m) % 2 == 0, 1.0, -np.inf)
    ru = np.where(np.arange(m) % 2 == 0, 1.0, 2.0)
    named.append(("windows_equal_lengths", _csc_lp(n, m, cols, rl, ru, 1)))
    # a 20000-entry column stored in descending order, and a column holding +0.0 and -0.0 in one row (-0.0 stored first)
    m, n = 24000, 300
    cols = [(np.arange(m - 1, m - 20001, -1), rng.standard_normal(20000)),
            (np.array([5, 7, 7, 3]), np.array([1.0, -0.0, 0.0, 2.0]))]
    for j in range(2, n):
        cols.append((np.sort(rng.choice(m, size=3, replace=False)), rng.standard_normal(3)))
    named.append(("long_descending_signed_zero", _csc_lp(n, m, cols, np.full(m, -1.0), np.full(m, 1.0), 2)))
    # no rows; empty rows and columns
    named.append(("no_rows", no_rows_lp()))
    named.append(("empty_rows_cols", midsize_lp(22, 700, 900, per_col=2, empty=True)))
    return named


# ---- cases
def case_prep_compare():
    named = instances(ordered_max=262144) + midsize_set() + edge_tree_lps()
    for mode in (0, 1, 2, 4, 5, 7):
        for ruiz in (0, 3):
            reps = engine.hipdlp_tree_prep_compare([lp for _, lp in named], scaling_mode=mode, ruiz_iterations=ruiz)
            bad = {nm: {k: v for k, v in r.items() if v != 0} for (nm, _), r in zip(named, reps) if any(v != 0 for v in r.values())}
            assert not bad, (mode, ruiz, bad)


def case_instances_tree(vi):
    def run():
        inst = instances()
        assert len(inst) > 40, len(inst)
        device_vs_host(inst, ordered_max=-1, **VARIANTS[vi])
    return run


def case_midsize():
    named = midsize_set() + [("near_cap", midsize_lp(8, 250000, 100000, per_col=2, long_rows=(3000,)))]
    f = engine.host_form_hipdlp(named[-1][1])
    assert 240000 <= max(f["n"], f["m"]) <= 262144, (f["n"], f["m"])
    got = device_vs_host(named, iter_limit=3000, tolerance=1e-4)
    assert any(g["restarts"] > 0 for g in got), [g["restarts"] for g in got]
    assert any(g["term_name"] == "OPTIMAL" for g in got), [g["term_name"] for g in got]


def case_mixed():
    """ordered and tree members interleaved: the ordered members equal solve_hipdlp_batch_device, the tree members solve_hipdlp"""
    small = small_set() + [("mixed1", mixed_lp(1)), ("no_rows", no_rows_lp())]
    mid = midsize_set()[:3]
    named = [small[0], mid[0], small[1], small[2], mid[1], small[3], mid[2], small[4], small[5], small[6]]
    kw = dict(iter_limit=2000, tolerance=1e-5)
    got = device_vs_host(named, single=False, **kw)
    ordered = [i for i, (nm, _) in enumerate(named) if nm not in dict(mid)]
    plain = engine.solve_hipdlp_batch_device([engine.lp_to_device(named[i][1], 0) for i in ordered], **kw)
    for i, p in zip(ordered, plain):
        assert_same(got[i], _host(p), named[i][0])
    for i, (nm, lp) in enumerate(named):
        if i not in ordered:
            assert_same_trace(got[i], engine.solve_hipdlp(lp, trace_cap=TRACE, **kw), nm)


def case_clusters():
    named = midsize_set()[:3] + [("mixed2", mixed_lp(2))]
    kw = dict(iter_limit=1200, tolerance=1e-6, ordered_max=-1)
    dlps = [engine.lp_to_device(lp, 0) for _, lp in named]
    runs = {}
    for c in ("1", "8"):
        os.environ["B200PDLP_BATCH_CLUSTER"] = c
        try:
            runs[c] = [_host(g) for g in engine.solve_hipdlp_batch_mixed_device(dlps, trace_cap=TRACE, **kw)]
        finally:
            del os.environ["B200PDLP_BATCH_CLUSTER"]
    for (nm, lp), a, b in zip(named, runs["1"], runs["8"]):
        assert_same_trace(a, b, f"{nm} C=1 vs C=8")
        assert_same_trace(a, engine.solve_hipdlp(lp, trace_cap=TRACE, **kw), nm)


def case_limits():
    named = small_set() + [("mixed3", mixed_lp(3)), ("no_rows", no_rows_lp()), ("zero_optimal", zero_optimal_lp())]
    for lim in (0, 1, 40, 41):
        got = device_vs_host(named, iter_limit=lim, tolerance=1e-9, ordered_max=-1)
        assert got[0]["kernel_launches"] == 1 + (-(-lim // 40) if lim > 0 else 0), (lim, got[0]["kernel_launches"])
    got = device_vs_host(named, single=False, time_limit=0.0, ordered_max=-1)
    assert all(g["term_iterate"] == 2 or g["term_name"] == "OPTIMAL" for g in got)
    got = device_vs_host(named, iter_limit=2000, ordered_max=-1)
    assert got[-1]["iters"] == 0 and got[-1]["term_name"] == "OPTIMAL", (got[-1]["iters"], got[-1]["term_name"])
    assert got[-2]["form_rows"] == 0
    device_vs_host(named + midsize_set()[:1], iter_limit=1000, tolerance=1e-5, ordered_max=-1, step_size_strategy=0)


# ---- errors: ERR_ARG naming the member, nothing written
def _raw_call(dlps, **params):
    """b200pdlp_solve_hipdlp_batch_mixed_device through the C ABI with NaN-filled device outputs and sentinel result fields"""
    import torch
    L = engine.lib()
    L.b200pdlp_solve_hipdlp_batch_mixed_device.argtypes = [C.c_int32, C.POINTER(engine.CLp), C.POINTER(engine.CHipdlpParams),
                                                           C.POINTER(engine.CResult)]
    count = len(dlps)
    clps, cres, outs = (engine.CLp * count)(), (engine.CResult * count)(), []
    for i, d in enumerate(dlps):
        clps[i] = d if isinstance(d, engine.CLp) else engine.make_clp_device(d)
        n, m = clps[i].num_col, clps[i].num_row
        v = [torch.full((max(k, 1),), float("nan"), dtype=torch.float64, device="cuda") for k in (n, n, m, m)]
        cres[i].col_value, cres[i].col_dual, cres[i].row_value, cres[i].row_dual = (C.cast(C.c_void_p(t.data_ptr()), engine._dp) for t in v)
        cres[i].term_code, cres[i].iters, cres[i].setup_seconds, cres[i].trace_len = -7, -7, -7.0, -7
        outs.append(v)
    prm = engine._hipdlp_params(params)
    rc = L.b200pdlp_solve_hipdlp_batch_mixed_device(count, clps, C.byref(prm), cres)
    for i in range(count):
        assert (cres[i].term_code, cres[i].iters, cres[i].setup_seconds, cres[i].trace_len) == (-7, -7, -7.0, -7), i
        assert all(bool(t.isnan().all()) for t in outs[i]), i
    return rc, L.b200pdlp_last_error().decode()


def case_errors():
    lps = [golden(nm) for nm in ("afiro", "avgas", "adlittle", "blending")]
    dlps = [engine.lp_to_device(lp, 0) for lp in lps]
    snap = _snapshot(dlps)
    clp2 = engine.make_clp_device(dlps[2])
    clp2.col_cost = engine._p(lps[2].col_cost_, engine._dp)
    rc, msg = _raw_call(dlps[:2] + [clp2] + dlps[3:], ordered_max=-1)
    assert rc == -1 and "b200pdlp_solve_hipdlp_batch_mixed_device: member 2: col_cost is not device memory" in msg, msg
    bad_index = dict(dlps[1])
    bad_index["a_index"] = bad_index["a_index"].clone()
    bad_index["a_index"][5] = lps[1].num_row_
    decreasing = dict(dlps[3])
    decreasing["a_start"] = decreasing["a_start"].clone()
    decreasing["a_start"][1] = decreasing["a_start"][2] + 1
    rc, msg = _raw_call([dlps[0], bad_index, dlps[2], decreasing], ordered_max=-1)
    assert rc == -1 and "member 1: " in msg and "a_index entry outside" in msg, msg
    rc, msg = _raw_call([dlps[0], dlps[1], dlps[2], decreasing])
    assert rc == -1 and "member 3: " in msg and "non-decreasing" in msg, msg
    # an over-cap member (member 1) before a malformed one (member 2): the lower one is named
    big = synthetic_lp(262145, 10, 1, 1)
    dbig = engine.lp_to_device(big, 0)
    rc, msg = _raw_call([dlps[0], dbig, decreasing])
    assert rc == -1 and "member 1: standard form 262145 x" in msg and "exceeds max(n, m) = 262144 of a tree member" in msg, msg
    rc, msg = _raw_call([dlps[0], decreasing, dbig])
    assert rc == -1 and "member 1: " in msg and "non-decreasing" in msg, msg
    _assert_unchanged(dlps, snap)


def case_inputs_untouched():
    named = midsize_set()[:2] + [("mixed1", mixed_lp(1)), ("afiro", golden("afiro"))]
    dlps = [engine.lp_to_device(lp, 0) for _, lp in named]
    snap = _snapshot(dlps)
    engine.solve_hipdlp_batch_mixed_device(dlps, iter_limit=400)
    engine.solve_hipdlp_batch_mixed_device(dlps, iter_limit=400, ordered_max=-1)
    _assert_unchanged(dlps, snap)


def case_kkt():
    named = midsize_set()[:2] + [("mixed1", mixed_lp(1)), ("afiro", golden("afiro")), ("adlittle", golden("adlittle"))]
    dlps = [engine.lp_to_device(lp, 0) for _, lp in named]
    got = engine.solve_hipdlp_batch_mixed_device(dlps, iter_limit=2000, tolerance=1e-6)
    dev = engine.kkt_check_batch_device(dlps, got)
    host = engine.kkt_check_batch([lp for _, lp in named], [_host(g) for g in got])
    for (nm, _), a, b in zip(named, dev, host):
        assert a.keys() == b.keys(), nm
        for k in a:   # floats bit for bit, everything else by value
            same = (np.float64(a[k]).tobytes() == np.float64(b[k]).tobytes()) if isinstance(a[k], float) else a[k] == b[k]
            assert same, (nm, k, a[k], b[k])


def case_twice():
    named = midsize_set()[:2] + [("afiro", golden("afiro"))]
    kw = dict(iter_limit=800, ordered_max=-1)
    dlps = [engine.lp_to_device(lp, 0) for _, lp in named]
    a = [_host(g) for g in engine.solve_hipdlp_batch_mixed_device(dlps, trace_cap=TRACE, **kw)]
    b = [_host(g) for g in engine.solve_hipdlp_batch_mixed_device(dlps, trace_cap=TRACE, **kw)]
    for (nm, lp), x, y in zip(named, a, b):
        assert_same_trace(x, y, nm)
        assert_same_trace(x, engine.solve_hipdlp(lp, trace_cap=TRACE, **kw), nm)


CASES = {"prep_compare": case_prep_compare}
CASES.update({f"instances_tree{v}": case_instances_tree(v) for v in range(len(VARIANTS))})
CASES.update(midsize=case_midsize, mixed=case_mixed, clusters=case_clusters, limits=case_limits, errors=case_errors,
             inputs_untouched=case_inputs_untouched, kkt=case_kkt, twice=case_twice)


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
