"""b200pdlp_kkt_check_batch and b200pdlp_kkt_check_batch_device on the GPU: every member's b200pdlp_kkt_info must equal what
the host twin (b200pdlp_kkt_check_host, which tests/test_kkt_host.py pins against the reference's lpKktCheck) returns for it
alone, field for field and bit for bit (a NaN matches any NaN), and lie within test_gpu_kkt._same's tolerances of the single
device check.  The device variant must equal the host variant on the same data and leave its input tensors unchanged."""
import ctypes as C
import glob
import math
import os
import struct

import numpy as np
import pytest

from conftest import GOLDEN, term_to_model_status
from test_gpu_kkt import _same

pytestmark = pytest.mark.gpu

FILES = sorted(glob.glob(os.path.join(GOLDEN, "instances", "*.b2lp")))
VECTORS = ("col_value", "col_dual", "row_value", "row_dual")
COUNTERS = ("num_primal_infeasibilities", "num_dual_infeasibilities", "num_relative_primal_infeasibilities",
            "num_relative_dual_infeasibilities", "num_primal_residual_errors", "num_dual_residual_errors",
            "num_relative_primal_residual_errors", "num_relative_dual_residual_errors", "num_complementarity_violations")
ITER_LIMIT = 500


def assert_bits(got, want, what=""):
    assert set(got) == set(want), what
    for k, w in want.items():
        g = got[k]
        if isinstance(w, float):
            assert (math.isnan(g) and math.isnan(w)) or struct.pack("<d", g) == struct.pack("<d", w), (what, k, g, w)
        else:
            assert g == w, (what, k, g, w)


def check_batch(lps, sols, statuses, kkt_tolerance, single=False):
    """kkt_check_batch against the host twin (bits) and, with single=True, against the single device check (_same)"""
    from highs_b200 import engine
    got = engine.kkt_check_batch(lps, sols, kkt_tolerance=kkt_tolerance, model_status=statuses)
    assert len(got) == len(lps)
    for i, (lp, sol, st, g) in enumerate(zip(lps, sols, statuses, got)):
        assert_bits(g, engine.kkt_check(lp, sol, kkt_tolerance=kkt_tolerance, model_status=st, on_device=False), i)
        if single:
            _same(engine.kkt_check(lp, sol, kkt_tolerance=kkt_tolerance, model_status=st), g)
    return got


def _ordered(lp):
    from highs_b200 import engine
    f = engine.host_form(lp, 1)
    return max(f["n"], f["m"]) <= 4096


def _host(sol):
    return {k: sol[k] if isinstance(sol[k], np.ndarray) else sol[k].cpu().numpy() for k in VECTORS}


def _damaged(lp, sol, seed):
    """noise as in test_kkt_host.py: bound violations, wrong-sign duals, inconsistent activities"""
    rng = np.random.default_rng(seed)
    bad = {k: np.array(sol[k], dtype=np.float64) for k in VECTORS}
    bad["col_value"] += 1e-2 * rng.standard_normal(lp.num_col_)
    bad["row_dual"] += 1e-2 * rng.standard_normal(lp.num_row_)
    bad["col_dual"] += 1e-3 * rng.standard_normal(lp.num_col_)
    return bad


@pytest.fixture(scope="module")
def instance_members():
    """all 74 instance fixtures: the ordered ones solved by solve_batch, the two others by solve; then a damaged copy of each"""
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    lps = [read_b2lp(p) for p in FILES]
    assert len(lps) == 74
    ordered = [i for i, lp in enumerate(lps) if _ordered(lp)]
    tree = [i for i in range(len(lps)) if i not in ordered]
    assert len(ordered) == 72 and len(tree) == 2
    sols = [None] * len(lps)
    for i, r in zip(ordered, engine.solve_batch([lps[i] for i in ordered], iter_limit=ITER_LIMIT)):
        sols[i] = r
    for i in tree:
        sols[i] = engine.solve(lps[i], iter_limit=ITER_LIMIT)
    statuses = [term_to_model_status(r["term_code"], r["iters"], ITER_LIMIT) for r in sols]
    sols = [_host(r) for r in sols]
    bad = [_damaged(lp, s, i) for i, (lp, s) in enumerate(zip(lps, sols))]
    return lps + lps, sols + bad, statuses + [(7, 15, 9, 14)[i % 4] for i in range(len(lps))]


@pytest.mark.parametrize("kkt_tolerance", [0.0, 1e-4])
def test_instances_in_one_batch(engine_lib, instance_members, kkt_tolerance):
    lps, sols, statuses = instance_members
    got = check_batch(lps, sols, statuses, kkt_tolerance, single=True)
    for k in COUNTERS:   # the damaged copies reach every counter
        assert max(g[k] for g in got) > 0, k
    assert {g["model_status"] for g in got} >= {7, 15}


# ---- synthetic edge members
def _lp(n, m, cols, cost, cl, cu, rl, ru, sense=1, offset=0.0):
    """a HighsLp from per-column (rows, values) lists, stored as given"""
    from highs_b200.lp import HighsLp, HighsSparseMatrix
    start = np.cumsum([0] + [len(r) for r, _ in cols]).astype(np.int32)
    index = np.asarray([i for r, _ in cols for i in r], dtype=np.int32)
    value = np.asarray([v for _, vs in cols for v in vs], dtype=np.float64)
    lp = HighsLp(n, m, cost, cl, cu, rl, ru, HighsSparseMatrix(n, m, start, index, value))
    lp.sense_, lp.offset_ = sense, offset
    return lp


def _bounds(rng, k):
    """every kind of bound pair: free, fixed, lower only, upper only, boxed, infinite and 1e30 (finite) bounds"""
    kinds = rng.integers(0, 6, k)
    lo = rng.uniform(-5, 0, k)
    up = lo + rng.uniform(0, 5, k)
    lo = np.where(kinds == 0, -np.inf, lo)
    up = np.where((kinds == 0) | (kinds == 2), np.inf, up)
    up = np.where(kinds == 1, lo, up)
    lo = np.where(kinds == 3, -np.inf, lo)
    lo = np.where(kinds == 5, -1e30, lo)
    return lo, up


def _point(rng, lo, up):
    """values at a bound, inside, or violating it"""
    k = len(lo)
    v = rng.uniform(-6, 6, k)
    pick = rng.integers(0, 4, k)
    v = np.where((pick == 0) & np.isfinite(lo), lo, v)
    v = np.where((pick == 1) & np.isfinite(up), up, v)
    return v


def _member(rng, n, m, per_col, sense=1, offset=0.0, unsorted=False, long_col=0):
    cols = []
    for j in range(n):
        k = long_col if (j == 0 and long_col) else min(per_col, m)
        rows = sorted(rng.choice(m, size=k, replace=False).tolist()) if m and k else []
        if unsorted and len(rows) > 1:
            rows = rows[::-1] + [rows[0]]   # descending, with a repeated row
        cols.append((rows, rng.standard_normal(len(rows)).tolist()))
    cl, cu = _bounds(rng, n)
    rl, ru = _bounds(rng, m)
    lp = _lp(n, m, cols, rng.standard_normal(n), cl, cu, rl, ru, sense, offset)
    x = _point(rng, cl, cu)
    a = lp.a_matrix_.to_scipy() if n and m else None
    rv = (a @ x if a is not None else np.zeros(m)) + np.where(rng.random(m) < 0.3, 1e-3 * rng.standard_normal(m), 0.0)
    sol = dict(col_value=x, col_dual=np.where(rng.random(n) < 0.3, 0.0, rng.standard_normal(n)), row_value=rv,
               row_dual=np.where(rng.random(m) < 0.3, 0.0, rng.standard_normal(m)))
    return lp, sol


def edge_members(large=True):
    rng = np.random.default_rng(7)
    named = [("no_rows", _member(rng, 6, 0, 0)), ("no_cols", _member(rng, 0, 5, 0)), ("empty_matrix", _member(rng, 5, 4, 0)),
             ("unsorted_duplicates", _member(rng, 30, 20, 4, unsorted=True)), ("bound_kinds", _member(rng, 200, 150, 3)),
             ("long_column", _member(rng, 40, 6000, 2, long_col=5000)),
             ("maximise_offset", _member(rng, 50, 40, 3, sense=-1, offset=12.5))]
    lp, sol = _member(rng, 60, 50, 3)
    sol = {k: v.copy() for k, v in sol.items()}
    sol["col_value"][[1, 2, 3]] = [np.inf, -np.inf, np.nan]
    sol["col_dual"][[4, 5]] = [np.nan, np.inf]
    sol["row_value"][[0, 1]] = [np.nan, -np.inf]
    sol["row_dual"][[2, 3]] = [np.inf, np.nan]
    named.append(("inf_nan", (lp, sol)))
    if large:
        from highs_b200.lp import synthetic_lp
        big = synthetic_lp(100_000, 100_000, 10, seed=12345, dense_col_nnz=20_000)
        brng = np.random.default_rng(3)
        x = brng.uniform(0, 1, big.num_col_)
        named.insert(3, ("s2_size", (big, dict(col_value=x, col_dual=brng.standard_normal(big.num_col_) * 1e-3,
                                                 row_value=big.a_matrix_.to_scipy() @ x,
                                                 row_dual=brng.standard_normal(big.num_row_) * 1e-3))))
    return named


@pytest.mark.parametrize("kkt_tolerance", [0.0, 1e-4])
def test_edge_members_in_one_batch(engine_lib, kkt_tolerance):
    named = edge_members()
    lps = [lp for _, (lp, _) in named]
    sols = [s for _, (_, s) in named]
    statuses = [(7, 15, 9, 14)[i % 4] for i in range(len(named))]
    check_batch(lps, sols, statuses, kkt_tolerance)


# ---- the device-pointer variant
def _to_device(sol):
    import torch
    return {k: torch.as_tensor(np.ascontiguousarray(sol[k], dtype=np.float64)).cuda() for k in VECTORS}


def _snapshot(dicts):
    return [{k: v.cpu().numpy().tobytes() for k, v in d.items() if hasattr(v, "is_cuda")} for d in dicts]


def _device_equals_host(lps, dlps, dsols, statuses, kkt_tolerance):
    from highs_b200 import engine
    snap = _snapshot(dlps) + _snapshot(dsols)
    got = engine.kkt_check_batch_device(dlps, dsols, kkt_tolerance=kkt_tolerance, model_status=statuses)
    want = check_batch(lps, [_host(s) for s in dsols], statuses, kkt_tolerance)
    for i, (g, w) in enumerate(zip(got, want)):
        assert_bits(g, w, i)
    assert _snapshot(dlps) + _snapshot(dsols) == snap
    return got


@pytest.mark.parametrize("solver", ["pdlp", "hipdlp"])
def test_device_variant_on_batch_device_results(engine_lib, solver):
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    lps = [lp for lp in (read_b2lp(p) for p in FILES) if _ordered(lp)]
    if solver == "hipdlp":
        lps = [lp for lp in lps if max(engine.host_form_hipdlp(lp)["n"], engine.host_form_hipdlp(lp)["m"]) <= 4096]
    dlps = [engine.lp_to_device(lp, 0) for lp in lps]
    solve = engine.solve_batch_device if solver == "pdlp" else engine.solve_hipdlp_batch_device
    res = solve(dlps, iter_limit=ITER_LIMIT)
    statuses = [term_to_model_status(r["term_code"], r["iters"], ITER_LIMIT) for r in res]
    for tol in (0.0, 1e-4):
        _device_equals_host(lps, dlps, res, statuses, tol)


def test_device_variant_on_edge_members(engine_lib):
    from highs_b200 import engine
    named = edge_members(large=False)
    lps = [lp for _, (lp, _) in named]
    dlps = [engine.lp_to_device(lp, 0) for lp in lps]
    dsols = [_to_device(s) for _, (_, s) in named]
    _device_equals_host(lps, dlps, dsols, [7, 15, 9, 14, 7, 15, 9, 14][:len(lps)], 1e-4)


def _device_call(dlps, csols):
    """b200pdlp_kkt_check_batch_device on ctypes solutions; returns (rc, message, inout untouched)"""
    from highs_b200 import engine
    L = engine.lib()
    count = len(dlps)
    clps = (engine.CLp * count)(*[engine.make_clp_device(d) for d in dlps])
    infos = (engine.CKktInfo * count)()
    C.memset(infos, 0x5A, C.sizeof(infos))
    before = bytes(infos)
    fn = L.b200pdlp_kkt_check_batch_device
    fn.argtypes = [C.c_int32, C.POINTER(engine.CLp), C.POINTER(engine.CSolution), C.POINTER(engine.CKktTolerances), C.c_int32,
                   C.POINTER(engine.CKktInfo)]
    rc = fn(count, clps, csols, C.byref(engine._kkt_tolerances(0.0)), 0, infos)
    return rc, L.b200pdlp_last_error().decode(), bytes(infos) == before


def _csols(dsols):
    import torch
    from highs_b200 import engine
    return (engine.CSolution * len(dsols))(*[engine.CSolution(*(engine._dev_ptr(s[k], torch.float64, engine._dp, k)
                                                                for k in VECTORS)) for s in dsols])


def test_device_variant_errors(engine_lib):
    import torch
    from highs_b200 import engine
    rng = np.random.default_rng(11)
    pairs = [_member(rng, 30, 20, 3) for _ in range(6)]
    lps = [lp for lp, _ in pairs]
    dlps = [engine.lp_to_device(lp, 0) for lp in lps]
    dsols = [_to_device(s) for _, s in pairs]
    rc, msg, untouched = _device_call(dlps, _csols(dsols))
    assert rc == 0, msg
    # a host array in member 3's row_dual
    csols = _csols(dsols)
    host_rd = np.ascontiguousarray(pairs[3][1]["row_dual"])
    csols[3].row_dual = engine._p(host_rd, engine._dp)
    rc, msg, untouched = _device_call(dlps, csols)
    assert rc == -1 and "member 3: row_dual is not device memory" in msg and untouched, msg
    # a decreasing a_start in member 2 and an a_index out of range in member 5: member 2 is named
    bad = [dict(d) for d in dlps]
    st = bad[2]["a_start"].clone()
    st[4], st[5] = st[5].item(), st[4].item() - 1
    bad[2]["a_start"] = st
    ix = bad[5]["a_index"].clone()
    ix[0] = lps[5].num_row_
    bad[5]["a_index"] = ix
    torch.cuda.synchronize()
    rc, msg, untouched = _device_call(bad, _csols(dsols))
    assert rc == -1 and "member 2: " in msg and "non-decreasing" in msg and untouched, msg
    bad[2] = dlps[2]
    rc, msg, untouched = _device_call(bad, _csols(dsols))
    assert rc == -1 and "member 5: " in msg and "a_index entry outside" in msg and untouched, msg


def test_device_variant_rejects_another_devices_pointer(engine_lib):
    import torch
    from highs_b200 import engine
    if engine.device_count() < 2:
        pytest.skip("needs two GPUs")
    rng = np.random.default_rng(12)
    pairs = [_member(rng, 30, 20, 3) for _ in range(2)]
    dlps = [engine.lp_to_device(lp, 0) for lp, _ in pairs]
    dsols = [_to_device(s) for _, s in pairs]
    dsols[1]["col_dual"] = dsols[1]["col_dual"].to("cuda:1")
    torch.cuda.synchronize()
    rc, msg, untouched = _device_call(dlps, _csols(dsols))
    assert rc == -1 and "member 1: col_dual is not device memory of device 0" in msg and untouched, msg


def test_bench_workload(engine_lib):
    """the 576 members of tools/kkt_batch_bench.py: every member equal to the host twin, on host and on device data"""
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    base = [lp for lp in (read_b2lp(p) for p in FILES) if _ordered(lp)]
    work = base * 8
    dlps = [engine.lp_to_device(lp, 0) for lp in work]
    res = engine.solve_batch_device(dlps, iter_limit=ITER_LIMIT)
    statuses = [term_to_model_status(r["term_code"], r["iters"], ITER_LIMIT) for r in res]
    sols = [_host(r) for r in res]
    got_host = engine.kkt_check_batch(work, sols, model_status=statuses)
    got_dev = engine.kkt_check_batch_device(dlps, res, model_status=statuses)
    twins = [engine.kkt_check(lp, s, model_status=st, on_device=False) for lp, s, st in zip(base, sols, statuses)]
    for i, (gh, gd) in enumerate(zip(got_host, got_dev)):
        assert_bits(gh, twins[i % len(base)], i)
        assert_bits(gd, twins[i % len(base)], i)
