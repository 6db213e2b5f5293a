"""Child process of tests/test_gpu_solve_device.py (own process: a faulting kernel must not poison the CUDA context of the test
session).  Runs one named case of b200pdlp_solve_device / b200pdlp_solve_hipdlp_device against b200pdlp_solve /
b200pdlp_solve_hipdlp on host copies of the same arrays.  "Identical" = byte equality of the ints (status, iterate,
iterations, passes, restarts, form dimensions), the six residual scalars, the four vectors and the trace rows; no input
tensor may change.
usage: python tests/solve_device_child.py CASE   -> one JSON line {CASE: "ok" | error text}"""
import ctypes as C
import json
import os
import sys
import tempfile
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

from conftest import GOLDEN, golden_lp, load_golden, options_to_params  # noqa: E402
from highs_b200 import engine  # noqa: E402
from highs_b200.lp import HighsLp, HighsSparseMatrix  # noqa: E402
from hipdlp_batch_child import INTS, SCALARS, VARIANTS, VECTORS, _bits, golden, instances, mixed_lp, no_rows_lp  # noqa: E402
from hipdlp_batch_mixed_child import midsize_lp, midsize_set  # noqa: E402

TRACE = 256
# PDLP option sets: the goldens' tags, scaling off, a fixed step, restarts off, and the limits; each bounded at 400 iterations
PDLP_SETS = [options_to_params(next(c for c in load_golden() if c["tag"] == t)["options"]) for t in ("default", "kkt1e-4")] + \
            [dict(scaling=0), dict(adaptive_step=0), dict(restart=0), dict(iter_limit=80), dict(time_limit=0.0)]
for _s in PDLP_SETS:
    _s["iter_limit"] = min(_s.get("iter_limit", 400), 400)


def _host(d):
    return {k: (v.cpu().numpy() if hasattr(v, "is_cuda") else v) for k, v in d.items()}


def assert_same(a, b, what):
    for k in INTS:
        assert a[k] == b[k], (what, k, a[k], b[k])
    for k in SCALARS:
        assert _bits(a[k]) == _bits(b[k]), (what, k, a[k], b[k])
    for k in VECTORS:
        assert np.array_equal(_bits(a[k]), _bits(b[k])), (what, k)
    if "trace" in a or "trace" in b:
        assert a["trace"].shape == b["trace"].shape, (what, "trace rows", a["trace"].shape, b["trace"].shape)
        assert np.array_equal(_bits(a["trace"]), _bits(b["trace"])), (what, "trace")


def _snapshot(tensors):
    return [t.cpu().numpy().tobytes() for t in tensors]


def _tensors(dlp, warm=None):
    return [v for v in dlp.values() if hasattr(v, "is_cuda")] + list(warm or ())


def _dev_warm(warm):
    import torch
    return None if warm is None else tuple(torch.as_tensor(np.asarray(v, dtype=np.float64)).cuda() for v in warm)


def _rc(e):
    return str(e).split("failed (")[1].split(")")[0]


def _vs_host(nm, dev_solve, host_solve, tensors):
    """dev_solve() against host_solve(): the same bits, or the same return code when the host-array solve fails too;
    the input tensors untouched"""
    snap = _snapshot(tensors)
    print(f"[{nm}]", flush=True)
    try:
        want = host_solve()
    except engine.EngineError as e:
        try:
            dev_solve()
        except engine.EngineError as d:
            assert _rc(d) == _rc(e), (nm, str(d), str(e))
        else:
            raise AssertionError((nm, "the host-array solve failed, the device-array solve did not", str(e)))
        return None
    got = _host(dev_solve())
    assert _snapshot(tensors) == snap, (nm, "an input changed")
    assert_same(got, want, nm)
    return got


def pdlp_vs_host(nm, lp, warm=None, trace_cap=TRACE, **kw):
    """solve_device on device copies of lp (and warm) against solve on the host arrays"""
    dlp, dwarm = engine.lp_to_device(lp, 0), _dev_warm(warm)
    return _vs_host(nm, lambda: engine.solve_device(dlp, warm=dwarm, trace_cap=trace_cap, **kw),
                    lambda: engine.solve(lp, warm=warm, trace_cap=trace_cap, **kw), _tensors(dlp, dwarm))


def hip_vs_host(nm, lp, trace_cap=TRACE, **kw):
    dlp = engine.lp_to_device(lp, 0)
    return _vs_host(nm, lambda: engine.solve_hipdlp_device(dlp, trace_cap=trace_cap, **kw),
                    lambda: engine.solve_hipdlp(lp, trace_cap=trace_cap, **kw), _tensors(dlp))


def rows_long():
    return midsize_lp(1, 6000, 5000, long_rows=(700, 1500, 2048, 2049, 4900))


def _csc(n, m, start, index, value, cost, cl, cu, rl, ru):
    return HighsLp(n, m, np.asarray(cost, float), np.asarray(cl, float), np.asarray(cu, float), np.asarray(rl, float),
                   np.asarray(ru, float), HighsSparseMatrix(n, m, np.asarray(start, np.int32), np.asarray(index, np.int32),
                                                            np.asarray(value, float)))


def degenerate_lps():
    """past ordered_max = 4096: no columns, and rows and columns without a nonzero"""
    rng = np.random.default_rng(3)
    n, m = 5000, 4500
    no_cols = _csc(0, m, [0], [], [], [], [], [], -rng.random(m), rng.random(m))
    empty = _csc(n, m, np.zeros(n + 1), [], [], rng.standard_normal(n), -np.ones(n), np.ones(n), -rng.random(m), rng.random(m))
    return [("no_cols_big", no_cols), ("empty_matrix_big", empty)]


def big_lp():
    """about 400k x 400k, past every batch cap (ordered_max and a tree member's 262144) in both modes"""
    return midsize_lp(7, 400000, 400000, per_col=3, long_rows=(5000,), long_cols=(3000,))


def classes_differ_lp():
    """FREE and ranged rows and 1e25 bounds at tree size: the two modes give different standard forms"""
    lp = midsize_lp(8, 12000, 10000, per_col=3, long_rows=(2100,))
    assert engine.host_form(lp, 1)["n"] != engine.host_form_hipdlp(lp)["n"]
    return lp


# ---- cases
def case_pdlp_instances(k):
    def run():
        inst = instances()
        assert len(inst) > 40, len(inst)
        for ordered_max in (0, -1):
            for nm, lp in inst:
                pdlp_vs_host(f"{nm} ordered_max={ordered_max}", lp, ordered_max=ordered_max, **PDLP_SETS[k])
    return run


def case_hip_instances(v):
    def run():
        for ordered_max in (0, -1):
            for nm, lp in instances():
                hip_vs_host(f"{nm} ordered_max={ordered_max}", lp, ordered_max=ordered_max, **VARIANTS[v])
    return run


def case_hot_starts():
    case = next(c for c in load_golden() if c["warm_from"])
    rlp = golden_lp(case)
    first = dict(np.load(os.path.join(GOLDEN, case["warm_from"])))
    kw = options_to_params(case["options"])
    for ordered_max in (0, -1):
        got = pdlp_vs_host("restart_lp hot", rlp, warm=(first["col_value"], first["row_value"], first["row_dual"]),
                           ordered_max=ordered_max, **kw)
        assert got["term_name"] == "OPTIMAL" and (ordered_max == -1 or got["iters"] == case["pdlp_iteration_count"]), got["iters"]
        for nm in ("afiro", "avgas", "adlittle", "blending", "e226", "boxed_row", "distillation"):
            lp = golden(nm)
            own = engine.solve(lp, iter_limit=20000, ordered_max=ordered_max)
            pdlp_vs_host(f"{nm} own solution", lp, warm=(own["col_value"], own["row_value"], own["row_dual"]),
                         ordered_max=ordered_max, iter_limit=2000)
    lp = rows_long()
    own = engine.solve(lp, iter_limit=600)
    pdlp_vs_host("rows_long own iterate", lp, warm=(own["col_value"], own["row_value"], own["row_dual"]), iter_limit=400)


def case_synthetic():
    named = midsize_set() + [("mixed1", mixed_lp(1)), ("classes_differ", classes_differ_lp())]
    for nm, lp in named:
        for ordered_max in (0, -1):
            pdlp_vs_host(nm, lp, ordered_max=ordered_max, iter_limit=1000, tol_primal=1e-5, tol_dual=1e-5)
            hip_vs_host(nm, lp, ordered_max=ordered_max, iter_limit=1000, tolerance=1e-5)


def case_big():
    lp = big_lp()
    assert engine.host_form(lp, 1)["n"] > 262144 and engine.host_form_hipdlp(lp)["n"] > 262144
    pdlp_vs_host("big", lp, iter_limit=300)
    hip_vs_host("big", lp, iter_limit=300)


def case_degenerate():
    # (PDLP mode leaves LPs without rows out: b200pdlp_solve itself did not return on one within 200 s on an H100)
    for ordered_max in (0, -1):
        hip_vs_host("no_rows", no_rows_lp(), ordered_max=ordered_max, iter_limit=2000)
    for nm, lp in degenerate_lps():
        for ordered_max in (0, -1):
            pdlp_vs_host(nm, lp, ordered_max=ordered_max, iter_limit=2000)
            hip_vs_host(nm, lp, ordered_max=ordered_max, iter_limit=2000)
        n, m = lp.num_col_, lp.num_row_
        rng = np.random.default_rng(1)
        pdlp_vs_host(f"{nm} warm", lp, warm=(rng.random(n), rng.random(m), rng.standard_normal(m)), iter_limit=2000)


def case_device_prep_off():
    """B200PDLP_DEVICE_PREP=0 and device_scaling / device_prep = -1 select the host prologue of the host-array solves; the
    device-array solves ignore them and return the bits they return without them"""
    named = [("rows_long", rows_long()), ("classes_differ", classes_differ_lp()), ("afiro", golden("afiro"))]
    for nm, lp in named:
        dlp = engine.lp_to_device(lp, 0)
        for solve, extra in ((engine.solve_device, dict(device_scaling=-1)), (engine.solve_hipdlp_device, dict(device_prep=-1))):
            want = _host(solve(dlp, trace_cap=TRACE, iter_limit=400, ordered_max=-1))
            assert_same(_host(solve(dlp, trace_cap=TRACE, iter_limit=400, ordered_max=-1, **extra)), want, nm)
            os.environ["B200PDLP_DEVICE_PREP"] = "0"
            try:
                assert_same(_host(solve(dlp, trace_cap=TRACE, iter_limit=400, ordered_max=-1)), want, nm)
            finally:
                del os.environ["B200PDLP_DEVICE_PREP"]


def _stderr_of(fn):
    """what the library prints to stderr (file descriptor 2) while fn() runs"""
    sys.stderr.flush()
    with tempfile.TemporaryFile(mode="w+") as f:
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return f.read()


def case_no_upload():
    """the tree route copies none of the LP to the device (B200PDLP_TIMING=1: 0 bytes), the host-array solve all of it"""
    lp = rows_long()
    dlp = engine.lp_to_device(lp, 0)
    os.environ["B200PDLP_TIMING"] = "1"
    try:
        for solve_dev, solve_host in ((engine.solve_device, engine.solve), (engine.solve_hipdlp_device, engine.solve_hipdlp)):
            dev = _stderr_of(lambda: solve_dev(dlp, iter_limit=40))
            host = _stderr_of(lambda: solve_host(lp, iter_limit=40))
            assert "LP arrays copied to the device: 0 bytes" in dev, dev[-2000:]
            n, m, nnz = lp.num_col_, lp.num_row_, int(lp.a_matrix_.start_[-1])
            assert f"LP arrays copied to the device: {4 * (n + 1) + 12 * nnz + 24 * n + 16 * m} bytes" in host, host[-2000:]
    finally:
        del os.environ["B200PDLP_TIMING"]


# ---- errors: ERR_ARG naming the field, nothing written
def _raw(dlp, hip, **params):
    """one call through the C ABI with NaN-filled device outputs and sentinel result fields, which must stay as they are"""
    import torch
    L = engine.lib()
    clp = dlp if isinstance(dlp, engine.CLp) else engine.make_clp_device(dlp)
    n, m = clp.num_col, clp.num_row
    v = [torch.full((max(k, 1),), float("nan"), dtype=torch.float64, device="cuda") for k in (n, n, m, m)]
    res = engine.CResult()
    res.col_value, res.col_dual, res.row_value, res.row_dual = (C.cast(C.c_void_p(t.data_ptr()), engine._dp) for t in v)
    res.term_code, res.iters, res.setup_seconds, res.trace_len = -7, -7, -7.0, -7
    if hip:
        L.b200pdlp_solve_hipdlp_device.argtypes = [C.POINTER(engine.CLp), C.POINTER(engine.CHipdlpParams), C.POINTER(engine.CResult)]
        rc = L.b200pdlp_solve_hipdlp_device(C.byref(clp), C.byref(engine._hipdlp_params(params)), C.byref(res))
    else:
        L.b200pdlp_solve_device.argtypes = [C.POINTER(engine.CLp), C.POINTER(engine.CParams), C.POINTER(engine.CWarm),
                                            C.POINTER(engine.CResult)]
        rc = L.b200pdlp_solve_device(C.byref(clp), C.byref(engine.make_params(**params)), None, C.byref(res))
    assert (res.term_code, res.iters, res.setup_seconds, res.trace_len) == (-7, -7, -7.0, -7)
    assert all(bool(t.isnan().all()) for t in v)
    return rc, L.b200pdlp_last_error().decode()


def case_errors():
    for nm, lp in (("adlittle", golden("adlittle")), ("rows_long", rows_long())):
        dlp = engine.lp_to_device(lp, 0)
        snap = _snapshot(_tensors(dlp))
        decreasing = dict(dlp)
        decreasing["a_start"] = dlp["a_start"].clone()
        decreasing["a_start"][1] = decreasing["a_start"][2] + 1
        negative_end = dict(dlp)   # a_start[0] == 0, a_start[num_col] < 0: check_lp's first a_start message
        negative_end["a_start"] = dlp["a_start"].clone()
        negative_end["a_start"][-1] = -1
        wild_end = dict(dlp)   # a descent and a last entry far past a_index's end: rejected before a_index is read
        wild_end["a_start"] = decreasing["a_start"].clone()
        wild_end["a_start"][-1] = 2000000000
        bad_index = dict(dlp)
        bad_index["a_index"] = dlp["a_index"].clone()
        bad_index["a_index"][5] = lp.num_row_
        for hip, who in ((False, "b200pdlp_solve_device"), (True, "b200pdlp_solve_hipdlp_device")):
            for om in (0, -1):
                host_cost = engine.make_clp_device(decreasing)   # a host pointer goes before a malformed a_start
                host_cost.col_cost = engine._p(lp.col_cost_, engine._dp)
                rc, msg = _raw(host_cost, hip, ordered_max=om)
                assert rc == -1 and msg == f"{who}: col_cost is not device memory of device 0", (nm, msg)
                rc, msg = _raw(decreasing, hip, ordered_max=om)
                assert rc == -1 and msg == f"{who}: b200pdlp: a_start must be non-decreasing", (nm, msg)
                rc, msg = _raw(negative_end, hip, ordered_max=om)
                assert rc == -1 and msg == f"{who}: b200pdlp: a_start[0] must be 0 and a_start[num_col] >= 0", (nm, msg)
                rc, msg = _raw(wild_end, hip, ordered_max=om)
                assert rc == -1 and msg == f"{who}: b200pdlp: a_start must be non-decreasing", (nm, msg)
                rc, msg = _raw(bad_index, hip, ordered_max=om)
                assert rc == -1 and msg == f"{who}: b200pdlp: a_index entry outside [0, num_row)", (nm, msg)
        assert _snapshot(_tensors(dlp)) == snap


def case_kkt():
    for nm, lp in (("afiro", golden("afiro")), ("rows_long", rows_long()), ("mixed1", mixed_lp(1))):
        dlp = engine.lp_to_device(lp, 0)
        for got in (engine.solve_device(dlp, iter_limit=2000, ordered_max=-1), engine.solve_device(dlp, iter_limit=2000),
                    engine.solve_hipdlp_device(dlp, iter_limit=2000, ordered_max=-1)):
            dev = engine.kkt_check_batch_device([dlp], [got])[0]
            host = engine.kkt_check_batch([lp], [_host(got)])[0]
            assert dev.keys() == host.keys(), nm
            for k in dev:   # floats bit for bit, everything else by value
                same = (np.float64(dev[k]).tobytes() == np.float64(host[k]).tobytes()) if isinstance(dev[k], float) else dev[k] == host[k]
                assert same, (nm, k, dev[k], host[k])


def case_twice():
    for nm, lp in (("rows_long", rows_long()), ("afiro", golden("afiro"))):
        dlp = engine.lp_to_device(lp, 0)
        for om in (0, -1):
            a = _host(engine.solve_device(dlp, trace_cap=TRACE, iter_limit=800, ordered_max=om))
            b = _host(engine.solve_device(dlp, trace_cap=TRACE, iter_limit=800, ordered_max=om))
            assert_same(a, b, nm)
            a = _host(engine.solve_hipdlp_device(dlp, trace_cap=TRACE, iter_limit=800, ordered_max=om))
            b = _host(engine.solve_hipdlp_device(dlp, trace_cap=TRACE, iter_limit=800, ordered_max=om))
            assert_same(a, b, nm)


CASES = {f"pdlp_instances{k}": case_pdlp_instances(k) for k in range(len(PDLP_SETS))}
CASES.update({f"hip_instances{v}": case_hip_instances(v) for v in range(len(VARIANTS))})
CASES.update(hot_starts=case_hot_starts, synthetic=case_synthetic, big=case_big, degenerate=case_degenerate,
             device_prep_off=case_device_prep_off, no_upload=case_no_upload, errors=case_errors, kkt=case_kkt,
             twice=case_twice)


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
