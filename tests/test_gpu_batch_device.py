"""b200pdlp_solve_batch_device on the GPU: LPs already in device memory, prologue and postsolve on the device.  Every member
must be identical to what b200pdlp_solve_batch returns for the same LP on the host -- byte equality of term_code,
term_iterate, iters, passes, restarts, the six residual scalars, trace columns 0-14, the four vectors and the form
dimensions -- and no input tensor may change."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

from conftest import GOLDEN, golden_lp, load_golden, options_to_params

pytestmark = pytest.mark.gpu

CASES = load_golden()
FILES = sorted(glob.glob(os.path.join(GOLDEN, "instances", "*.b2lp")))
TAGS = ["default", "kkt1e-4", "limit80", "norestart"]
INTS = ("term_code", "term_iterate", "iters", "passes", "restarts", "form_cols", "form_rows", "form_nnz", "form_neq")
SCALARS = ("primal_obj", "dual_obj", "primal_feas", "dual_feas", "gap", "rel_gap")
VECTORS = ("col_value", "col_dual", "row_value", "row_dual")


def _bits(v):
    return np.ascontiguousarray(v, dtype=np.float64).view(np.uint64)


def _host(t):
    return t.cpu().numpy()


def assert_same(dev, host, what=""):
    for k in INTS:
        assert dev[k] == host[k], (what, k, dev[k], host[k])
    for k in SCALARS:
        assert _bits(dev[k]) == _bits(host[k]), (what, k, dev[k], host[k])
    for k in VECTORS:
        assert np.array_equal(_bits(_host(dev[k])), _bits(host[k])), (what, k)
    if "trace" in dev or "trace" in host:
        assert dev["trace"].shape == host["trace"].shape, (what, dev["trace"].shape, host["trace"].shape)
        assert np.array_equal(_bits(dev["trace"][:, :15]), _bits(host["trace"][:, :15])), (what, "trace")


def _ordered(lp, ordered_max=4096):
    from highs_b200 import engine
    f = engine.host_form(lp, 1)
    return max(f["n"], f["m"]) <= ordered_max


def _instances():
    from highs_b200.lp import read_b2lp
    out = []
    for p in FILES:
        lp = read_b2lp(p)
        if _ordered(lp):
            out.append((os.path.basename(p)[:-5], lp))
    return out


def _read(name):
    from highs_b200.lp import read_b2lp
    return read_b2lp(os.path.join(GOLDEN, name + ".b2lp"))


def _snapshot(dlps):
    return [{k: _host(v).tobytes() for k, v in d.items() if hasattr(v, "is_cuda")} for d in dlps]


def _assert_unchanged(dlps, snap):
    for i, (d, s) in enumerate(zip(dlps, snap)):
        for k, b in s.items():
            assert _host(d[k]).tobytes() == b, (i, k)


def _check(lps, names, warms=None, trace_cap=0, **kw):
    """solve_batch_device on device copies of `lps` against solve_batch on the host arrays, inputs untouched"""
    import torch
    from highs_b200 import engine
    dlps = [engine.lp_to_device(lp, 0) for lp in lps]
    dwarms = None if warms is None else [None if w is None else tuple(torch.as_tensor(np.asarray(v, dtype=np.float64)).cuda()
                                                                      for v in w) for w in warms]
    snap = _snapshot(dlps)
    wsnap = None if dwarms is None else [[_host(v).tobytes() for v in w] if w is not None else None for w in dwarms]
    got = engine.solve_batch_device(dlps, warms=dwarms, trace_cap=trace_cap, **kw)
    want = engine.solve_batch(lps, warms=warms, trace_cap=trace_cap, **kw)
    assert len(got) == len(lps)
    for nm, g, w in zip(names, got, want):
        assert_same(g, w, nm)
    _assert_unchanged(dlps, snap)
    if dwarms is not None:
        for w, s in zip(dwarms, wsnap):
            if w is not None:
                assert [_host(v).tobytes() for v in w] == s
    return got


@pytest.mark.parametrize("tag", TAGS)
def test_instances_equal_host_batch(engine_lib, tag):
    """every ordered-mode instance file in one batch, each option set bounded at 400 iterations"""
    inst = _instances()
    assert len(inst) > 40
    params = options_to_params(next(c for c in CASES if c["tag"] == tag)["options"])
    params["iter_limit"] = min(params.get("iter_limit", 400), 400)
    _check([lp for _, lp in inst], [nm for nm, _ in inst], trace_cap=64, **params)


@pytest.mark.parametrize("tag", TAGS)
def test_goldens_iteration_counts(engine_lib, tag):
    from highs_b200 import engine
    cases = [c for c in CASES if c["tag"] == tag and c["warm_from"] is None]
    lps = [golden_lp(c) for c in cases]
    keep = [i for i, lp in enumerate(lps) if _ordered(lp)]
    assert keep
    params = options_to_params(cases[0]["options"])
    got = engine.solve_batch_device([engine.lp_to_device(lps[i], 0) for i in keep], **params)
    for i, g in zip(keep, got):
        assert g["iters"] == cases[i]["pdlp_iteration_count"], (cases[i]["name"], g["iters"])


def test_warm_and_cold_members(engine_lib):
    from highs_b200 import engine
    case = [c for c in CASES if c["warm_from"]][0]
    rlp = golden_lp(case)
    first = dict(np.load(os.path.join(GOLDEN, case["warm_from"])))
    rwarm = (first["col_value"], first["row_value"], first["row_dual"])
    avgas, afiro = _read("avgas"), _read("afiro")
    kw = options_to_params(case["options"])
    own = engine.solve(avgas, **kw)
    awarm = (own["col_value"], own["row_value"], own["row_dual"])
    got = _check([rlp, afiro, avgas, rlp, avgas], ["warm", "afiro", "avgas warm", "cold", "avgas"],
                 warms=[rwarm, None, awarm, None, None], trace_cap=512, **kw)
    assert got[0]["iters"] == case["pdlp_iteration_count"] and got[0]["term_name"] == "OPTIMAL"
    assert got[2]["iters"] == 0


def _edge_lps():
    """empty rows and columns; ranged (BOUND) and free rows; a maximisation with an offset; columns stored with descending
    rows.  (A matrix without any nonzero is left out: amax = 0 makes PDHG's steps infinite, in every solve path.)"""
    from highs_b200.lp import HighsLp, HighsSparseMatrix, synthetic_lp
    inf = np.inf
    af = _read("afiro")
    a = af.a_matrix_
    # afiro with an empty row (ranged) and an empty row (free) appended and two empty columns in front
    start = np.concatenate([[0, 0], a.start_]).astype(np.int32)
    empty = HighsLp(af.num_col_ + 2, af.num_row_ + 2, np.concatenate([[1.0, -1.0], af.col_cost_]),
                    np.concatenate([[0.0, -1.0], af.col_lower_]), np.concatenate([[1.0, 2.0], af.col_upper_]),
                    np.concatenate([af.row_lower_, [-1.0, -inf]]), np.concatenate([af.row_upper_, [1.0, inf]]),
                    HighsSparseMatrix(af.num_col_ + 2, af.num_row_ + 2, start, a.index_.copy(), a.value_.copy()))
    ranged = synthetic_lp(60, 50, 3, 7)
    ranged.row_upper_ = ranged.row_lower_ + 2.0
    ranged.row_lower_[::7] = -inf
    ranged.row_upper_[::7] = inf     # free rows
    ranged.row_upper_[1::7] = ranged.row_lower_[1::7]     # and equalities
    afiro = _read("afiro")
    maxi = _read("afiro")
    maxi.col_cost_ = -maxi.col_cost_
    maxi.sense_, maxi.offset_ = -1, 3.5
    rev = _read("afiro")
    a = rev.a_matrix_
    for j in range(rev.num_col_):
        s, e = a.start_[j], a.start_[j + 1]
        a.index_[s:e] = a.index_[s:e][::-1].copy()
        a.value_[s:e] = a.value_[s:e][::-1].copy()
    return [empty, ranged, maxi, rev, afiro], ["empty", "ranged_free", "maximise_offset", "descending_rows", "afiro"]


def test_edge_members(engine_lib):
    lps, names = _edge_lps()
    _check(lps, names, trace_cap=256, iter_limit=3000)


@pytest.mark.parametrize("flags", [dict(scaling=0), dict(adaptive_step=0), dict(iter_limit=0), dict(time_limit=0.0)])
def test_switches(engine_lib, flags):
    lps, names = _edge_lps()
    lps += [_read(nm) for nm in ("avgas", "distillation", "boxed_row")]
    names += ["avgas", "distillation", "boxed_row"]
    kw = dict(tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4, iter_limit=2000)
    kw.update(flags)
    _check(lps, names, trace_cap=64, **kw)


def test_replicated_576(engine_lib):
    inst = _instances()
    lps = [lp for _, lp in inst] * 8
    while len(lps) < 576:
        lps.append(inst[0][1])
    lps = lps[:576]
    _check(lps, [f"member {i}" for i in range(576)], iter_limit=100)


@pytest.mark.parametrize("scaling", [1, 0])
def test_prep_compare(engine_lib, scaling):
    from highs_b200 import engine
    inst = _instances()
    lps, names = _edge_lps()
    lps += [lp for _, lp in inst]
    names += [nm for nm, _ in inst]
    reps = engine.batch_prep_compare(lps, scaling=scaling)
    bad = {nm: {k: v for k, v in r.items() if v != 0} for nm, r in zip(names, reps) if any(v != 0 for v in r.values())}
    assert not bad, bad


# ---- errors: ERR_ARG naming the member, nothing written, nothing read back into the inputs

def _raw_call(dlps, **params):
    """b200pdlp_solve_batch_device through the C ABI with NaN-filled device outputs and sentinel result fields"""
    import torch
    from highs_b200 import engine
    L = engine.lib()
    L.b200pdlp_solve_batch_device.argtypes = [C.c_int32, C.POINTER(engine.CLp), C.POINTER(engine.CParams),
                                              C.POINTER(engine.CWarm), C.POINTER(engine.CResult)]
    count = len(dlps)
    clps, cres, outs = (engine.CLp * count)(), (engine.CResult * count)(), []
    for i, d in enumerate(dlps):
        clps[i] = d if isinstance(d, engine.CLp) else engine.make_clp_device(d)
        n, m = clps[i].num_col, clps[i].num_row
        v = [torch.full((k,), float("nan"), dtype=torch.float64, device="cuda") for k in (n, n, m, m)]
        cres[i].col_value, cres[i].col_dual, cres[i].row_value, cres[i].row_dual = (C.cast(C.c_void_p(t.data_ptr()), engine._dp) for t in v)
        cres[i].term_code, cres[i].iters, cres[i].setup_seconds = -7, -7, -7.0
        outs.append(v)
    prm = engine.make_params(**params)
    rc = L.b200pdlp_solve_batch_device(count, clps, C.byref(prm), None, cres)
    for i in range(count):
        assert cres[i].term_code == -7 and cres[i].iters == -7 and cres[i].setup_seconds == -7.0, i
        assert all(bool(t.isnan().all()) for t in outs[i]), i
    return rc, L.b200pdlp_last_error().decode()


def _bad_batch():
    from highs_b200 import engine
    lps = [_read(nm) for nm in ("afiro", "avgas", "adlittle", "blending")]
    return lps, [engine.lp_to_device(lp, 0) for lp in lps]


def test_host_pointer_is_rejected(engine_lib):
    from highs_b200 import engine
    lps, dlps = _bad_batch()
    snap = _snapshot(dlps)
    clp2 = engine.make_clp_device(dlps[2])
    clp2.col_cost = engine._p(lps[2].col_cost_, engine._dp)
    rc, msg = _raw_call(dlps[:2] + [clp2] + dlps[3:])
    assert rc == -1 and "member 2: col_cost is not device memory" in msg, msg
    _assert_unchanged(dlps, snap)


def test_bad_arrays_name_the_lowest_member(engine_lib):
    lps, dlps = _bad_batch()
    bad_index = dict(dlps[1])
    bad_index["a_index"] = bad_index["a_index"].clone()
    bad_index["a_index"][5] = lps[1].num_row_
    decreasing = dict(dlps[3])
    decreasing["a_start"] = decreasing["a_start"].clone()
    decreasing["a_start"][1] = decreasing["a_start"][2] + 1
    batch = [dlps[0], bad_index, dlps[2], decreasing]
    snap = _snapshot(batch)
    rc, msg = _raw_call(batch)
    assert rc == -1 and "member 1: " in msg and "a_index entry outside" in msg, msg
    rc, msg = _raw_call([dlps[0], dlps[1], dlps[2], decreasing])
    assert rc == -1 and "member 3: " in msg and "non-decreasing" in msg, msg
    _assert_unchanged(batch, snap)


def test_too_large_member_is_rejected(engine_lib):
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lps, dlps = _bad_batch()
    big = engine.lp_to_device(synthetic_lp(5000, 4000, 3, 1), 0)
    batch = dlps[:2] + [big] + dlps[2:]
    snap = _snapshot(batch)
    rc, msg = _raw_call(batch)
    assert rc == -1 and "member 2: standard form 5000 x 4000 exceeds ordered_max = 4096" in msg, msg
    rc, msg = _raw_call(dlps, ordered_max=30)
    assert rc == -1 and "member 0: " in msg and "exceeds ordered_max = 30" in msg, msg
    _assert_unchanged(batch, snap)
