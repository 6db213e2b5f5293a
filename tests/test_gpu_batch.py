"""b200pdlp_solve_batch on the GPU: every member returns the bits b200pdlp_solve returns for it alone (and, where the single
solve reproduces the oracle bit for bit, the oracle's bits).  "Identical" = byte equality of term_code, term_iterate, iters,
passes, restarts, the six residual scalars, trace columns 0-14 and the four HighsSolution vectors."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

from conftest import GOLDEN, golden_lp, load_golden, options_to_params

pytestmark = pytest.mark.gpu

CASES = load_golden()
FILES = sorted(glob.glob(os.path.join(GOLDEN, "instances", "*.b2lp")))
INTS = ("term_code", "term_iterate", "iters", "passes", "restarts")
SCALARS = ("primal_obj", "dual_obj", "primal_feas", "dual_feas", "gap", "rel_gap")
VECTORS = ("col_value", "col_dual", "row_value", "row_dual")


def _bits(v):
    return np.ascontiguousarray(v, dtype=np.float64).view(np.uint64)


def assert_same(a, b, what=""):
    for k in INTS:
        assert a[k] == b[k], (what, k, a[k], b[k])
    for k in SCALARS:
        assert _bits(a[k]) == _bits(b[k]), (what, k, a[k], b[k])
    for k in VECTORS:
        assert np.array_equal(_bits(a[k]), _bits(b[k])), (what, k)
    if "trace" in a or "trace" in b:
        assert a["trace"].shape == b["trace"].shape, (what, a["trace"].shape, b["trace"].shape)
        assert np.array_equal(_bits(a["trace"][:, :15]), _bits(b["trace"][:, :15])), (what, "trace")


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


def _check_against_single(lps, names, trace_cap=0, **kw):
    from highs_b200 import engine
    got = engine.solve_batch(lps, trace_cap=trace_cap, **kw)
    assert len(got) == len(lps)
    for lp, nm, g in zip(lps, names, got):
        assert_same(g, engine.solve(lp, trace_cap=trace_cap, **kw), nm)
    return got


TAGS = ["default", "kkt1e-4", "limit80", "norestart"]


@pytest.mark.parametrize("tag", TAGS)
def test_batch_equals_single_solve_goldens(engine_lib, tag):
    cases = [c for c in CASES if c["tag"] == tag and c["warm_from"] is None]
    lps = [golden_lp(c) for c in cases]
    keep = [i for i, lp in enumerate(lps) if _ordered(lp)]
    assert keep
    params = options_to_params(cases[0]["options"])
    got = _check_against_single([lps[i] for i in keep], [cases[i]["name"] for i in keep], trace_cap=4096, **params)
    for i, g in zip(keep, got):
        assert g["iters"] == cases[i]["pdlp_iteration_count"], (cases[i]["name"], g["iters"])


@pytest.mark.parametrize("tag", TAGS)
def test_batch_equals_single_solve_instances(engine_lib, tag):
    """every ordered-mode instance file in one batch, each option set bounded at 400 iterations (as tests/test_gpu_instances.py)"""
    inst = _instances()
    assert len(inst) > 40
    params = options_to_params(next(c for c in CASES if c["tag"] == tag)["options"])
    params["iter_limit"] = min(params.get("iter_limit", 400), 400)
    _check_against_single([lp for _, lp in inst], [nm for nm, _ in inst], trace_cap=64, **params)


def _ragged_lp(seed):
    import importlib.util
    spec = importlib.util.spec_from_file_location("_tgs", os.path.join(os.path.dirname(__file__), "test_gpu_solve.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod._ragged_lp(seed)


ORACLE_GROUPS = [
    ({}, ["avgas", "afiro", "adlittle", "boxed_row", "restart_lp", "sctest", "chip"]),
    (dict(tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4), ["distillation", "e226"]),
    (dict(adaptive_step=0, tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4), ["afiro"]),
    (dict(scaling=0, tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4), ["afiro"]),
]


@pytest.mark.parametrize("group", range(len(ORACLE_GROUPS)))
def test_batch_equals_oracle_trajectories(engine_lib, oracle, group):
    """the cases of test_trajectory_bit_exact: trace and vectors equal the oracle's, iteration counts the goldens'"""
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    kw, names = ORACLE_GROUPS[group]
    lps = [read_b2lp(os.path.join(GOLDEN, nm + ".b2lp")) for nm in names]
    got = engine.solve_batch(lps, trace_cap=4096, **kw)
    for nm, lp, g in zip(names, lps, got):
        orc = oracle.solve(lp, trace_cap=4096, **kw)
        assert g["iters"] == orc["iters"] and g["term_code"] == orc["term_code"], nm
        assert len(g["trace"]) == len(orc["trace"]) > 0
        assert np.array_equal(_bits(g["trace"][:, :15]), _bits(orc["trace"][:, :15])), nm
        for k in VECTORS:
            assert np.array_equal(_bits(g[k]), _bits(orc[k])), (nm, k)
        tag = "kkt1e-4" if kw.get("tol_primal") == 1e-4 else "default"
        gold = [c for c in CASES if c["name"] == nm and c["tag"] == tag]
        if gold and "adaptive_step" not in kw and "scaling" not in kw:
            assert g["iters"] == gold[0]["pdlp_iteration_count"], nm


def test_batch_equals_oracle_ragged(engine_lib, oracle):
    from highs_b200 import engine
    lps = [_ragged_lp(seed) for seed in (1, 2, 3, 4)]
    kw = dict(tol_primal=1e-5, tol_dual=1e-5, tol_gap=1e-5, iter_limit=40000)
    got = engine.solve_batch(lps, trace_cap=2048, **kw)
    for lp, g in zip(lps, got):
        orc = oracle.solve(lp, trace_cap=2048, **kw)
        assert g["term_code"] == orc["term_code"] and g["iters"] == orc["iters"]
        assert np.array_equal(_bits(g["trace"][:, :15]), _bits(orc["trace"][:, :15]))
        for k in VECTORS:
            assert np.array_equal(_bits(g[k]), _bits(orc[k])), k


def test_position_and_replication(engine_lib):
    """2 001 members (more CTAs than are resident at once): afiro first, in the middle and last, the instances repeated
    around them; every copy equals its LP solved alone and in a batch of one"""
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    kw = dict(iter_limit=300)
    inst = _instances()
    afiro = read_b2lp(os.path.join(GOLDEN, "afiro.b2lp"))
    names, lps = [], []
    k = 0
    while len(lps) < 2001:
        if len(lps) in (0, 1000, 2000):
            names.append("afiro"); lps.append(afiro)
        else:
            nm, lp = inst[k % len(inst)]
            names.append(nm); lps.append(lp)
            k += 1
    got = engine.solve_batch(lps, **kw)
    alone = {}
    for nm, lp in [("afiro", afiro)] + inst:
        alone[nm] = engine.solve(lp, **kw)
        assert_same(engine.solve_batch([lp], **kw)[0], alone[nm], nm + " batch of one")
    for i, (nm, g) in enumerate(zip(names, got)):
        assert_same(g, alone[nm], f"{nm} at {i}")


def test_hot_start(engine_lib):
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    case = [c for c in CASES if c["warm_from"]][0]
    rlp = golden_lp(case)
    first = dict(np.load(os.path.join(GOLDEN, case["warm_from"])))
    rwarm = (first["col_value"], first["row_value"], first["row_dual"])
    avgas = read_b2lp(os.path.join(GOLDEN, "avgas.b2lp"))
    afiro = read_b2lp(os.path.join(GOLDEN, "afiro.b2lp"))
    kw = options_to_params(case["options"])
    own = engine.solve(avgas, **kw)
    awarm = (own["col_value"], own["row_value"], own["row_dual"])
    lps = [rlp, afiro, avgas, rlp, avgas]
    warms = [rwarm, None, awarm, None, None]
    got = engine.solve_batch(lps, warms=warms, trace_cap=512, **kw)
    for lp, w, g in zip(lps, warms, got):
        assert_same(g, engine.solve(lp, warm=w, trace_cap=512, **kw))
    assert got[0]["iters"] == case["pdlp_iteration_count"] and got[0]["term_name"] == "OPTIMAL"
    assert got[2]["iters"] == 0 and got[2]["term_name"] == "OPTIMAL"


def _small_set():
    from highs_b200.lp import read_b2lp
    return [read_b2lp(os.path.join(GOLDEN, nm + ".b2lp")) for nm in ("afiro", "avgas", "distillation", "boxed_row", "blending")]


def test_iteration_limit(engine_lib):
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    lp = read_b2lp(os.path.join(GOLDEN, "distillation.b2lp"))
    got = _check_against_single([lp] + _small_set(), ["distillation"] * 6, trace_cap=64,
                                tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4, iter_limit=80)
    assert got[0]["iters"] == 79 and got[0]["term_name"] == "TIMELIMIT_OR_ITERLIMIT"
    for lim in (0, 1):
        _check_against_single(_small_set(), ["small"] * 5, trace_cap=8, iter_limit=lim)


def test_time_limit_zero(engine_lib):
    from highs_b200 import engine
    got = engine.solve_batch(_small_set(), trace_cap=8, time_limit=0.0)
    for g in got:
        assert g["iters"] == 0 and g["term_name"] == "TIMELIMIT_OR_ITERLIMIT" and len(g["trace"]) == 1
    for lp, g in zip(_small_set(), got):
        assert_same(g, engine.solve(lp, trace_cap=8, time_limit=0.0))


def test_infeasible_and_unbounded(engine_lib):
    lps = [golden_lp(c) for c in CASES if c["name"] in ("infeasible", "unbounded") and c["tag"] == "kkt1e-4"]
    assert len(lps) == 2
    got = _check_against_single(lps, ["infeasible", "unbounded"], trace_cap=256,
                                tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4)
    assert all(g["term_code"] in (1, 2, 3) for g in got)


@pytest.mark.parametrize("flags", [dict(scaling=0), dict(adaptive_step=0), dict(restart=0)])
def test_feature_switches(engine_lib, flags):
    _check_against_single(_small_set(), ["small"] * 5, trace_cap=1024, tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4,
                          iter_limit=20000, **flags)


@pytest.mark.parametrize("interval", [200, 333])
def test_power_table_refill(engine_lib, interval):
    """check_interval > kPowTab (128): a round runs out of step-rule powers before its check, the host refills them"""
    from highs_b200.lp import read_b2lp
    lps = [read_b2lp(os.path.join(GOLDEN, nm + ".b2lp")) for nm in ("adlittle", "distillation")]
    _check_against_single(lps, ["adlittle", "distillation"], trace_cap=1024, check_interval=interval,
                          tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4)


def test_rejection_writes_nothing(engine_lib):
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp, synthetic_lp
    lps = [read_b2lp(os.path.join(GOLDEN, "afiro.b2lp")), synthetic_lp(5000, 5000, 4, 3)]
    clps, cres, keep, arrays = (engine.CLp * 2)(), (engine.CResult * 2)(), [], []
    for i, lp in enumerate(lps):
        clps[i], k = engine.make_clp(lp)
        keep.append(k)
        cres[i], a = engine._mk_result(lp)
        for v in a:
            v.fill(7.0)
        cres[i].term_code, cres[i].iters = -7, -7
        arrays.append(a)
    prm = engine.make_params()
    assert engine_lib.b200pdlp_solve_batch(2, clps, C.byref(prm), None, cres) == -1
    assert b"member 1" in engine_lib.b200pdlp_last_error()
    for i in range(2):
        assert cres[i].term_code == -7 and cres[i].iters == -7
        assert all((v == 7.0).all() for v in arrays[i])
