"""The HiPDLP mode's kernels (reflected Halpern PDHG, solver=hipdlp) against numpy restatements of the HiPDLP oracle
(oracle/hipdlp_oracle.c: halpern_step, fixed_point_error, check_convergence, update_primal_weight, power_method), through the
kernel-level entry points b200pdlp_hipdlp_step / _check / _problem_power_method (engine.HipProblem).  The restatements run on
the oracle's processed and scaled form (oracle.hipdlp_form), which is bit-equal to the engine's host and device prologues.

a. One Halpern step under every SpMV launch shape a matrix family admits (test_gpu_spmv_shapes.py's families and arms):
   x', rx, xn and hslack bit for bit (the device is built with -fmad=false, the oracle's operation order is kept); A * rx
   and so y', yn, ry bit for bit on ordinary rows (<= 512 entries, summed in ascending column order like the oracle's l_ax),
   within the a-priori bound gamma_k sum |a_ij rx_j| on long rows; A'y' likewise per column; a minor step leaves xn, hslack,
   yn and ry alone; every shape returns the same bits, except long rows under the tiled shape.
b. One check in tree and ordered mode, major 0 and 1, scaled and unscaled, with an objective offset: the vectors ax, aty, atdy
   as in (a), the slacks sp, sn bit for bit, and the nine sums -- in ordered mode equal to the sequential index-order sums,
   in tree mode within gamma_N sum |t_i| of the exact sum of their terms (N terms) -- at shapes (n, m) that reach one block,
   n >> m and m >> n, lengths 256 k +- 1, and max(n, m) > 606 208 (the check kernel's grid-stride loop wraps).
c. The device power method: bit for bit in ordered mode; in tree mode within POWER_FACTOR times the spread of the oracle's
   own estimate under three summation orders (hip_set_sum_block 0, 256, 4096).  Measured on an H100 (the spread is a CPU
   number): relative spreads 8.4e-15 (S2), 6.7e-16 (mixed rows), 6.5e-15 (long rows).
d. Trajectories: in ordered mode the engine's per-block trace equals the oracle's trace bit for bit on the five multi-variant
   instances of hipdlp_child.py; in tree mode (S2-size LPs) every trace row up to the first block whose restart decision
   differs stays within TRACE_FACTOR times the oracle's own spread under the three summation orders (floor 1e-10 (1 + |v|)).
   Measured: over 800 iterations (20 blocks, no restart decision differs) the oracle's spread per column is 6e-16 .. 1.3e-13
   relative to 1 + |v|, so the floor decides.

The GPU work runs in child processes (this file with `child <case>`), one JSON line {key: "ok" | error} each: a faulting
kernel must not poison the test session.
"""
import json
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

U = 2.0 ** -53
HALPERN = [(0, 1), (0, 40), (10 ** 6, 7)]   # (halpern_iteration, k_offset)
POWER_FACTOR = 8.0       # tree-mode power method: |lambda - oracle| <= POWER_FACTOR x the oracle's spread over sum orders
TRACE_FACTOR = 10.0      # tree-mode trajectories: the same for every trace column
TRACE_FLOOR = 1e-10      # ... but never tighter than this relative to 1 + |v|
ORACLE_TRACE_COLS = list(range(10)) + list(range(14, 20))
SUM_BLOCKS = (0, 256, 4096)


# ----------------------------------------------------------------------------------------------------------- references
def dmax(a, b):   # std::max(a, b) = a < b ? b : a
    return np.where(a < b, b, a)


def dmin(a, b):   # std::min(a, b) = b < a ? b : a
    return np.where(b < a, b, a)


def hip_form(lp, scaling_mode=5, ruiz_iterations=10):
    """the oracle's processed + scaled form, with its row-major copy (columns ascending within a row)"""
    from oracle import binding as ob
    f = ob.hipdlp_form(lp, scaling_mode, ruiz_iterations)
    n, m = f["n"], f["m"]
    cbeg = f["cbeg"].astype(np.int64)
    cols = np.repeat(np.arange(n), np.diff(cbeg))
    rows = f["cidx"].astype(np.int64)
    order = np.lexsort((cols, rows))
    f["rbeg"] = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=m))]).astype(np.int64)
    f["ridx"], f["rval"] = cols[order].astype(np.int32), f["cval"][order]
    f["cbeg"] = cbeg
    f["scaled"] = scaling_mode != 0
    return f


def _seq(beg, idx, val, v):
    from test_gpu_spmv_shapes import sequential_rows
    return sequential_rows(beg, idx, val, v)


def _row_bound(beg, idx, val, v):
    """gamma_k sum_j |a_ij v_j| per row (k = its length), computed in long double"""
    ld = np.longdouble
    ln = np.diff(beg)
    mag = np.zeros(len(ln), ld)
    nz = np.flatnonzero(ln > 0)
    if nz.size:
        mag[nz] = np.add.reduceat(np.abs(val.astype(ld) * v[idx].astype(ld)), beg[:-1][nz])
    k = ln.astype(ld)
    return (k * ld(U) / (1 - k * ld(U)) * mag * (1 + ld(2.0 ** -40))).astype(np.float64)


def check_spmv(got, beg, idx, val, v, what):
    """ordinary rows bit for bit against the sequential sum, every row within the a-priori bound"""
    from test_gpu_spmv_shapes import LONG, assert_within_bound
    seq = _seq(beg, idx, val, v)
    ln = np.diff(beg)
    bad = np.flatnonzero((ln <= LONG) & (got != seq))
    assert bad.size == 0, (what, f"{bad.size} ordinary rows differ, e.g. {bad[0]}: {got[bad[0]]!r} vs {seq[bad[0]]!r}")
    assert_within_bound(got, beg, idx, val, v, what)
    return seq


def ref_primal(f, ps, w, major, x, xa, aty, xn, hslack):
    """halpern_step's x side (oracle order): -> x', rx, xn, hslack"""
    rho = 1.0
    temp = x - ps * (f["cost"] - aty)
    proj = dmax(f["lower"], dmin(temp, f["upper"]))
    if major:
        xn, hslack = proj, (proj - temp) / ps
    rx = 2.0 * proj - x
    blended = rho * rx + (1.0 - rho) * x
    return w * blended + (1.0 - w) * xa, rx, xn, hslack


def ref_dual(f, ds, w, major, s, y, ya, yn, ry):
    """halpern_step's y side for s = A rx: -> y', yn, ry, and the intermediate temp"""
    rho = 1.0
    temp = y / ds - s
    proj = dmax(-f["rup"], dmin(temp, -f["rlo"]))
    pd = (temp - proj) * ds
    refl = 2.0 * pd - y
    if major:
        yn, ry = pd, refl
    blended = rho * refl + (1.0 - rho) * y
    return w * blended + (1.0 - w) * ya, yn, ry, temp


def check_terms(f, major, x, y, xa, ya, rx, ry, got):
    """the terms of the nine sums, formed elementwise as the kernels form them, from the vectors the check returned"""
    n, m, neq = f["n"], f["m"], f["neq"]
    c, lo, up, rlo = f["cost"], f["lower"], f["upper"], f["rlo"]
    z_n, z_m = np.zeros(n), np.zeros(m)
    t = [None] * 9
    t[0] = (x - rx) * (x - rx) if major else z_n
    t[1] = (y - ry) * (y - ry) if major else z_m
    t[2] = (x - rx) * got["atdy"] if major else z_n
    r = got["ax"] - rlo
    r[neq:] = dmin(0.0, r[neq:])
    if f["scaled"]:
        r = r * f["row_scale"]
    t[3] = r * r
    r = ((c - got["aty"]) - got["sp"]) + got["sn"]
    if f["scaled"]:
        r = r * f["col_scale"]
    t[4] = r * r
    t[5] = c * x
    with np.errstate(invalid="ignore"):   # inf * 0 in the skipped entries
        lo_t = np.where(lo > -np.inf, lo * got["sp"], 0.0)
        up_t = np.where(up < np.inf, -(up * got["sn"]), 0.0)
    t[6] = np.concatenate([rlo * y, lo_t, up_t])
    t[7] = (x - xa) * (x - xa)
    t[8] = (y - ya) * (y - ya)
    return t


def ref_slacks(f, major, hslack, aty):
    if major:
        slack = hslack
    else:
        dres = f["cost"] - aty
        hl, hu = f["lower"] > -np.inf, f["upper"] < np.inf
        slack = np.where(hl & hu, dres, np.where(hl, dmax(0.0, dres), np.where(hu, dmin(0.0, dres), 0.0)))
    return dmax(0.0, slack), dmax(0.0, -slack)


def seq_sum(terms, init=0.0):
    """the sequential index-order sum from `init` (np.add.accumulate adds strictly left to right)"""
    return float(np.add.accumulate(np.concatenate([[init], terms]))[-1])


def step_inputs(f, seed):
    """x, aty and xa that make both bounds of the box projection active where they are finite, y on both sides of -rlo"""
    rng = np.random.default_rng(seed)
    n, m = f["n"], f["m"]
    lo, up = f["lower"], f["upper"]
    mid = np.where(np.isfinite(lo), lo, np.where(np.isfinite(up), up, 0.0))
    x = mid + 2.0 * rng.standard_normal(n)
    aty = f["cost"] + 3.0 * rng.standard_normal(n)
    xa = mid + rng.random(n)
    y = -f["rlo"] * 0.7 + rng.standard_normal(m)
    ya = rng.standard_normal(m)
    return dict(x=x, xa=xa, aty=aty, y=y, ya=ya)


# ----------------------------------------------------------------------------------------------------------- LP families
def mixed_cols_lp(m=6000, n=5000, seed=7):
    """mixed_rows_lp (every row class, a 1e25 row bound, boxed / fixed columns, maximised with an offset) with upper-only and
    free columns as well; the slack columns of free rows are free too"""
    from test_gpu_hipdlp_device_prep import mixed_rows_lp
    from highs_b200.lp import kHighsInf
    lp = mixed_rows_lp(m, n, seed)
    lp.col_lower_[5::13] = -kHighsInf                # upper-only
    lp.col_lower_[6::17] = -kHighsInf                # free
    lp.col_upper_[6::17] = kHighsInf
    return lp


def _planted(m, n, rows, cols, seed, name):
    from test_gpu_spmv_shapes import _planted_lp
    return _planted_lp(m, n, np.asarray(rows), np.asarray(cols), np.random.default_rng(seed), name)


def check_shape_lps():
    """(name, lp): one block, n >> m and m >> n beyond 606 208 (the grid-stride loop wraps), lengths 256 k +- 1"""
    from highs_b200.lp import synthetic_lp
    rng = np.random.default_rng(5)
    out = [("one_block", synthetic_lp(150, 120, 4, 3))]
    n = 650_001                                        # wide: every column has 2 entries among 2049 rows
    out.append(("wide_650001x2049", _planted(2049, n, rng.integers(0, 2049, 2 * n), np.repeat(np.arange(n), 2), 1, "wide")))
    m = 650_003                                        # tall: every row has 2 entries among 1023 columns
    out.append(("tall_1023x650003", _planted(m, 1023, np.repeat(np.arange(m), 2), rng.integers(0, 1023, 2 * m), 2, "tall")))
    out.append(("len_256k_pm1", synthetic_lp(256 * 40 - 1, 256 * 40 + 1, 5, 9)))
    out.append(("mixed_cols", mixed_cols_lp()))
    return out


# ----------------------------------------------------------------------------------------------------------- child side
def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _problem_with_shape(lp, arm, **prm):
    """engine.HipProblem(lp) with the arm's environment; returns (problem, shapes parsed from the `SpMV shapes:` line)"""
    from highs_b200 import engine
    from test_gpu_spmv_shapes import ARMS, _ENV, _SHAPE_RE
    for k in _ENV:
        os.environ.pop(k, None)
    os.environ.update(ARMS[arm][0])
    os.environ["B200PDLP_TIMING"] = "1"
    sys.stderr.flush()
    with tempfile.TemporaryFile() as tf:
        saved = os.dup(2)
        os.dup2(tf.fileno(), 2)
        try:
            prob = engine.HipProblem(lp, **prm)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            for k in _ENV + ("B200PDLP_TIMING",):
                os.environ.pop(k, None)
        tf.seek(0)
        err = tf.read().decode(errors="replace")
    found = _SHAPE_RE.findall(err)
    assert found, f"{arm}: no SpMV shape line"
    g = found[-1]
    return prob, {"A": (g[0], int(g[1]), int(g[2]), int(g[3])), "A'": (g[4], int(g[5]), int(g[6]), int(g[7]))}


def _step_case(f, prob, ins, hi, ko, major, memo):
    """one step on the device and its checks against the restatement; returns the device's outputs.  memo keeps what does
    not depend on the launch shape (the restatement, and A'y' for a y' already checked)"""
    n, m = f["n"], f["m"]
    ps, ds = 0.37, 1.9
    k = hi + ko
    w = k / (k + 1.0)
    rng = np.random.default_rng(hi + 31 * ko + major)
    sent = dict(xn=rng.standard_normal(n), hslack=rng.standard_normal(n), yn=rng.standard_normal(m), ry=rng.standard_normal(m))
    got = prob.step(ps, ds, hi, ko, major, ins["x"], ins["xa"], ins["aty"], ins["y"], ins["ya"], **sent)
    tag = (hi, ko, major)
    xr, rx, xn, hs = ref_primal(f, ps, w, major, ins["x"], ins["xa"], ins["aty"], sent["xn"], sent["hslack"])
    for key, ref in (("x", xr), ("rx", rx), ("xn", xn), ("hslack", hs)):
        assert got[key].tobytes() == ref.tobytes(), (tag, key, np.flatnonzero(got[key] != ref)[:5])
    if not major:
        for key in ("xn", "hslack", "yn", "ry"):
            assert got[key].tobytes() == sent[key].tobytes(), (tag, "a minor step wrote", key)
    # A rx: rows of ordinary length bit for bit (so y', yn, ry too); long rows within the bound
    from test_gpu_spmv_shapes import LONG
    rlen = np.diff(f["rbeg"])
    if tag not in memo:
        s_seq = _seq(f["rbeg"], f["ridx"], f["rval"], rx)
        bnd = _row_bound(f["rbeg"], f["ridx"], f["rval"], rx)
        memo[tag] = (bnd, ref_dual(f, ds, w, major, s_seq, ins["y"], ins["ya"], sent["yn"], sent["ry"]))
    bnd, (yr, ynr, ryr, temp) = memo[tag]
    ordinary = rlen <= LONG
    for key, ref in (("y", yr), ("yn", ynr), ("ry", ryr)):
        bad = np.flatnonzero(ordinary & (got[key] != ref))
        assert bad.size == 0, (tag, key, bad[:5], got[key][bad[:3]], ref[bad[:3]])
        if (~ordinary).any():
            # y' moves by at most 2 w ds |ds| per unit of A rx; plus the rounding of the intermediate temp and of y'
            lim = 2.0 * ds * (bnd + 4 * U * np.abs(temp)) + 4 * U * (np.abs(ref) + np.abs(ins["ya"]) + np.abs(ins["y"]))
            dev = np.abs(got[key] - ref)
            bad = np.flatnonzero(~ordinary & (dev > lim))
            assert bad.size == 0, (tag, key, "long rows", bad[:5], dev[bad[:3]], lim[bad[:3]])
    seen = memo.setdefault(("aty", tag), {})
    key = (got["y"].tobytes(), got["aty"].tobytes())
    if key not in seen:
        check_spmv(got["aty"], f["cbeg"], f["cidx"], f["cval"], got["y"], (tag, "A'y'"))
        seen[key] = True
    return got


def _child_step(family):
    from test_gpu_spmv_shapes import ARMS, FAMILIES, LONG, _family, assert_shape
    sms = _sm_count()
    if family == "mixed_cols":
        # (6000 rows: too few for a persistent grid)
        lp, arms = mixed_cols_lp(), ("default", "tiled_bulk_copy", "tiled_cooperative_loads")
    else:
        lp, arms = _family(family, sms), FAMILIES[family]
    f = hip_form(lp)
    ins = step_inputs(f, 3)
    out, got, memo = {}, {}, {}
    rlen = np.diff(f["rbeg"])
    for arm in arms:
        key = f"{family}#{arm}"
        try:
            prob, shapes = _problem_with_shape(lp, arm, ordered_max=-1)
            try:
                assert_shape(arm, shapes, {"A": f["m"], "A'": f["n"]}, sms)
                got[arm] = {}
                for hi, ko in HALPERN:
                    for major in (0, 1):
                        got[arm][(hi, ko, major)] = _step_case(f, prob, ins, hi, ko, major, memo)
            finally:
                prob.close()
            out[key] = "ok"
        except Exception as e:   # noqa: BLE001
            out[key] = f"{type(e).__name__}: {e}"[:600]
    base = got.get(arms[0])
    for arm, g in got.items():
        if base is None or arm == arms[0]:
            continue
        key = f"{family}#{arm}#same_bits"
        try:
            for case, r in g.items():
                for k, v in r.items():
                    u = base[case][k]
                    if ARMS[arm][1] == "tiled" and k in ("y", "yn", "ry", "aty"):
                        # long rows of A (and every column of A'y' whose sum reads one of them) may differ
                        keep = (rlen <= LONG) if k != "aty" else np.zeros(f["n"], bool)
                        u, v = u[keep], v[keep]
                    assert u.tobytes() == v.tobytes(), (case, k)
            out[key] = "ok"
        except Exception as e:   # noqa: BLE001
            out[key] = f"{type(e).__name__}: {e}"[:600]
    return out


def _check_case(f, prob, ordered, major, offset, seed):
    rng = np.random.default_rng(seed)
    n, m = f["n"], f["m"]
    x, xa, rx, hslack = (rng.standard_normal(n) for _ in range(4))
    y, ya, ry = (rng.standard_normal(m) for _ in range(3))
    got = prob.check(major, x, y, xa, ya, rx if major else None, ry if major else None, hslack if major else None)
    tag = ("ordered" if ordered else "tree", major)
    check_spmv(got["ax"], f["rbeg"], f["ridx"], f["rval"], x, (tag, "A x"))
    check_spmv(got["aty"], f["cbeg"], f["cidx"], f["cval"], y, (tag, "A'y"))
    if major:
        check_spmv(got["atdy"], f["cbeg"], f["cidx"], f["cval"], y - ry, (tag, "A'(y - ry)"))
    else:
        assert not got["atdy"].any(), tag
    sp, sn = ref_slacks(f, major, hslack, got["aty"])
    assert got["sp"].tobytes() == sp.tobytes() and got["sn"].tobytes() == sn.tobytes(), (tag, "slacks")
    t = check_terms(f, major, x, y, xa, ya, rx, ry, got)
    s = got["sums"]
    for q in range(9):
        init = offset if q in (5, 6) else 0.0
        if ordered:
            ref = seq_sum(t[q], init)
            assert s[q] == ref or (s[q] != s[q] and ref != ref), (tag, q, s[q], ref)
        else:
            if not major and q < 3:
                assert s[q] == 0.0, (tag, q, s[q])
                continue
            N = len(t[q])
            exact = math.fsum(np.concatenate([t[q], [init]]))
            lim = N * U / (1 - N * U) * math.fsum(np.abs(t[q])) * (1 + 2.0 ** -40) + 2 * U * abs(s[q])
            assert abs(s[q] - exact) <= lim, (tag, q, s[q], exact, lim)
    return got


def _child_check(lp_name):
    from highs_b200.lp import synthetic_lp
    if lp_name == "ordered_mixed":
        lps = [("ordered_mixed", mixed_cols_lp(3000, 2500, 5))]
    elif lp_name == "scaling_modes":
        lps = [("synthetic_12k", synthetic_lp(12000, 9000, 6, 21))]
    else:
        lps = [(nm, lp) for nm, lp in check_shape_lps() if nm == lp_name]
    out = {}
    for name, lp in lps:
        lp.offset_ = 2.75
        for scaling_mode in (5, 0):
            f = hip_form(lp, scaling_mode)
            ordered = lp_name == "ordered_mixed"
            key0 = f"{name}#scaling{scaling_mode}"
            try:
                if ordered:
                    assert max(f["n"], f["m"]) <= 4096
                prm = dict(scaling_mode=scaling_mode) if ordered else dict(scaling_mode=scaling_mode, ordered_max=-1)
                from highs_b200 import engine
                prob = engine.HipProblem(lp, **prm)
                try:
                    assert (prob.n, prob.m) == (f["n"], f["m"])
                    for major in (0, 1):
                        _check_case(f, prob, ordered, major, lp.offset_, 17 + major)
                finally:
                    prob.close()
                out[key0] = "ok"
            except Exception as e:   # noqa: BLE001
                out[key0] = f"{type(e).__name__}: {e}"[:600]
    return out


def _child_power():
    """the device power method: ordered mode bit for bit; tree mode within POWER_FACTOR x the oracle's order spread"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    from oracle import binding as ob
    out, spreads = {}, {}
    cases = [("afiro_like_ordered", synthetic_lp(900, 700, 5, 2), True), ("mixed_ordered", mixed_cols_lp(3000, 2500, 5), True),
             ("s2_tree", synthetic_lp(100_000, 100_000, 10, 12345), False),
             ("mixed_tree", mixed_cols_lp(), False),
             ("long_rows_tree", __import__("test_gpu_hipdlp_device_prep").long_rows_lp(), False)]
    for name, lp, ordered in cases:
        try:
            lam = {}
            try:
                for b in SUM_BLOCKS:
                    ob.hipdlp_set_sum_block(b)
                    lam[b] = ob.hipdlp_form(lp)["op_norm_sq"]
            finally:
                ob.hipdlp_set_sum_block(0)
            prob = engine.HipProblem(lp, **({} if ordered else dict(ordered_max=-1)))
            try:
                got = prob.power_method()
                again = prob.power_method()
            finally:
                prob.close()
            assert got == again, ("not deterministic", got, again)
            if ordered:
                assert got == lam[0], (got, lam[0])
            else:
                spread = max(lam.values()) - min(lam.values())
                spreads[name] = spread / lam[0]
                lim = max(POWER_FACTOR * spread, 4 * U * lam[0])
                assert abs(got - lam[0]) <= lim, (got, lam, lim)
            out[name] = "ok"
        except Exception as e:   # noqa: BLE001
            out[name] = f"{type(e).__name__}: {e}"[:600]
    out["_spreads"] = json.dumps(spreads)
    return out


def _child_trace_ordered():
    """the engine's per-block trace against the oracle's, bit for bit, on the five multi-variant instances"""
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp
    from oracle import binding as ob
    import hipdlp_child
    out = {}
    for name in ("afiro", "adlittle", "sctest", "e226", "25fv47"):
        lp = read_b2lp(os.path.join(ROOT, "tests", "golden", "instances", name + ".b2lp"))
        for vi, prm in enumerate(hipdlp_child.VARIANTS):
            key = f"{name}#{vi}"
            try:
                cap = prm["iter_limit"] // 40 + 2
                ref = ob.hipdlp_solve(lp, max_iterations=prm["iter_limit"], tolerance=prm.get("tolerance", 1e-7),
                                      scaling_mode=prm.get("scaling_mode", 5), ruiz_iterations=prm.get("ruiz_iterations", 10),
                                      step_size_strategy=prm.get("step_size_strategy", 3), trace_cap=cap)
                res = engine.solve_hipdlp(lp, trace_cap=cap, **prm)
                assert max(res["form_cols"], res["form_rows"]) <= 4096
                rt, et = ref["trace"][:, ORACLE_TRACE_COLS], res["trace"]
                assert res["trace_len"] == len(rt) == len(et) > 0, (res["trace_len"], len(rt))
                bad = np.argwhere(rt != et)
                assert bad.size == 0, ("first divergence (row, column)", bad[0].tolist(), et[tuple(bad[0])], rt[tuple(bad[0])])
                # without a trace buffer the solve is the same
                plain = engine.solve_hipdlp(lp, **prm)
                assert plain["iters"] == res["iters"] and plain["trace_len"] == 0
                for k in ("col_value", "row_dual"):
                    assert plain[k].tobytes() == res[k].tobytes(), k
                out[key] = "ok"
            except Exception as e:   # noqa: BLE001
                out[key] = f"{type(e).__name__}: {e}"[:600]
    return out


def tree_trace_lps():
    from highs_b200.lp import synthetic_lp
    from test_gpu_hipdlp_device_prep import mixed_rows_lp
    return {"s2": synthetic_lp(100_000, 100_000, 10, 12345), "s2_banded": synthetic_lp(100_000, 100_000, 10, 12345, band=2048),
            "mixed_rows": mixed_rows_lp()}


TREE_ITERS = 800


def _child_trace_tree(name, strategy):
    """tree mode: the trace up to the first restart decision that differs, within the oracle's own order spread"""
    from highs_b200 import engine
    from oracle import binding as ob
    lp = tree_trace_lps()[name]
    prm = dict(max_iterations=TREE_ITERS, tolerance=1e-4, step_size_strategy=strategy)
    cap = TREE_ITERS // 40 + 2
    refs = {}
    try:
        for b in SUM_BLOCKS:
            ob.hipdlp_set_sum_block(b)
            refs[b] = ob.hipdlp_solve(lp, trace_cap=cap, **prm)
    finally:
        ob.hipdlp_set_sum_block(0)
    res = engine.solve_hipdlp(lp, trace_cap=cap, iter_limit=TREE_ITERS, tolerance=1e-4, step_size_strategy=strategy,
                              ordered_max=-1)
    r0 = refs[0]["trace"][:, ORACLE_TRACE_COLS]
    et = res["trace"]
    # rows the oracle itself agrees on: up to the first restart decision any order changes
    rows = min(len(r0), len(et), *(len(r["trace"]) for r in refs.values()))
    for r in refs.values():
        d = np.flatnonzero(r["trace"][:rows, 14] != refs[0]["trace"][:rows, 14])
        rows = min(rows, d[0] if d.size else rows)
    d = np.flatnonzero(et[:rows, 10] != r0[:rows, 10])
    keep = min(rows, d[0] + 1 if d.size else rows)   # the first differing row still has to agree on the sums
    assert keep >= 2, ("too few comparable blocks", keep, rows)
    spread = np.zeros(16)
    for b in SUM_BLOCKS[1:]:
        rb = refs[b]["trace"][:rows, ORACLE_TRACE_COLS]
        spread = np.maximum(spread, (np.abs(rb - r0[:rows]) / (1 + np.abs(r0[:rows]))).max(axis=0))
    tol = np.maximum(TRACE_FACTOR * spread, TRACE_FLOOR)
    dev = np.abs(et[:keep] - r0[:keep]) / (1 + np.abs(r0[:keep]))
    cols = [1, 2, 3, 4, 5, 6, 7, 8, 9, 11, 12, 13, 14]
    bad = [(int(i), int(j)) for i, j in np.argwhere(dev[:, cols] > tol[cols])]
    assert not bad, ("outside the order spread (row, column)", [(i, cols[j]) for i, j in bad[:5]],
                     dev[:, cols].max(axis=0).tolist(), tol[cols].tolist())
    assert np.array_equal(et[:keep, 0], r0[:keep, 0])
    conv_e, conv_o = res["term_code"] == 0, refs[0]["term_code"] == 0
    assert conv_e == conv_o, ("status", res["term_code"], refs[0]["term_code"], res["iters"], refs[0]["iters"])
    if conv_e:
        t = max(TRACE_FACTOR * spread[6], TRACE_FLOOR)
        po, pe = refs[0]["pobj"], res["primal_obj"]
        assert abs(pe - po) <= t * (1 + abs(po)) or abs(pe - po) <= 1e-4 * (1 + abs(po)), (pe, po)
    return {f"{name}#{strategy}": "ok", f"_spread#{name}#{strategy}": json.dumps(
        dict(rows=int(keep), spread=[float(v) for v in spread[cols]]))}


def _child_mode_mismatch():
    """each family of kernel-level entry points rejects the other family's problems (B200PDLP_ERR_ARG)"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(900, 700, 5, 2)
    out = {}
    hp = engine.HipProblem(lp)
    pp = engine.Problem(lp)
    try:
        L = engine.lib()
        v = np.zeros(4 * (pp.n + pp.m + hp.n + hp.m))
        pv = engine._p(v, engine._dp)
        d = engine.C.c_double()
        f4 = (engine.C.c_float * 4)()
        prm, res = engine.make_params(iter_limit=40), engine.CResult()
        calls = {"spmv_ax": lambda: L.b200pdlp_spmv_ax(hp._h, pv, pv), "spmv_aty": lambda: L.b200pdlp_spmv_aty(hp._h, pv, pv),
                 "primal_step": lambda: L.b200pdlp_primal_step(hp._h, pv, pv, 1.0, pv, engine.C.byref(d)),
                 "dual_step": lambda: L.b200pdlp_dual_step(hp._h, pv, pv, pv, 1.0, pv, pv, engine.C.byref(d)),
                 "residuals": lambda: L.b200pdlp_residuals(hp._h, pv, pv, pv),
                 "bench_spmv": lambda: L.b200pdlp_bench_spmv(hp._h, 0, 1, engine.C.byref(engine.C.c_float())),
                 "bench_pass": lambda: L.b200pdlp_bench_pass(hp._h, 1, f4),
                 "problem_solve": lambda: L.b200pdlp_problem_solve(hp._h, engine.C.byref(prm), None, engine.C.byref(res)),
                 "hipdlp_step": lambda: L.b200pdlp_hipdlp_step(pp._h, 1.0, 1.0, 0, 1, 1, *([pv] * 10)),
                 "hipdlp_check": lambda: L.b200pdlp_hipdlp_check(pp._h, 1, *([pv] * 13)),
                 "hipdlp_power_method": lambda: L.b200pdlp_hipdlp_problem_power_method(pp._h, pv)}
        for what, call in calls.items():
            rc = call()
            msg = L.b200pdlp_last_error().decode()
            out[what] = "ok" if rc == -1 and "HiPDLP" in msg else f"rc {rc}: {msg}"[:300]
        # both problems still work afterwards
        hp.power_method()
        pp.spmv_ax(np.ones(pp.n))
        # an LP without rows (host prologue): no empty permutation is indexed
        from highs_b200.lp import HighsLp, HighsSparseMatrix
        e0 = HighsLp(3, 0, np.array([1.0, -1.0, 0.5]), np.zeros(3), np.full(3, 4.0), np.zeros(0), np.zeros(0),
                     HighsSparseMatrix(3, 0, np.zeros(4, np.int32), np.zeros(0, np.int32), np.zeros(0)), 1, 0.0, "no_rows")
        p0 = engine.HipProblem(e0, ordered_max=-1)
        try:
            z = np.zeros(0)
            r = p0.step(0.5, 1.0, 0, 1, 1, np.array([1.0, 2.0, 5.0]), np.zeros(3), np.zeros(3), z, z)
            assert r["xn"].tolist() == [0.5, 2.5, 4.0], r["xn"]
            c = p0.check(0, r["x"], z, np.zeros(3), z)
            assert math.isclose(c["sums"][5], float(e0.col_cost_ @ r["x"]), rel_tol=1e-15, abs_tol=1e-15), c["sums"]
            assert p0.power_method() == 1.0
            out["no_rows"] = "ok"
        finally:
            p0.close()
    finally:
        hp.close()
        pp.close()
    return out


def child_main(case):
    kind, _, arg = case.partition(":")
    if kind == "step":
        out = _child_step(arg)
    elif kind == "check":
        out = _child_check(arg)
    elif kind == "power":
        out = _child_power()
    elif kind == "trace_ordered":
        out = _child_trace_ordered()
    elif kind == "trace_tree":
        name, strategy = arg.split(",")
        try:
            out = _child_trace_tree(name, int(strategy))
        except Exception as e:   # noqa: BLE001
            out = {f"{name}#{strategy}": f"{type(e).__name__}: {e}"[:800]}
    elif kind == "mode":
        out = _child_mode_mismatch()
    else:
        raise KeyError(case)
    print(json.dumps(out), flush=True)
    return 0


# ----------------------------------------------------------------------------------------------------------- parent side
def _run_child(case, timeout=900):
    from test_gpu_spmv_shapes import _ENV
    env = {k: v for k, v in os.environ.items() if k not in _ENV + ("B200PDLP_TIMING", "B200PDLP_DEVICE_PREP")}
    try:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "child", case], capture_output=True, text=True,
                           timeout=timeout, cwd=ROOT, env=env)
    except subprocess.TimeoutExpired:
        pytest.fail(f"child {case} did not finish in {timeout} s (killed)")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert lines and r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-3000:])
    out = json.loads(lines[-1])
    info = {k: v for k, v in out.items() if k.startswith("_")}
    if info:
        print(case, info)
    return {k: v for k, v in out.items() if not k.startswith("_")}


def _assert_all_ok(out, at_least):
    bad = {k: v for k, v in out.items() if v != "ok"}
    assert len(out) >= at_least and not bad, (len(out), bad)


pytestmark = pytest.mark.gpu

STEP_FAMILIES = ["ragged", "random", "banded_staged", "banded_mixed", "banded_synthetic", "mixed_cols"]


@pytest.mark.parametrize("family", STEP_FAMILIES)
def test_step_under_every_shape(family):
    out = _run_child(f"step:{family}")
    _assert_all_ok(out, 3)


@pytest.mark.parametrize("lp_name", ["one_block", "wide_650001x2049", "tall_1023x650003", "len_256k_pm1", "mixed_cols",
                                     "scaling_modes", "ordered_mixed"])
def test_check_sums_and_vectors(lp_name):
    _assert_all_ok(_run_child(f"check:{lp_name}"), 2)


def test_power_method():
    _assert_all_ok(_run_child("power"), 5)


def test_ordered_trace_equals_oracle_trace():
    _assert_all_ok(_run_child("trace_ordered", timeout=1200), 25)


@pytest.mark.parametrize("name", ["s2", "s2_banded", "mixed_rows"])
@pytest.mark.parametrize("strategy", [0, 3])
def test_tree_trace_within_order_spread(name, strategy):
    _assert_all_ok(_run_child(f"trace_tree:{name},{strategy}", timeout=1200), 1)


def test_mode_mismatch_and_empty_rows():
    _assert_all_ok(_run_child("mode"), 9)


if __name__ == "__main__" and len(sys.argv) >= 3 and sys.argv[1] == "child":
    sys.exit(child_main(sys.argv[2]))
