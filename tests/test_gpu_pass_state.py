"""Everything one tree-mode PDHG pass on one GPU leaves behind, under every SpMV launch shape and both L2 cache policies.

b200pdlp_pass_state (engine.Problem.pass_state) seeds both halves of the double buffers, the four average / light-check
sums and the PdhgState scalars, zeroes the two nonzero bitmaps, runs K1 (primal step), K2 (A x' + dual step), K3 (A'y' +
interaction) and K4 (step rule) through the launchers of the solve's pass graph, and returns all of it.  Each test builds
one problem per L2 policy (B200PDLP_L2_HINTS forced to 0 and 1) for one launch shape of test_gpu_pass_partials.SHAPES,
confirmed from the B200PDLP_TIMING=1 lines, and runs eight states on both:

  a cold pass (nothing pending)             e  rejected step (eta far above the limit)
  b dense-check phase (iter 9, cur 1)       f  inter == 0 (x at its lower bound, A'y = c - 1: x' = x, lim = inf)
  c first pass past it (iter 10)            g  fixed step (adaptive 0)
  d light check off                         h  not due (iter == stop_iter): nothing may change

For every state: x' and y' equal numpy replays of primal_update / dual_update bit for bit; A x' and A'y' are within gamma_k
of an extended-precision sum on every row and equal the entry-order sum on rows of <= 512 entries; half `cur` of every
buffer is unchanged; the sums are replayed exactly (xSum and ySum under `pending`, A xSum and A'ySum, which add the OLD
A x and A'y, under pending && light_on && iter < 10); a 0 in a nonzero bitmap means an exact zero, and the y' bitmap is 1
on long rows; the long-row slots and K4's sums equal the replays of test_gpu_pass_partials; the state after the step rule
equals mg_kernels_child.step_rule_replay bit for bit.  The two L2 policies return the same bytes, slots included; the
shapes return the same iterates, sums and bitmaps (long rows of the tiled shape are summed by 1024 threads: bound only).
"""
import hashlib
import math
import re

import numpy as np
import pytest
import scipy.sparse as sp

from mg_kernels_child import dual_replay, gamma_ok, primal_replay, step_rule_replay
from test_gpu_pass_partials import LONG, SHAPES, check_long_slots, k4_sum, long_lines_lp
from test_gpu_spmv_shapes import (ARMS, TILE_ROWS, _ENV, _SHAPE_RE, _long_lines, _planted_lp, _with_long_lines, assert_shape,
                                  assert_within_bound, row_bounds, sequential_rows, sm_count)
from test_gpu_zero_skip import _ZS_RE

pytestmark = pytest.mark.gpu

_L2_RE = re.compile(r"L2 policies: (on|off)")
DENSE = 10          # kDenseChecks
NOT_DUE = 7         # iter == stop_iter of state h
FAR = 1 << 30       # stop_iter of every other state


def _bits(v):
    return np.asarray(v, dtype=np.float64).view(np.uint64)


def _digest(*arrays):
    h = hashlib.sha1()
    for a in arrays:
        h.update(b"-" if a is None else np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


# ---------------------------------------------------------------- LPs
def tails_lp(m=24 * TILE_ROWS - 15, n=24 * TILE_ROWS - 31, seed=17):
    """banded, 0..16 entries per row, a long row and a long column of 5000 and 513 entries (and of 512: ordinary), the
    first 5 % of the rows equalities.  m = 17 (mod 32): the last slice is partly empty; n = 33 (mod 64): K1's odd tail and
    its last bitmap word.  24 tiles (the tiled shape is forced) and enough rows for persistent grids; 12 nnz below the
    H100's L2."""
    rng = np.random.default_rng(seed)
    lr, lc = _long_lines(m, n)
    ln = rng.integers(0, 17, size=m)
    ln[list(lr)] = 0
    rows = np.repeat(np.arange(m), ln)
    cols = np.clip(rows * n // m + rng.integers(-600, 601, size=rows.size), 0, n - 1)
    rows, cols = _with_long_lines(m, n, rows, cols, lr, lc, lambda i, L: i * n // m - L // 2 + np.arange(L),
                                  lambda j, L: j * m // n - L // 2 + np.arange(L))
    lp = _planted_lp(m, n, rows, cols, rng, f"tails_{m}x{n}")
    lp.row_upper_[: m // 20] = lp.row_lower_[: m // 20]   # (contiguous: the standard form puts equality rows first)
    return lp


def tiny_lp(m=17, n=33, seed=4):
    """n < 64: one word of the x' bitmap, written by the odd tail's lane; one slice of rows; two equality rows"""
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(m), 5)
    cols = np.concatenate([rng.choice(n, 5, replace=False) for _ in range(m)])
    lp = _planted_lp(m, n, rows, cols, rng, "tiny_17x33")
    lp.row_upper_[[3, 11]] = lp.row_lower_[[3, 11]]
    return lp


LPS = {"long_lines": lambda: long_lines_lp()[0], "tails": tails_lp, "tiny": tiny_lp}
_LP_CACHE = {}


def get_lp(name):
    if name not in _LP_CACHE:
        _LP_CACHE[name] = LPS[name]()
    return _LP_CACHE[name]


class Form:
    """the problem's own standard form (Problem.vector / csr / neq)"""

    def __init__(self, prob):
        self.n, self.m, self.neq = prob.n, prob.m, prob.neq
        self.c, self.lo, self.up, self.b = (prob.vector(k) for k in ("cost", "lower", "upper", "rhs"))
        rp, col, val = prob.csr()
        self.A = sp.csr_matrix((val, col, rp), shape=(self.m, self.n))
        self.A.sort_indices()
        self.AT = self.A.T.tocsr()
        self.rlen, self.clen = np.diff(self.A.indptr), np.diff(self.AT.indptr)


_FORMS = {}


# ---------------------------------------------------------------- states
BASE = dict(tau=0.37, sigma=0.61, beta=1.7, eta=1e-9, w_pending=0.25, sum_step=1.5, step_iter=5, adaptive=1,
            stop_iter=FAR, light_on=1, pending=1)
STATES = {
    "a_cold": dict(BASE, pending=0, light_on=0, iter=0, step_iter=0, cur=0),
    "b_dense": dict(BASE, iter=DENSE - 1, cur=1),
    "c_past_dense": dict(BASE, iter=DENSE, cur=0),
    "d_light_off": dict(BASE, light_on=0, iter=4, cur=1),
    "e_reject": dict(BASE, eta=1e300, iter=3, step_iter=40, cur=0),
    "f_inter_zero": dict(BASE, iter=2, cur=1),
    "g_fixed": dict(BASE, adaptive=0, iter=6, cur=0),
    "h_not_due": dict(BASE, iter=NOT_DUE, stop_iter=NOT_DUE, cur=1),
}
STATE_FIELDS = ("tau", "sigma", "tau_try", "sigma_try", "eta", "sum_step", "w_pending", "mov", "lim", "iter", "step_iter",
                "cur", "pending", "passes", "rejects")


def state_inputs(f, name):
    """both halves of x, aty, y, ax and the four sums of state `name`.  Half cur: half of the columns at x = 0 with
    aty = c - 1 - |N| (x' = 0 exactly), half of the rows at y = -1e6 (y' = 0 exactly on inequality rows); the other half
    holds values the pass must not read (its outputs overwrite them, or, not due, must leave them)."""
    n, m = f.n, f.m
    rng = np.random.default_rng(sum(map(ord, name)) + 7 * n + m)
    cur = STATES[name]["cur"]
    x = rng.standard_normal((2, n)) * 3.0
    aty = rng.standard_normal((2, n))
    y = rng.standard_normal((2, m))
    ax = rng.standard_normal((2, m))
    if name == "f_inter_zero":
        x[cur], aty[cur] = f.lo, f.c - 1.0
    else:
        zero = rng.random(n) < 0.5
        x[cur] = np.where(zero, f.lo, np.clip(f.lo + rng.random(n), f.lo, f.up))
        aty[cur] = np.where(zero, f.c - 1.0 - np.abs(rng.standard_normal(n)), f.c + rng.standard_normal(n))
    y[cur] = np.where(np.arange(m) % 2 == 0, -1e6, rng.standard_normal(m))
    sums = dict(xsum=rng.standard_normal(n), atysum=rng.standard_normal(n), ysum=rng.standard_normal(m),
                axsum=rng.standard_normal(m))
    return dict(x=x, aty=aty, y=y, ax=ax, **sums)


# ---------------------------------------------------------------- references (cached per LP and input vector)
_SPMV = {}


def spmv_reference(lp_name, which, M, v, got, what):
    """(sequential sums, long rows, their (ref, bound)) of M v; the first call for a vector checks `got` on every row
    against the full bound (assert_within_bound), later calls reuse the long rows' bounds"""
    key = (lp_name, which, _digest(v))
    if key not in _SPMV:
        beg, idx, val = M.indptr.astype(np.int64), M.indices, M.data
        ref, bound = row_bounds(beg, idx, val, v)
        assert_within_bound(got, beg, idx, val, v, what, bounds=(ref, bound))
        longr = np.flatnonzero(np.diff(beg) > LONG)
        _SPMV[key] = (sequential_rows(beg, idx, val, v), longr, ref[longr], bound[longr])
    return _SPMV[key]


def check_spmv(lp_name, which, M, v, got, what):
    seq, longr, ref, bound = spmv_reference(lp_name, which, M, v, got, what)
    body = np.ones(got.size, bool)
    body[longr] = False
    bad = np.flatnonzero(body & (_bits(got) != _bits(seq)))
    assert bad.size == 0, (what, f"{bad.size} rows <= 512 differ from the entry-order sum", bad[:5].tolist())
    dev = np.abs(got[longr].astype(np.longdouble) - ref)
    bad = np.flatnonzero(dev > bound)
    assert bad.size == 0, (what, "long rows outside the bound", longr[bad[:5]].tolist())


# what every arm of an LP and state must share: (lp, state) -> digest, set by the first arm that ran
_ALL_ARMS, _NON_TILED = {}, {}


def same_as_before(store, key, digest, what):
    assert store.setdefault(key, digest) == digest, (what, "differs from an earlier arm")


# ---------------------------------------------------------------- the problems
def create(engine, lp, shape, hints, monkeypatch, capfd, tiny):
    """engine.Problem(lp) in tree mode under the shape's environment and B200PDLP_L2_HINTS=hints; asserts the SpMV shapes,
    zero-skip and the L2 policies the engine reports.  tiny: an LP too small for a persistent grid, and tiled only where
    its tiles' windows fit (B200PDLP_TILE_FORCE), so those arms fall back to one slice per warp."""
    arm, zs = SHAPES[shape]
    for k in _ENV + ("B200PDLP_ZERO_SKIP", "B200PDLP_L2_HINTS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in ARMS[arm][0].items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("B200PDLP_ZERO_SKIP", str(zs))
    monkeypatch.setenv("B200PDLP_L2_HINTS", str(hints))
    monkeypatch.setenv("B200PDLP_TIMING", "1")
    capfd.readouterr()
    prob = engine.Problem(lp, ordered_max=-1)
    err = capfd.readouterr().err
    for k in _ENV + ("B200PDLP_ZERO_SKIP", "B200PDLP_L2_HINTS", "B200PDLP_TIMING"):
        monkeypatch.delenv(k, raising=False)
    try:
        found, zsk, l2 = _SHAPE_RE.findall(err), _ZS_RE.findall(err), _L2_RE.findall(err)
        assert found and zsk and l2, f"{shape}: the engine printed no SpMV shape, zero-skip or L2 policy line"
        g = found[-1]
        shapes = {"A": (g[0], int(g[1]), int(g[2]), int(g[3])), "A'": (g[4], int(g[5]), int(g[6]), int(g[7]))}
        tiled = {w: s[0] == "tiled" for w, s in shapes.items()}
        if not tiny:
            assert_shape(arm, shapes, {"A": prob.m, "A'": prob.n}, sm_count())
        else:
            for w, (name, _, staged, tiles) in shapes.items():
                fits = ARMS[arm][1] == "tiled" and tiles > 0 and 10 * staged >= 9 * tiles
                assert name == ("tiled" if fits else "one slice per warp"), (shape, w, shapes[w])
        a, at = (int(v) for v in zsk[-1])
        assert (a > 0) == (zs == 1 and not tiled["A"]) and (at > 0) == (zs == 1 and not tiled["A'"]), (shape, a, at)
        assert l2[-1] == ("on" if hints else "off"), (shape, hints, l2[-1])
    except BaseException:
        prob.close()
        raise
    return prob, tiled


# ---------------------------------------------------------------- the checks of one pass
def check_pass(lp_name, f, name, inp, r, tiled, what):
    s = dict(STATES[name])
    cur, nxt = s["cur"], 1 - s["cur"]
    due = s["iter"] < s["stop_iter"]
    # the half the pass reads is never written
    for k in ("x", "aty", "y", "ax"):
        assert r[k][cur].tobytes() == inp[k][cur].tobytes(), (what, k, "half cur changed")

    if not due:
        for k in ("x", "aty", "y", "ax", "xsum", "atysum", "ysum", "axsum"):
            assert r[k].tobytes() == inp[k].tobytes(), (what, k, "changed by a pass that is not due")
        for k in ("x_nz", "y_nz"):
            assert r[k] is None or not r[k].any(), (what, k, "written by a pass that is not due")
        want = dict(tau=s["tau"], sigma=s["sigma"], tau_try=s["tau"], sigma_try=s["sigma"], eta=s["eta"],
                    sum_step=s["sum_step"], w_pending=s["w_pending"], mov=0.0, lim=0.0, iter=s["iter"],
                    step_iter=s["step_iter"], cur=cur, pending=s["pending"], passes=0, rejects=0, dx2=0.0, dy2=0.0, inter=0.0)
        for k, v in want.items():
            assert _bits(float(r[k])) == _bits(float(v)), (what, k, r[k], v)
        return

    x, aty, y, ax = inp["x"][cur], inp["aty"][cur], inp["y"][cur], inp["ax"][cur]
    xn, atyn, yn, axn = r["x"][nxt], r["aty"][nxt], r["y"][nxt], r["ax"][nxt]
    # 1. x' and y', bit for bit; A x' and A'y' against the references
    xr = primal_replay(x, f.c, aty, f.lo, f.up, s["tau"])
    bad = np.flatnonzero(_bits(xr) != _bits(xn))
    assert bad.size == 0, (what, "x'", f"{bad.size} columns", bad[:5].tolist(), xn[bad[:3]].tolist(), xr[bad[:3]].tolist())
    check_spmv(lp_name, "A", f.A, xn, axn, (what, "A x'"))
    yr = dual_replay(y, f.b, axn, ax, s["sigma"], f.neq)
    bad = np.flatnonzero(_bits(yr) != _bits(yn))
    assert bad.size == 0, (what, "y'", f"{bad.size} rows", bad[:5].tolist(), yn[bad[:3]].tolist(), yr[bad[:3]].tolist())
    check_spmv(lp_name, "A'", f.AT, yn, atyn, (what, "A'y'"))

    # 2. the sums: replayed exactly; A xSum and A'ySum add the A x and A'y of the iterate the pass started from
    w = s["w_pending"]
    pend, carry = s["pending"] != 0, s["pending"] != 0 and s["light_on"] != 0 and s["iter"] < DENSE
    want = dict(xsum=inp["xsum"] + w * x if pend else inp["xsum"], ysum=inp["ysum"] + w * y if pend else inp["ysum"],
                axsum=inp["axsum"] + w * ax if carry else inp["axsum"],
                atysum=inp["atysum"] + w * aty if carry else inp["atysum"])
    for k, v in want.items():
        bad = np.flatnonzero(_bits(v) != _bits(r[k]))
        assert bad.size == 0, (what, k, f"{bad.size} entries", bad[:5].tolist())

    # 3. the nonzero bitmaps: bit = (value != 0), long rows of A always 1; enough zeros to mean something
    if r["x_nz"] is not None:
        bad = np.flatnonzero(r["x_nz"] != (xn != 0.0))
        assert bad.size == 0, (what, "x' bitmap", f"{bad.size} columns", bad[:5].tolist(), xn[bad[:3]].tolist())
        assert (r["x_nz"] == 0).mean() >= 0.3, (what, "x' has too few exact zeros", (r["x_nz"] == 0).mean())
    if r["y_nz"] is not None:
        want_y = np.where(f.rlen > LONG, 1, yn != 0.0)
        bad = np.flatnonzero(r["y_nz"] != want_y)
        assert bad.size == 0, (what, "y' bitmap", f"{bad.size} rows", bad[:5].tolist(), yn[bad[:3]].tolist())
        assert (r["y_nz"] == 0).mean() >= 0.3, (what, "y' has too few exact zeros", (r["y_nz"] == 0).mean())

    # 4. slots and K4
    dx = x - xn
    d = y - yn
    dx_t, dy_t, in_t = dx * dx, d * d, dx * (aty - atyn)
    for slots, recs, t, lengths, which in ((r["k2"], r["long_a"], dy_t, f.rlen, "K2 |dy|^2"),
                                           (r["k3"], r["long_at"], in_t, f.clen, "K3 interaction")):
        if (lengths > LONG).any():
            check_long_slots(slots, recs, t, lengths, (what, which))
        else:
            assert recs.shape[0] == 0, (what, which, "long-row records without long rows")
    for k, key in (("k1", "dx2"), ("k2", "dy2"), ("k3", "inter")):
        assert _bits(k4_sum(r[k])) == _bits(r[key]), (what, key, r[key], k4_sum(r[k]))
    for key, t in (("dx2", dx_t), ("dy2", dy_t), ("inter", in_t)):
        gamma_ok(r[key], t, (what, key), extra=2048)
    if name == "f_inter_zero":
        assert r["inter"] == 0.0 and r["lim"] == math.inf, (what, r["inter"], r["lim"])

    # 5. the state after the step rule
    st = step_rule_replay(s, r["dx2"], r["dy2"], r["inter"])
    for k in STATE_FIELDS:
        assert _bits(float(r[k])) == _bits(float(st[k])), (what, k, r[k], st[k])
    branch = {"e_reject": (cur, 1), "g_fixed": (nxt, 0)}.get(name, (nxt, 0))
    assert (r["cur"], r["rejects"]) == branch, (what, "branch", r["cur"], r["rejects"])

    # 6. what every arm shares, and what the non-tiled arms share (tiled long rows: 1024-thread sums)
    key = (lp_name, name)
    same_as_before(_ALL_ARMS, key + ("x",), _digest(xn, r["xsum"], r["ysum"], r["axsum"], r["atysum"]), (what, "x', sums"))
    for k in ("x_nz", "y_nz"):
        if r[k] is not None:
            same_as_before(_ALL_ARMS, key + (k,), _digest(r[k]), (what, k))
    if not any(tiled.values()):
        same_as_before(_NON_TILED, key, _digest(yn, axn, atyn), (what, "y', A x', A'y'"))


# ---------------------------------------------------------------- the tests
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("lp_name", list(LPS))
def test_pass_state(engine_lib, monkeypatch, capfd, lp_name, shape):
    """every state on both L2 policies of one launch shape: each pass against the replays, the two policies byte-equal"""
    from highs_b200 import engine
    lp = get_lp(lp_name)
    probs = []
    try:
        for hints in (0, 1):
            probs.append(create(engine, lp, shape, hints, monkeypatch, capfd, tiny=lp_name == "tiny"))
        (p0, tiled), (p1, _) = probs
        if lp_name not in _FORMS:
            _FORMS[lp_name] = Form(p0)
        f = _FORMS[lp_name]
        if lp_name == "tiny":
            assert f.n < 64 and f.neq > 0
        else:
            assert (f.rlen > LONG).any() and (f.clen > LONG).any()
        if lp_name == "tails":
            assert f.n % 64 == 33 and f.m % 32 == 17 and f.neq > 0
        states = [k for k in STATES if k != "f_inter_zero" or np.isfinite(f.lo).all()]
        assert "f_inter_zero" in states, "every LP here has finite lower bounds"
        for name in states:
            inp = state_inputs(f, name)
            rs = [p.pass_state(**inp, **{k: v for k, v in STATES[name].items()}) for p, _ in probs]
            what = (lp_name, shape, name)
            check_pass(lp_name, f, name, inp, rs[0], tiled, what + ("hints 0",))
            # the L2 policies change no byte
            for k, v in rs[0].items():
                if k == "l2_hints":
                    continue
                u = rs[1][k]
                if isinstance(v, np.ndarray) or v is None:
                    assert (v is None and u is None) or (v.shape == u.shape and v.tobytes() == u.tobytes()), (what, k)
                else:
                    assert _bits(float(v)) == _bits(float(u)), (what, k, v, u)
            assert (rs[0]["l2_hints"], rs[1]["l2_hints"]) == (0, 1), what
    finally:
        for p, _ in probs:
            p.close()


def test_defaults_are_pass_partials(engine_lib):
    """pass_state given only tau and sigma is the pass b200pdlp_pass_partials runs: the same bytes for the new iterates,
    the slots and K4's sums, the sums untouched, and the step rule taken (one accepted, adaptive pass)"""
    from highs_b200 import engine
    prob = engine.Problem(get_lp("tails"), ordered_max=-1)
    try:
        n, m = prob.n, prob.m
        rng = np.random.default_rng(9)
        x, aty, y, ax = np.abs(rng.standard_normal(n)), rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)
        sums = dict(xsum=rng.standard_normal(n), atysum=rng.standard_normal(n), ysum=rng.standard_normal(m),
                    axsum=rng.standard_normal(m))
        r = prob.pass_state(np.stack([x, x]), np.stack([aty, aty]), np.stack([y, y]), np.stack([ax, ax]), **sums,
                            tau=0.37, sigma=0.61)
        q = prob.pass_partials(x, y, ax, aty, 0.37, 0.61)
    finally:
        prob.close()
    for k, v in (("x", "x_new"), ("aty", "aty_new"), ("y", "y_new"), ("ax", "ax_new")):
        assert r[k][1].tobytes() == q[v].tobytes(), k
    for k in ("k1", "k2", "k3", "long_a", "long_at"):
        assert r[k].tobytes() == q[k].tobytes(), k
    for k in ("dx2", "dy2", "inter"):
        assert _bits(r[k]) == _bits(q[k]), k
    for k, v in sums.items():
        assert r[k].tobytes() == v.tobytes(), k
    assert (r["passes"], r["iter"], r["step_iter"], r["cur"]) == (1, 1, 1, 1), (r["passes"], r["iter"], r["cur"])


def test_l2_size_rule(engine_lib, monkeypatch, capfd):
    """with B200PDLP_L2_HINTS unset the policies are on where 12 bytes per entry of the matrix reach the L2 size: the
    long-lines LP (above) on, the tails LP (below) off"""
    import torch
    from highs_b200 import engine
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    monkeypatch.delenv("B200PDLP_L2_HINTS", raising=False)
    for lp_name, on in (("long_lines", True), ("tails", False)):
        monkeypatch.setenv("B200PDLP_TIMING", "1")
        capfd.readouterr()
        prob = engine.Problem(get_lp(lp_name), ordered_max=-1)
        err = capfd.readouterr().err
        monkeypatch.delenv("B200PDLP_TIMING")
        try:
            assert (12 * prob.nnz >= l2) == on, (lp_name, prob.nnz, l2)
            assert _L2_RE.findall(err)[-1] == ("on" if on else "off"), (lp_name, _L2_RE.findall(err))
        finally:
            prob.close()
