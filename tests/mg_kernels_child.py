"""Child process of tests/test_gpu_mg_kernels.py: one fused multi-GPU PDHG pass on G logical shards of one device
(b200pdlp_pass_partials_mg), checked rank by rank against numpy replays and extended-precision references.  Run in its own
process so that a stuck barrier can be killed by PID without taking the test session along.
usage: python tests/mg_kernels_child.py <case> <world>      prints one JSON line and exits 0 on success"""
import json
import math
import os
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

from highs_b200 import engine  # noqa: E402
from test_gpu_pass_partials import k4_sum  # noqa: E402  (the 1024-thread order of step_rule_kernel and of the barriers)

SEG = 2048        # entries per segment of a long row (kNnzBlk)
LONG = 512        # rows longer than this are long rows
HUGE = 66_000     # more than 32 segments
U = 2.0 ** -53
ERR_ARG = -1


def _bits(v):
    return np.asarray(v, dtype=np.float64).view(np.uint64)


# ---------------------------------------------------------------- LPs (tree mode, the standard form is A itself)
def long_lines_lp(m=36_000, n=70_001, seed=41, neq=150):
    """banded rows of 0..16 entries; 30 long rows of 2..8 segments spread over all rows (so every row block of 2, 3 or 4
    ranks holds several) and one of HUGE entries; 12 long columns of 2..8 segments, each contiguous over about a tenth to
    a third of the rows, so that A_g' has long rows on several ranks.  n is odd and n mod 3 != 0: the last shard is
    shorter and padded.  The first `neq` rows are equalities: they all fall into rank 0's row block."""
    from test_gpu_spmv_shapes import _planted_lp, _with_long_lines
    rng = np.random.default_rng(seed)
    rlens = [HUGE] + rng.integers(SEG + 1, 8 * SEG + 1, size=30).tolist()
    clens = rng.integers(2 * SEG + 1, 6 * SEG + 1, size=12).tolist()
    ri = (np.linspace(0.02, 0.98, len(rlens)) * m).astype(np.int64)
    ci = (np.linspace(0.04, 0.96, len(clens)) * n).astype(np.int64)
    lr = dict(zip(ri.tolist(), rng.permutation(rlens).tolist()))
    lc = dict(zip(ci.tolist(), clens))
    ln = rng.integers(0, 17, size=m)
    rows = np.repeat(np.arange(m), ln)
    cols = np.clip(rows * n // m + rng.integers(-400, 401, size=rows.size), 0, n - 1)
    free_c, free_r = np.setdiff1d(np.arange(n), list(lc)), np.setdiff1d(np.arange(m), list(lr))

    def around(free, centre, L):
        k = min(max(int(np.searchsorted(free, centre)) - L // 2, 0), free.size - L)
        return free[k:k + L]

    rows, cols = _with_long_lines(m, n, rows, cols, lr, lc, lambda i, L: around(free_c, i * n // m, L),
                                  lambda j, L: around(free_r, j * m // n, L))
    lp = _planted_lp(m, n, rows, cols, rng, f"mg_long_lines_{m}x{n}")
    lp.row_upper_[:neq] = lp.row_lower_[:neq]
    return lp


def random_lp():
    """600k x 90k, six entries per column and a dense column of 30000 entries (a long row of A_g' on every rank).  At world 2
    each row block has about 300k rows, so A_g x' writes more than 1024 slots and the barriers' 1024 threads add several
    slots each"""
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(600_000, 90_000, 6, seed=23, dense_col_nnz=30_000)
    lp.row_upper_[:40] = lp.row_lower_[:40]
    return lp


def tiny_lp():
    """9 columns, 7 rows: at world 4 the shard length is ((9 + 3) / 4 + 1) & ~1 = 4, and the ranks own 4, 4, 1 and 0 columns"""
    from test_gpu_spmv_shapes import _planted_lp
    rng = np.random.default_rng(5)
    rows = np.repeat(np.arange(7), 4)
    cols = np.concatenate([rng.choice(9, 4, replace=False) for _ in range(7)])
    lp = _planted_lp(7, 9, rows, cols, rng, "mg_tiny")
    lp.row_upper_[:2] = lp.row_lower_[:2]
    return lp


LPS = {"long_lines": long_lines_lp, "random": random_lp, "tiny": tiny_lp}


# ---------------------------------------------------------------- references
def rank_order(vals):
    s = 0.0
    for v in vals:
        s = s + float(v)
    return s


def primal_replay(x, c, aty, lo, up, tau):
    """primal_shard_p2p_kernel's expression (= primal_update, pdhg_arith.cuh)"""
    v = x + (-tau) * c
    v = v + tau * aty
    v = np.where(v < up, v, up)
    return np.where(v > lo, v, lo)


def dual_replay(y, b, ax_new, ax, sigma, neq):
    """dual_update (pdhg_arith.cuh), projected on the rows from neq on"""
    v = y + sigma * b
    v = v + (-2.0 * sigma) * ax_new
    v = v + sigma * ax
    ineq = np.arange(y.size) >= neq
    return np.where(ineq & ~(v > 0.0), 0.0, v)


# the fields of b200pdlp_pass_mg_out that step_rule_replay predicts
MG_STATE = ("step_iter", "iter", "tau", "sigma", "sum_step", "w_pending", "pending", "eta", "tau_try", "sigma_try",
            "accepted_last")


def step_rule_replay(s, dx2, dy2, inter):
    """step_rule (pdhg_arith.cuh) with the power tables fill_pow_tables leaves (glibc pow through math.pow), from the state
    the kernel-level entry points seed: s's scalars, tau_try = tau, sigma_try = sigma, lim 0, passes and rejects 0 (cur,
    adaptive: 0 and 1 unless s has them).  The fixed step (adaptive 0) keeps tau, sigma, eta and the trial steps."""
    rb = math.sqrt(s["beta"])
    mov = dx2 * 0.5 * rb + dy2 / (2.0 * rb)
    r = dict(step_iter=s["step_iter"], iter=s["iter"], tau=s["tau"], sigma=s["sigma"], sum_step=s.get("sum_step", 0.0),
             w_pending=s.get("w_pending", 0.0), pending=s.get("pending", 0), eta=s["eta"], tau_try=s["tau"],
             sigma_try=s["sigma"], cur=s.get("cur", 0), passes=1, rejects=0, mov=mov, lim=0.0)
    if not s.get("adaptive", 1):
        w = math.sqrt(r["tau"] * r["sigma"])
        r.update(sum_step=r["sum_step"] + w, w_pending=w, pending=1, cur=r["cur"] ^ 1, iter=s["iter"] + 1)
        return r
    k = s["step_iter"] + 1
    eta = s["eta"]
    lim = mov / abs(inter) if inter != 0.0 else math.inf
    accept = eta <= lim
    pr, pg = math.pow(k + 1.0, -0.3), math.pow(k + 1.0, -0.6)
    eta_new = min((1.0 - pr) * lim, (1.0 + pg) * eta)
    r.update(step_iter=k, lim=lim)
    if accept:
        r["tau"], r["sigma"] = eta_new / rb, eta_new * rb
        w = math.sqrt(r["tau"] * r["sigma"])
        r.update(sum_step=r["sum_step"] + w, w_pending=w, pending=1, iter=s["iter"] + 1, eta=w, cur=r["cur"] ^ 1)
    else:
        r.update(eta=eta_new, pending=0, rejects=1)
    r.update(tau_try=r["eta"] / rb, sigma_try=r["eta"] * rb, accepted_last=int(accept))
    return r


def gamma_ok(got, terms, what, extra=0):
    """|got - sum(terms)| <= gamma_k sum |terms|, k = number of terms (+ extra additions), exact sum by math.fsum"""
    t = np.asarray(terms, dtype=np.float64)
    k = t.size + extra + 1
    g = k * U / (1 - k * U)
    ex = math.fsum(t.tolist())
    bound = g * math.fsum(np.abs(t).tolist()) * (1 + 2.0 ** -40) + abs(ex) * U
    assert abs(got - ex) <= bound, (what, got, ex, bound)


class Checker:
    def __init__(self):
        self.fails, self.checked = [], 0

    def __call__(self, name, fn, *a):
        self.checked += 1
        try:
            fn(*a)
        except AssertionError as e:
            self.fails.append(f"{name}: {str(e)[:600]}")
        except Exception:   # noqa: BLE001 -- a crash in a check is a failure of that check
            self.fails.append(f"{name}: {traceback.format_exc()[-600:]}")


# ---------------------------------------------------------------- the standard form, assembled from the ranks
class Form:
    def __init__(self, probs):
        import scipy.sparse as sp
        p0 = probs[0]
        self.n, self.m, self.neq = p0.n, p0.m, p0.neq
        self.c, self.lo, self.up, self.b = (p0.vector(k) for k in ("cost", "lower", "upper", "rhs"))
        self.blocks = []
        for q in probs:
            rp, col, val = q.csr()
            A = sp.csr_matrix((val, col, rp), shape=(q.m_local, self.n))
            self.blocks.append((q.row_offset, q.m_local, A))
        self.A = sp.vstack([a for _, _, a in self.blocks]).tocsr()
        self.rlen = np.diff(self.A.indptr)


def pass_inputs(f, rng, world, part=True):
    n, m = f.n, f.m
    x = np.where(rng.random(n) < 0.4, 0.0, rng.random(n))
    x = np.clip(x, f.lo, f.up)
    y, ax, aty = rng.standard_normal(m), rng.standard_normal(m), rng.standard_normal(n)
    part_in = rng.standard_normal((world, n)) if part else None
    sums = dict(xsum=rng.standard_normal(n), ysum=rng.standard_normal(m), axsum=rng.standard_normal(m),
                atysum=rng.standard_normal(n))
    return dict(x=x, y=y, ax=ax, aty=aty, part_in=part_in, **sums)


def check_pass(ck, f, lp, world, inp, s, r, one=None, tag=""):
    """every check of one pass: inp the inputs, s the scalars, r the result of engine.pass_partials_mg"""
    from test_gpu_spmv_shapes import assert_within_bound
    n, m = f.n, f.m
    ranks = r["ranks"]
    tau, sigma = s["tau"], s["sigma"]
    # the split of the columns and rows
    sl = ranks[0]["shard_len"]

    def split():
        assert sl == ((n + world - 1) // world + 1) & ~1, ("shard_len", sl)
        for g, q in enumerate(ranks):
            assert (q["c0"], q["nl_real"], q["seg_len"]) == (g * sl, max(0, min(sl, n - g * sl)), sl + 2), (g, q["c0"], q["nl_real"])
        assert sum(q["ml"] for q in ranks) == m and [q["r0"] for q in ranks] == [b[0] for b in f.blocks]
    ck(tag + "split", split)

    # 1. x_new: the primal kernel's expression, bit for bit; the A'y it used: the rank-order sum of part_in
    aty_used = r["aty_used"]

    def aty_sum():
        if inp["part_in"] is None:
            assert np.array_equal(_bits(aty_used), _bits(inp["aty"])), "aty changed without part_in"
        else:
            want = np.zeros(n)
            for g in range(world):
                want = want + inp["part_in"][g]
            bad = np.flatnonzero(_bits(want) != _bits(aty_used))
            assert bad.size == 0, (f"{bad.size} columns", bad[:5].tolist(), aty_used[bad[:3]].tolist(), want[bad[:3]].tolist())
    ck(tag + "aty_used", aty_sum)
    xr = primal_replay(inp["x"], f.c, aty_used, f.lo, f.up, tau)

    def xnew():
        bad = np.flatnonzero(_bits(xr) != _bits(r["x_new"]))
        assert bad.size == 0, (f"{bad.size} columns", bad[:5].tolist(), r["x_new"][bad[:3]].tolist(), xr[bad[:3]].tolist())
        if one is not None:
            bad = np.flatnonzero(_bits(one["x_new"]) != _bits(r["x_new"]))
            assert bad.size == 0, (f"{bad.size} columns differ from the one-GPU pass", bad[:5].tolist())
    ck(tag + "x_new", xnew)
    x_new = r["x_new"]

    # 2. ax_new and the partial A_g'y'
    y_new = r["y_new"]
    h = engine.host_layout_eval(lp, world, -1, x_new, y_new)
    clen_g = [np.bincount(a.indices, minlength=n) for _, _, a in f.blocks]

    def ax():
        short = f.rlen <= LONG
        bad = np.flatnonzero(short & (_bits(h["ax"]) != _bits(r["ax_new"])))
        assert bad.size == 0, (f"{bad.size} rows <= 512 differ from form_layout_eval", bad[:5].tolist())
        assert_within_bound(r["ax_new"], f.A.indptr, f.A.indices, f.A.data, x_new, "ax_new")
    ck(tag + "ax_new", ax)

    def parts():
        for g, (r0, ml, a) in enumerate(f.blocks):
            short = clen_g[g] <= LONG
            bad = np.flatnonzero(short & (_bits(h["parts"][g]) != _bits(r["part"][g])))
            assert bad.size == 0, (g, f"{bad.size} columns <= 512 differ from form_layout_eval", bad[:5].tolist())
            at = a.T.tocsr()
            assert_within_bound(r["part"][g], at.indptr, at.indices, at.data, y_new[r0:r0 + ml], f"part {g}")
        want = np.zeros(n)
        for g in range(world):
            want = want + r["part"][g]
        bad = np.flatnonzero(_bits(want) != _bits(r["aty_new"]))
        assert bad.size == 0, (f"reduced aty_new: {bad.size} columns differ from the rank-order sum of part", bad[:5].tolist())
    ck(tag + "part", parts)

    # 3. y_new: dual_update, bit for bit
    def ynew():
        yr = dual_replay(inp["y"], f.b, r["ax_new"], inp["ax"], sigma, f.neq)
        bad = np.flatnonzero(_bits(yr) != _bits(y_new))
        assert bad.size == 0, (f"{bad.size} rows", bad[:5].tolist(), y_new[bad[:3]].tolist(), yr[bad[:3]].tolist())
    ck(tag + "y_new", ynew)

    # 4. the slots of A_g x' per rank, both accumulators; the primal kernel's slots
    dxt = (inp["x"] - x_new) ** 2
    d = inp["y"] - y_new
    dyt = d * d
    it = (inp["ax"] - r["ax_new"]) * d

    def slots():
        for g, q in enumerate(ranks):
            r0, ml, _ = f.blocks[g]
            lens = f.rlen[r0:r0 + ml]
            recs = q["long_a"]
            assert np.array_equal(np.sort(recs[:, 0]), r0 + np.flatnonzero(lens > LONG)), (g, "long rows of A_g")
            assert np.array_equal(recs[:, 2], -(-f.rlen[recs[:, 0]] // SEG)), (g, "segment counts")
            at_long = np.flatnonzero(clen_g[g] > LONG)
            assert np.array_equal(np.sort(q["long_at"][:, 0]), at_long), (g, "long rows of A_g'")
            nb = q["slots"][1]
            order = np.argsort(recs[:, 1])
            first, nseg = recs[order, 1], recs[order, 2]
            body = nb - int(nseg.sum())
            assert recs.shape[0] == 0 or (first[0] == body and np.array_equal(first[1:], first[:-1] + nseg[:-1])), (g, "slots")
            for key, t in (("k2_dy2", dyt), ("k2_inter", it)):
                sv = q[key]
                bad = []
                for row, fs, ns in recs:
                    seg = _bits(sv[fs:fs + ns])
                    if seg[0] != _bits(np.float64(t[row]) + 0.0) or (seg[1:] != 0).any():
                        bad.append(f"row {row} ({ns} segments): term {t[row]!r}, nonzero segments {np.flatnonzero(seg != 0).tolist()}")
                assert not bad, (g, key, f"{len(bad)} of {len(recs)} long rows", bad[:4])
                rows = r0 + np.flatnonzero(lens <= LONG)
                gamma_ok(math.fsum(sv[:body].tolist()), t[rows], (g, key, "body"))
        # the primal kernel's slots of all ranks hold the real columns' terms; the padding adds +0.0
        gamma_ok(math.fsum(np.concatenate([q["k1"] for q in ranks]).tolist()), dxt, "k1 of all ranks")
    ck(tag + "slots", slots)

    # 5. the scalars: the rank-order sums of every rank's 1024-thread slot sums, on every rank; the step rule
    def scalars():
        dx2 = rank_order(k4_sum(q["k1"]) for q in ranks)
        dy2 = rank_order(k4_sum(q["k2_dy2"]) for q in ranks)
        inter = rank_order(k4_sum(q["k2_inter"]) for q in ranks)
        for g, q in enumerate(ranks):
            for k, v in (("dx2", dx2), ("dy2", dy2), ("inter", inter)):
                assert _bits(q[k]) == _bits(v), (g, k, q[k], v)
        gamma_ok(dx2, dxt, "dx2", extra=world + 2048)
        gamma_ok(dy2, dyt, "dy2", extra=world + 2048)
        gamma_ok(inter, it, "inter", extra=world + 2048)
        want = step_rule_replay(s, dx2, dy2, inter)
        for g, q in enumerate(ranks):
            for k in MG_STATE:
                assert _bits(float(q[k])) == _bits(float(want[k])), (g, k, q[k], want[k])
    ck(tag + "scalars", scalars)

    # 6. the dense-phase sums
    def sums():
        w = s.get("w_pending", 0.0)
        pend, accum = s.get("pending", 0) != 0, s.get("pending", 0) != 0 and s.get("light_on", 0) != 0 and s["iter"] < 10
        want = dict(xsum=inp["xsum"] + w * inp["x"] if pend else inp["xsum"],
                    ysum=inp["ysum"] + w * inp["y"] if pend else inp["ysum"],
                    axsum=inp["axsum"] + w * inp["ax"] if accum else inp["axsum"],
                    atysum=inp["atysum"] + w * aty_used if accum else inp["atysum"])
        for k, v in want.items():
            bad = np.flatnonzero(_bits(v) != _bits(r[k]))
            assert bad.size == 0, (k, f"{bad.size} entries", bad[:5].tolist())
    ck(tag + "sums", sums)


def run(case, world):
    lp = LPS[case]()
    out = dict(case=case, world=world)
    ck = Checker()
    rng = np.random.default_rng(100 + world)
    with engine.linked_shards(lp, world, ordered_max=-1) as probs:
        f = Form(probs)
        out.update(n=f.n, m=f.m, neq=f.neq)
        stats_len = [int(v[9]) for v in engine.host_layout_eval(lp, world, -1)["stats"]]
        base = dict(beta=1.7, eta=1e-9, tau=0.37, sigma=0.61, step_iter=5, iter=3, pending=1, w_pending=0.25,
                    sum_step=1.5, light_on=1)
        runs = [("accept_part", dict(base), True),
                ("reject_part", dict(base, eta=1e12, iter=12, step_iter=40), True),
                ("accept_no_part", dict(base, iter=11, pending=1, light_on=1), False),
                ("not_pending", dict(base, pending=0, eta=1e12), True)]
        parities, results = [], []
        for name, s, part in runs:
            inp = pass_inputs(f, rng, world, part)
            r = engine.pass_partials_mg(probs, **inp, **s)
            parities.append([q["parity"] for q in r["ranks"]])
            results.append((name, s, inp, r))
        ones = []
        one_p = engine.Problem(lp, ordered_max=-1)
        try:
            for _, s0, inp0, r0 in results:
                ones.append(one_p.pass_partials(inp0["x"], inp0["y"], inp0["ax"], r0["aty_used"], s0["tau"], s0["sigma"]))
        finally:
            one_p.close()
        for i, (name, s, inp, r) in enumerate(results):
            check_pass(ck, f, lp, world, inp, s, r, ones[i], tag=name + ": ")

        def split():
            q = results[0][3]["ranks"]
            assert stats_len == [r["shard_len"] for r in q], ("shard_len against form_layout_eval", stats_len)
            if case == "tiny" and world == 4:
                assert [r["nl_real"] for r in q] == [4, 4, 1, 0], [r["nl_real"] for r in q]
            got = [r[3]["ranks"][0]["accepted_last"] for r in results]
            assert got == [1, 0, 1, 0], ("accept / reject branches", got)
            if case == "random" and world == 2:
                assert min(r["slots"][1] for r in q) > 1024, ("A_g's slots do not exceed the barrier's threads", [r["slots"] for r in q])
        ck("split and branches", split)

        # 7. parity alternates call by call and is the same on every rank; a repeat on the same inputs returns the same bytes
        def parity():
            for p in parities:
                assert len(set(p)) == 1, ("ranks disagree on the parity", p)
            seq = [p[0] for p in parities]
            assert all(a != b for a, b in zip(seq, seq[1:])), ("parity does not alternate", seq)
        ck("parity", parity)
        name, s, inp, r = results[-1]
        again = engine.pass_partials_mg(probs, **inp, **s)

        def repeat():
            for k in ("x_new", "y_new", "ax_new", "aty_used", "aty_new", "part", "xsum", "ysum", "axsum", "atysum"):
                assert r[k].tobytes() == again[k].tobytes(), k
            for g, (a, b) in enumerate(zip(r["ranks"], again["ranks"])):
                for k, v in a.items():
                    if k == "parity":
                        assert b[k] != v, (g, "the repeat used the same parity")
                    elif isinstance(v, np.ndarray):
                        assert v.tobytes() == b[k].tobytes(), (g, k)
                    else:
                        assert v == b[k] or _bits(float(v)) == _bits(float(b[k])), (g, k, v, b[k])
        ck("repeat", repeat)
    out["parities"] = parities
    out["checked"] = ck.checked
    out["fails"] = ck.fails
    out["ok"] = not ck.fails
    return out


def rejections():
    """argument errors on real problems: ERR_ARG, nothing written, and no barrier launched (the call returns at once)"""
    import ctypes as C
    import time
    L = engine.lib()
    lp = tiny_lp()
    fails = []
    n, m = 9, 7
    cap, long_cap = 4096, 4

    def call(handles, world, cap=cap, long_cap=long_cap, **cin_kw):
        vs = [np.full(4 * max(n, m), 7.0) for _ in range(15)]
        slots = np.full(4 * 3 * cap, 7.0)
        lr = np.full(4 * 3 * long_cap, 7, dtype=np.int32)
        outs = (engine.CPassMgOut * 4)()
        C.memset(outs, 0x5A, C.sizeof(outs))
        before = bytes(outs)
        cin = engine.CPassIn(**dict(dict(tau=0.5, sigma=0.5, beta=1.0, eta=1.0), **cin_kw))
        arr = (C.c_void_p * len(handles))(*handles)
        t0 = time.monotonic()
        rc = L.b200pdlp_pass_partials_mg(arr, world, C.byref(cin), *(engine._p(v, engine._dp) for v in vs), engine._p(slots, engine._dp),
                                         cap, engine._p(lr, engine._ip), long_cap, outs)
        dt = time.monotonic() - t0
        clean = all((v == 7.0).all() for v in vs) and (slots == 7.0).all() and (lr == 7).all() and bytes(outs) == before
        return rc, L.b200pdlp_last_error().decode(), dt, clean

    def expect(what, res, text):
        rc, msg, dt, clean = res
        if rc != ERR_ARG or text not in msg or dt > 5.0 or not clean:
            fails.append(f"{what}: rc {rc}, {msg!r}, {dt:.1f} s, nothing written: {clean}")

    unlinked = [engine.Problem(lp, rank=g, world=2, ordered_max=-1) for g in range(2)]
    try:
        expect("unlinked", call([q._h for q in unlinked], 2), "is not linked")
    finally:
        for q in unlinked:
            q.close()
    with engine.linked_shards(lp, 2, ordered_max=-1) as probs:
        h = [q._h for q in probs]
        expect("rank order", call(h[::-1], 2), "is not rank 0")
        expect("world 1", call(h[:1], 1), "world must be")
        expect("world 17", call(h, 17), "world must be")
        expect("null problem", call([h[0], None], 2), "null argument")
        expect("cap", call(h, 2, cap=0), "cap must be")
        expect("iter < 0", call(h, 2, iter=-1), "iter and step_iter")
        expect("step_iter < 0", call(h, 2, step_iter=-1), "iter and step_iter")
        with engine.linked_shards(lp, 2, ordered_max=-1) as other:
            expect("two worlds", call([h[0], other[1]._h], 2), "is not linked")
        hip = engine.HipProblem(lp)
        try:
            expect("HiPDLP problem", call([h[0], hip._h], 2), "a HiPDLP problem")
        finally:
            hip.close()
    # an LP with a row of 700 entries: each rank's A_g or A_g' has a long row, so long_cap = 0 is too small
    from test_gpu_spmv_shapes import _planted_lp
    rng = np.random.default_rng(8)
    rows = np.concatenate([np.zeros(700, np.int64), rng.integers(1, 60, size=600)])
    cols = np.concatenate([np.arange(700), rng.integers(0, 700, size=600)])
    with engine.linked_shards(_planted_lp(60, 700, rows, cols, rng, "mg_one_long_row"), 2, ordered_max=-1) as probs:
        expect("long_cap", call([q._h for q in probs], 2, long_cap=0), "long_cap >= ")
        # the check on linked ranks: its own scalar rules, and the same problem rules
        vs = [np.full(4096, 7.0) for _ in engine.CHECK_VECTORS]
        outs = (engine.CCheckOut * 2)()
        C.memset(outs, 0x5A, C.sizeof(outs))
        before = bytes(outs)
        arr = (C.c_void_p * 2)(*[q._h for q in probs])
        for what, kw, text in (("check interval 0", dict(interval=0), "interval must be"),
                               ("check light past the dense phase", dict(interval=40, iter=10, light=1), "light check needs"),
                               ("check iter < 0", dict(interval=40, iter=-1), "interval must be")):
            rc = L.b200pdlp_check_device_mg(arr, 2, C.byref(engine.CCheckIn(**kw)), *(engine._p(v, engine._dp) for v in vs), outs)
            msg = L.b200pdlp_last_error().decode()
            if rc != ERR_ARG or text not in msg:
                fails.append(f"{what}: rc {rc}, {msg!r}")
        rc = L.b200pdlp_check_device_mg((C.c_void_p * 2)(arr[1], arr[0]), 2, C.byref(engine.CCheckIn(interval=40)),
                                        *(engine._p(v, engine._dp) for v in vs), outs)
        if rc != ERR_ARG or "is not rank 0" not in L.b200pdlp_last_error().decode():
            fails.append(f"check rank order: rc {rc}")
        if not (all((v == 7.0).all() for v in vs) and bytes(outs) == before):
            fails.append("a rejected check wrote its outputs")
    # (no ordered-mode case: the layout takes ordered mode on one rank only, so every rank of a world is in tree mode)
    return dict(case="rejections", fails=fails, ok=not fails)


# ---------------------------------------------------------------- the check iteration on linked ranks
class LinkedCheck:
    """stands in for the one-GPU problem in test_gpu_check_device's cases: check_device runs b200pdlp_check_device_mg on the
    linked ranks and b200pdlp_check_device on the one-GPU problem with the same inputs, and asserts what the ranks must share
    with each other and with one GPU before the case's own verify() judges rank 0's result"""

    def __init__(self, probs, one, f):
        self.probs, self.one = probs, one
        self.rlen, self.clen = np.diff(f["rbeg"]), np.diff(f["cbeg"])
        self.compared_restarts = 0

    def check_device(self, **kw):
        got = engine.check_device_mg(self.probs, **kw)
        ref = self.one.check_device(**kw)
        assert all(r == got["raw"][0] for r in got["raw"]), "the ranks' b200pdlp_check_out differ"
        # A xbar and A'ybar (split variant) as in the pass: lines of <= 512 entries bit for bit form_layout_eval (A'ybar: the
        # rank-order sum of the ranks' partials); every line within gamma_k of an extended-precision sum (verify, through
        # the bound-only check_spmv installed by run_check)
        if not kw.get("light"):
            h = engine.host_layout_eval(self.one.lp, len(self.probs), -1, got["xavg"], got["yavg"])
            for k, hk, ln in (("axavg", "ax", self.rlen), ("atyavg", "aty", self.clen)):
                bad = np.flatnonzero((ln <= LONG) & (_bits(got[k]) != _bits(h[hk])))
                assert bad.size == 0, (k, f"{bad.size} lines <= 512 differ from form_layout_eval", bad[:5].tolist())
        for k in ("xavg", "yavg"):
            bad = np.flatnonzero(_bits(got[k]) != _bits(ref[k]))
            assert bad.size == 0, (k, f"{bad.size} entries differ from the one-GPU check", bad[:5].tolist())
        if got["restart_choice"] and got["restart_choice"] == ref["restart_choice"]:
            keys = ("x", "y", "xsum", "ysum", "xlr", "ylr") + (("axsum", "atysum") if kw.get("light") else ())
            for k in keys:
                bad = np.flatnonzero(_bits(got[k]) != _bits(ref[k]))
                assert bad.size == 0, (k, "after the restart", f"{bad.size} entries differ from the one-GPU check", bad[:5].tolist())
            self.compared_restarts += 1
        return got


def run_check(world):
    """test_gpu_check_device's verdict scenarios (every split and light case, both infeasibility rays in the current iterate
    and in the average) on `world` linked ranks"""
    from oracle import binding as ob
    import test_gpu_hipdlp_kernels
    from test_gpu_check_device import LIGHT_CASES, SPLIT_CASES, _matrix, check_lp, ray_case, run_case
    from test_gpu_spmv_shapes import assert_within_bound
    # A'ybar on several ranks adds the ranks' partial sums: no line is one sequential sum, so verify() holds the products to
    # the extended-precision bound only, and LinkedCheck checks them bit for bit against form_layout_eval
    test_gpu_hipdlp_kernels.check_spmv = lambda got, beg, idx, val, x, what: assert_within_bound(got, beg, idx, val, x, what)
    out = dict(case="check", world=world)
    fails, hits, measured, compared = [], set(), {}, 0
    lps = [("planted", check_lp(30_001, 20_001, 4_000, sense=-1, offset=2.5, seed=31), SPLIT_CASES + LIGHT_CASES),
           ("farkas", check_lp(30_000, 30_001, 3_000, kind="farkas", sense=1, offset=0.5, seed=41), "primal"),
           ("recession", check_lp(30_001, 30_000, 1_000, kind="recession", sense=-1, offset=1.0, seed=43), "dual")]
    for name, (lp, x0, y0, ray), cases in lps:
        f = ob.formulate_and_scale(lp)
        assert np.array_equal(f["row_new_idx"], np.arange(f["m"]))
        A = _matrix(f)
        one = engine.Problem(lp, ordered_max=-1)
        try:
            with engine.linked_shards(lp, world, ordered_max=-1) as probs:
                shim = LinkedCheck(probs, one, f)
                rng = np.random.default_rng(7 + world)
                todo = [(c[0], c) for c in cases] if isinstance(cases, list) else [(where, where) for where in ("current", "average")]
                for key, c in todo:
                    try:
                        if isinstance(c, str):
                            hits |= ray_case(shim, f, A, lp, x0, y0, ray, cases, c, rng, measured)
                        else:
                            base = (x0 * f["col_scale"], y0 * f["row_scale"])
                            hits |= run_case(shim, f, A, base, c, rng, lp.sense_, lp.offset_, measured)
                    except BaseException as e:   # noqa: BLE001  (pytest.fail raises a BaseException)
                        fails.append(f"{name}#{key}: {type(e).__name__}: {e}"[:700])
                compared += shim.compared_restarts
        finally:
            one.close()
    out.update(fails=fails, hits=sorted(hits), compared_restarts=compared, measured=measured, ok=not fails)
    return out


def main():
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")   # one hardware queue per logical rank's stream
    case = sys.argv[1]
    if case == "rejections":
        out = rejections()
    elif case == "check":
        out = run_check(int(sys.argv[2]))
    else:
        out = run(case, int(sys.argv[2]))
    print(json.dumps(out))
    return 0 if out["ok"] else 1


if __name__ == "__main__":
    sys.exit(main())
