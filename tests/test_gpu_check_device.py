"""The device check iteration of the tree-mode PDLP solve (engine.cu enqueue_check_device: C1 check_avg_xy_kernel, C2 two
plain SpMVs, C3 check_cols_sweep_kernel / check_rows_sweep_kernel, C4 check_decide_kernel -> decide_from_sums, C5
restart_sweep_kernel, C6 check_finish_kernel -> finish_scalars) against a numpy restatement of cuPDLP's check, through the
kernel-level entry point b200pdlp_check_device (engine.Problem.check_device).

The restatement (cupdlp_step.c / cupdlp_solver.c / cupdlp_restart.c / cupdlp_proj.c):
  PDHG_Compute_Average_Iterate        xSum += w x (pending weight), xbar = xSum * (1 / sum_step), scale 1 when sum_step = 0
  PDHG_Compute_Residuals, _Infeas_*   the 28 sums of the fused sweeps (row_terms / col_terms), then the 2 x 10 residuals
  Check_Termination[_Average]         pfeas < tol_p, dfeas < tol_d, relgap < tol_gap on the current, then the average
  Check_Infeasibility                 pinf_obj > 0 and pinf_res < 1e-8 pinf_obj, dinf_obj < 0 and dinf_res < -1e-8 dinf_obj
  limits                              the time-limit word, iter >= iter_limit - 1
  PDHG_Check_Restart_GPU              first check after a restart, artificial (>= 0.36 iter), sufficient (0.2), necessary (0.8)
  PDHG_Restart_Iterate_GPU            copies, cleared sums, |x - x_lr|^2, |y - y_lr|^2
  Compute_Step_Size_Ratio             beta, tau, sigma; the next pass's eta, tau_try, sigma_try
  the next check iteration and the step-rule power tables (k + 1)^-0.3, (k + 1)^-0.6

What each case asserts: averages and flushed sums bit for bit; A xbar / A'ybar bit for bit on ordinary rows and within
gamma_k sum |a x| on long rows; each of the 28 sums within gamma_N sum |t_i| of the exact sum of its terms (formed here
elementwise in double exactly as the sweeps form them); the residuals bit for bit against decide_from_sums's arithmetic on the
device's own sums, and within the bound propagated from the sums to the exact values; term, term_iterate, the restart choice
and the memo equal to the rules applied to the device residuals -- and to the exact residuals, with every deciding comparison
at least MARGIN (relative) away from its threshold, so that no case rests on a tie; after a restart the copies, the cleared
sums and the new restart point bit for bit and |dx|^2, |dy|^2 within their bound; beta, tau, sigma, eta, tau_try, sigma_try
within BETA_ULPS-based bounds of glibc's log / exp (bit for bit when beta is kept); the power tables within POW_ULPS ulps of
glibc's pow (CUDA documents 2 ulps); stop_iter equal to next_check_iter.  The measured spreads are noted beside
POW_ULPS / BETA_ULPS below.

Every verdict and restart branch is reached by construction and the suite asserts that each was hit (see BRANCHES).  The GPU
work runs in child processes (this file with `child <case>`): a faulting kernel must not poison the test session.
"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

U = 2.0 ** -53
EPS = 2.0 ** -52          # one ulp relative to the leading bit
FEAS_TOL = 1e-8           # dFeasTol (cupdlp_utils.c:889)
MARGIN = 1e-6             # deciding comparisons: at least this far (relative) from their thresholds
POW_ULPS = 4.0            # device pow (2 ulps, CUDA C Programming Guide) + glibc pow (< 1 ulp)
BETA_ULPS = 8.0           # beta = exp(lg)^2: plus 4 ulps per unit of |0.5 log(dy/dx)| + |0.5 log sqrt(beta)| (beta_update)
# Measured on an H100 80GB HBM3 (max over every case of this file, relative to glibc): the device's beta, tau, sigma, eta,
# tau_try and sigma_try after a restart equal glibc's log / exp results bit for bit (0 ulps); the power tables are within
# 0.84 ulps of glibc's pow.

BRANCHES = {"term0_current", "term0_average", "term3_primal", "term3_dual", "term4_time", "term4_iter_limit", "go_on",
            "first_after_restart", "artificial_1", "artificial_2", "artificial_exact", "sufficient_1", "sufficient_2",
            "necessary_1", "necessary_2", "no_restart", "beta_kept", "restart_off", "pending0", "pending1",
            "sum_step0", "adaptive0", "adaptive1", "split", "light"}


# ======================================================================================================== the restatement
def next_check_iter(it, interval, iter_limit):
    """cupdlp_solver.c:953-962"""
    nxt = it + 1
    while not (nxt < 10 or nxt % interval == 0 or nxt == iter_limit - 1):
        nxt += 1
    return nxt


def row_terms(y, ax, b, sc, ineq):
    """the four row-side terms of one iterate, as row_terms forms them (every product and sum rounded separately)"""
    r = ax - b
    r = np.where(ineq & ~(r < 0.0), 0.0, r)
    r = r * sc
    k = np.where(ineq & ~(ax < 0.0), 0.0, ax)
    k = k * sc
    return [y * b, r * r, y * y, k * k]


def col_terms(x, aty, c, lo, up, sc):
    """the ten column-side terms of one iterate, as col_terms forms them"""
    hl, hu = lo > -np.inf, up < np.inf
    lf, uf = np.where(hl, lo, 0.0), np.where(hu, up, 0.0)
    isc = 1.0 / sc
    rc = c - aty
    sp = np.where(hl, np.where(rc > 0.0, rc, 0.0), 0.0)
    sn = np.where(hu, np.where(rc < 0.0, -rc, 0.0), 0.0)
    rr = ((rc - sp) + sn) * sc
    k = ((aty + sp) - sn) * sc
    bl = np.where(hl, np.where(x < 0.0, x, 0.0) * isc, 0.0)
    bu = np.where(hu, np.where(x > 0.0, x, 0.0) * isc, 0.0)
    return [x * c, sp * lf, sn * uf, rr * rr, sp * sp, sn * sn, x * x, k * k, bl * bl, bu * bu]


def all_terms(f, x, aty, xa, atya, y, ax, ya, axa):
    """the 28 term vectors in sum order: rows of the current iterate, rows of the average, columns of both"""
    ineq = np.arange(f["m"]) >= f["neq"]
    b, rs = f["rhs"], f["row_scale"]
    c, lo, up, cs = f["cost"], f["lower"], f["upper"], f["col_scale"]
    return (row_terms(y, ax, b, rs, ineq) + row_terms(ya, axa, b, rs, ineq) + col_terms(x, aty, c, lo, up, cs) +
            col_terms(xa, atya, c, lo, up, cs))


def exact_sum(t):
    """(sum, err): the sum of t in extended precision and a bound on its own error"""
    ld = np.longdouble
    if t.size == 0:
        return 0.0, 0.0
    if np.finfo(ld).nmant >= 63:
        a = t.astype(ld)
        s = np.sum(a)   # pairwise: error <= log2(N) eps_ld sum |t|
        err = float(math.ceil(math.log2(t.size) + 1) * float(np.finfo(ld).eps) * float(np.sum(np.abs(a))))
        return float(s), err + U * abs(float(s))
    return math.fsum(t.tolist()), 0.0


def sums_with_bounds(terms):
    """exact sums (as doubles nearest to the extended ones) and gamma_N sum |t| bounds of any double summation order"""
    ex, bd = [], []
    for t in terms:
        s, e = exact_sum(t)
        N = t.size
        mag = float(np.sum(np.abs(t.astype(np.longdouble)))) if N else 0.0
        ex.append(s)
        bd.append(N * U / (1 - N * U) * mag * (1 + 2.0 ** -40) + e + 2 * U * abs(s))
    return ex, bd


def residuals_from_sums(tot, sense, offset):
    """decide_from_sums's scalar arithmetic (pdhg_kernels.cu) on the 28 sums -> [current, average] of 10 values each"""
    out = []
    for t in range(2):
        a = tot[8 + 10 * t: 18 + 10 * t]
        r = tot[4 * t: 4 * t + 4]
        pobj = a[0] * sense + offset
        pfeas = math.sqrt(r[1])
        dobj = ((r[0] + a[1]) - a[2]) * sense + offset
        dfeas = math.sqrt(a[3])
        gap = pobj - dobj
        relgap = abs(pobj - dobj) / (1.0 + abs(pobj) + abs(dobj))
        dscale = math.sqrt(r[2] + a[4] + a[5])
        if dscale < 1e-8:
            dscale = 1.0
        pscale = math.sqrt(a[6])
        if pscale < 1e-8:
            pscale = 1.0
        out.append(dict(pobj=pobj, dobj=dobj, pfeas=pfeas, dfeas=dfeas, gap=gap, relgap=relgap,
                        pinf_obj=(dobj - offset) / sense / dscale, pinf_res=math.sqrt(a[7]) / dscale,
                        dinf_obj=(pobj - offset) / sense / pscale, dinf_res=math.sqrt(r[3] + a[8] + a[9]) / pscale,
                        _dscale=dscale, _pscale=pscale))
    return out


def residual_bounds(ex, bd, R, offset):
    """first-order bounds (x 2) of |residual(device sums) - residual(exact sums)| from the sums' bounds bd and the exact
    residuals R; |sqrt(a) - sqrt(b)| <= sqrt(|a - b|) for the norms"""
    out = []
    for t in range(2):
        a, ab = ex[8 + 10 * t: 18 + 10 * t], bd[8 + 10 * t: 18 + 10 * t]
        r, rb = ex[4 * t: 4 * t + 4], bd[4 * t: 4 * t + 4]
        Q = R[t]
        e = {}
        e["pobj"] = ab[0] + 2 * U * (abs(a[0]) + abs(Q["pobj"]))
        e["dobj"] = rb[0] + ab[1] + ab[2] + 4 * U * (abs(r[0]) + abs(a[1]) + abs(a[2]) + abs(offset))
        e["pfeas"] = math.sqrt(rb[1]) + 2 * U * Q["pfeas"]
        e["dfeas"] = math.sqrt(ab[3]) + 2 * U * Q["dfeas"]
        e["gap"] = e["pobj"] + e["dobj"] + 2 * U * abs(Q["gap"])
        den = 1.0 + abs(Q["pobj"]) + abs(Q["dobj"])
        e["relgap"] = (e["gap"] + Q["relgap"] * (e["pobj"] + e["dobj"])) / den + 4 * U * Q["relgap"]
        eds = math.sqrt(rb[2] + ab[4] + ab[5]) + 2 * U * Q["_dscale"]
        eps_ = math.sqrt(ab[6]) + 2 * U * Q["_pscale"]
        ds, ps = Q["_dscale"], Q["_pscale"]
        e["pinf_obj"] = (e["dobj"] + 2 * U * abs(Q["dobj"] - offset)) / ds + abs(Q["pinf_obj"]) * eds / ds + 4 * U * abs(Q["pinf_obj"])
        e["pinf_res"] = (math.sqrt(ab[7]) + 2 * U * math.sqrt(a[7])) / ds + Q["pinf_res"] * eds / ds + 4 * U * Q["pinf_res"]
        e["dinf_obj"] = (e["pobj"] + 2 * U * abs(Q["pobj"] - offset)) / ps + abs(Q["dinf_obj"]) * eps_ / ps + 4 * U * abs(Q["dinf_obj"])
        dr = math.sqrt(r[3] + a[8] + a[9])
        e["dinf_res"] = (math.sqrt(rb[3] + ab[8] + ab[9]) + 2 * U * dr) / ps + Q["dinf_res"] * eps_ / ps + 4 * U * Q["dinf_res"]
        out.append({k: 2 * v for k, v in e.items()})
    return out


def score(beta, pf, df, gap):
    """PDHG_Restart_Score_GPU (cupdlp_restart.c:113-124)"""
    return math.sqrt(beta * pf * pf + df * df / beta + gap * gap)


class Margins:
    """records each deciding comparison a < b (or a > b) with its relative distance"""

    def __init__(self):
        self.items = []

    def lt(self, a, b, what):
        self.items.append((what, abs(a - b) / max(abs(a), abs(b), 1e-300)))
        return a < b


def decide(R, sc, memo, margins=None):
    """Check_Termination[_Average], Check_Infeasibility, the limits and PDHG_Check_Restart_GPU as decide_from_sums /
    decide_restart_dev run them.  sc: the check's scalars; memo: pf_lr .. gap_lc, last_restart_iter.  Returns
    (term, term_iterate, choice, memo after, branch name)"""
    mg = margins or Margins()
    L, A = R
    memo = dict(memo)
    for ti, Q in enumerate((L, A)):
        if (mg.lt(Q["pfeas"], sc["tol_p"], f"pfeas{ti}") and mg.lt(Q["dfeas"], sc["tol_d"], f"dfeas{ti}") and
                mg.lt(Q["relgap"], sc["tol_gap"], f"relgap{ti}")):
            return 0, ti, 0, memo, "term0_" + ("current" if ti == 0 else "average")
    inf = None
    for Q in (L, A):
        if mg.lt(0.0, Q["pinf_obj"], "pinf_obj") and mg.lt(Q["pinf_res"], FEAS_TOL * Q["pinf_obj"], "pinf_res"):
            inf = inf or "term3_primal"
        if mg.lt(Q["dinf_obj"], 0.0, "dinf_obj") and mg.lt(Q["dinf_res"], -FEAS_TOL * Q["dinf_obj"], "dinf_res"):
            inf = inf or "term3_dual"
    if inf:
        return 3, 0, 0, memo, inf
    if sc["time_flag"]:
        return 4, 0, 0, memo, "term4_time"
    if sc["iter"] >= sc["iter_limit"] - 1:
        return 4, 0, 0, memo, "term4_iter_limit"
    if not sc["restart_on"]:
        return -1, 0, 0, memo, "restart_off"
    it, last, beta = sc["iter"], memo["last_restart_iter"], sc["beta"]
    if it == last:
        for k in ("pf", "df", "gap"):
            memo[k + "_lr"] = memo[k + "_lc"] = L["pfeas" if k == "pf" else "dfeas" if k == "df" else "gap"]
        return -1, 0, 0, memo, "first_after_restart"
    mu_cur, mu_avg = score(beta, L["pfeas"], L["dfeas"], L["gap"]), score(beta, A["pfeas"], A["dfeas"], A["gap"])
    better_cur = mg.lt(mu_cur, mu_avg, "mu_cur<mu_avg")
    choice = 2 if better_cur else 1
    mu_cand = mu_cur if better_cur else mu_avg
    if (it - last) >= 0.36 * it:
        branch = "artificial"
    else:
        mu_lr = score(beta, memo["pf_lr"], memo["df_lr"], memo["gap_lr"])
        if mg.lt(mu_cand, 0.2 * mu_lr, "sufficient"):
            branch = "sufficient"
        else:
            mu_lc = score(beta, memo["pf_lc"], memo["df_lc"], memo["gap_lc"])
            if mg.lt(mu_cand, 0.8 * mu_lr, "necessary_0.8") and mg.lt(mu_lc, mu_cand, "necessary_lc"):
                branch = "necessary"
            else:
                branch, choice = "no_restart", 0
    C = L if better_cur else A
    memo["pf_lc"], memo["df_lc"], memo["gap_lc"] = C["pfeas"], C["dfeas"], C["gap"]
    return -1, 0, choice, memo, branch + (f"_{choice}" if choice else "")


def beta_update(beta, tau, sigma, d2x, d2y, adaptive):
    """PDHG_Compute_Step_Size_Ratio (cupdlp_step.c:147-176) and the next pass's step sizes; glibc log / exp.  Returns the
    values and the relative bound on beta of the device's log / exp"""
    mean = math.sqrt(tau * sigma)
    dxn, dyn = math.sqrt(d2x), math.sqrt(d2y)
    kept = not (min(dxn, dyn) > 1e-10)
    bound = 0.0
    if not kept:
        upd = dyn / dxn
        l1, l2 = 0.5 * math.log(upd), 0.5 * math.log(math.sqrt(beta))
        lg = l1 + l2
        beta = math.exp(lg) * math.exp(lg)
        bound = (BETA_ULPS + 4.0 * (abs(l1) + abs(l2))) * EPS
    tau = mean / math.sqrt(beta)
    sigma = tau * beta
    eta = math.sqrt(tau * sigma)
    if adaptive:
        tt, st = eta / math.sqrt(beta), eta * math.sqrt(beta)
    else:
        tt, st = tau, sigma
    return dict(beta=beta, tau=tau, sigma=sigma, eta=eta, tau_try=tt, sigma_try=st), kept, bound


# ================================================================================================================= LPs
def check_lp(m, n, neq, kind="planted", sense=1, offset=0.0, seed=3, per_row=(1, 6), long_lines=True):
    """A banded LP with an EQ block (rows 0 .. neq-1, they stay first in the standard form) and GEQ rows, columns of every
    kind by j % 5 (lower only, boxed, free, upper only, fixed), one long row and one long column (> 512 entries), and a
    planted optimal pair (x*, y*) in the original space.  kind "farkas": the last two GEQ rows are v'x >= t and -v'x >= 1 - t
    (a Farkas ray e_{m-2} + e_{m-1}); kind "recession": column 5 (x >= 0) has positive entries in GEQ rows only and cost -1
    in the minimisation form.  Returns (lp, x*, y*, ray) with ray = the Farkas y or the recession direction x."""
    from highs_b200.lp import HighsLp, HighsSparseMatrix, kHighsInf
    rng = np.random.default_rng(seed)
    ln = rng.integers(per_row[0], per_row[1] + 1, size=m)
    rows = np.repeat(np.arange(m, dtype=np.int64), ln)
    band = max(8, min(n // 4, 600))
    cols = np.clip(rows * n // m + rng.integers(-band, band + 1, size=rows.size), 0, n - 1)
    if long_lines and min(m, n) > 3000:
        lr, lc = neq + 7 if neq < m - 10 else 3, 11 if n > 20 else 0
        keep = (rows != lr) & (cols != lc)
        rows, cols = rows[keep], cols[keep]
        L1 = min(n - 40, 2049)
        c1 = np.setdiff1d(rng.choice(n, L1 + 8, replace=False), [lc])[:L1 - 1]
        L2 = min(m - 40, 1500)
        r1 = np.setdiff1d(rng.choice(m, L2 + 8, replace=False), [lr, m - 1, m - 2])[:L2]
        rows = np.concatenate([rows, np.full(c1.size, lr), r1])
        cols = np.concatenate([cols, c1, np.full(r1.size, lc)])
    key = np.unique(cols * m + rows)
    c, r = key // m, key % m
    val = rng.uniform(0.5, 2.0, key.size) * np.where(rng.random(key.size) < 0.5, -1.0, 1.0)
    if kind == "recession":
        j0 = 5
        drop = (c == j0) & (r < neq)
        c, r, val = c[~drop], r[~drop], val[~drop]
        val[c == j0] = np.abs(val[c == j0])
    if kind == "farkas":   # the last two rows: the same pattern, opposite values
        drop = r >= m - 2
        c, r, val = c[~drop], r[~drop], val[~drop]
        pc = np.unique(rng.choice(n, 12, replace=False))
        pv = rng.uniform(0.5, 2.0, pc.size)
        c = np.concatenate([c, pc, pc]); r = np.concatenate([r, np.full(pc.size, m - 2), np.full(pc.size, m - 1)])
        val = np.concatenate([val, pv, -pv])
        o = np.lexsort((r, c))
        c, r, val = c[o], r[o], val[o]
    t = np.arange(n) % 5
    lo = np.where(t == 2, -kHighsInf, np.where(t == 3, -kHighsInf, rng.uniform(-2, 1, n)))
    up = np.where(t == 1, lo + rng.uniform(0.5, 3, n), np.where(t == 3, rng.uniform(-1, 2, n), kHighsInf))
    up = np.where(t == 4, lo, up)
    if kind == "recession":
        lo[5], up[5] = 0.0, kHighsInf
    # planted x* and reduced costs z (complementary)
    u01 = rng.random(n)
    x = np.where(t == 2, rng.uniform(-1, 1, n), lo)
    z = np.zeros(n)
    at_lo = (t == 0) & (u01 < 0.6) | (t == 1) & (u01 < 0.4)
    at_up = (t == 1) & (u01 > 0.7) | (t == 3) & (u01 < 0.6)
    interior = ~(at_lo | at_up) & (t != 4)
    x = np.where(at_up, up, x)
    with np.errstate(invalid="ignore"):   # (inf - inf where the other kinds are masked out)
        x = np.where(interior & (t == 0), lo + rng.uniform(0.1, 1, n), x)
        x = np.where(interior & (t == 1), lo + (up - lo) * rng.uniform(0.2, 0.8, n), x)
        x = np.where(interior & (t == 3), up - rng.uniform(0.1, 1, n), x)
    z = np.where(at_lo, rng.uniform(0.1, 1, n), z)
    z = np.where(at_up, -rng.uniform(0.1, 1, n), z)
    z = np.where(t == 4, rng.uniform(-1, 1, n), z)
    ax = np.bincount(r, weights=val * x[c], minlength=m)
    y = np.where(np.arange(m) < neq, rng.uniform(-1, 1, m), np.where(rng.random(m) < 0.5, rng.uniform(0.1, 1, m), 0.0))
    rl = np.where((np.arange(m) >= neq) & (y == 0), ax - rng.uniform(0.1, 1, m), ax)
    ru = np.where(np.arange(m) < neq, rl, kHighsInf)
    ray = None
    if kind == "farkas":
        y[m - 2:] = 0.0
        tt = float(ax[m - 2])
        rl[m - 2], rl[m - 1] = tt, 1.0 - tt
        ray = np.zeros(m); ray[m - 2:] = 1.0
    cmin = np.bincount(c, weights=val * y[r], minlength=n) + z
    if kind == "recession":
        cmin[5] = -1.0
        ray = np.zeros(n); ray[5] = 1.0
    start = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(c, minlength=n), out=start[1:])
    lp = HighsLp(n, m, cmin * sense, lo, up, rl, ru, HighsSparseMatrix(n, m, start.astype(np.int32), r.astype(np.int32), val),
                 sense, offset, f"check_{kind}_{m}x{n}")
    return lp, x, y, ray


# ========================================================================================================== one check
def _matrix(f):
    import scipy.sparse as sp
    return sp.csr_matrix((f["rval"], f["ridx"], f["rbeg"]), shape=(f["m"], f["n"]))


def build_inputs(f, A, base, rng, cur_eps, avg_eps, S, pending, w, light, lr_eps=1e-1, xlr_equal=False):
    """the vectors of one check: current = base + cur_eps noise, average target = base + avg_eps noise, the sums that give
    that average (S = sum_step, with the pending weight w of the current iterate), a restart point lr_eps away"""
    bx, by = base
    nx = lambda v, e: v + e * rng.standard_normal(v.size) * (1 + np.abs(v))
    x, y = nx(bx, cur_eps), nx(by, cur_eps)
    xa, ya = nx(bx, avg_eps), nx(by, avg_eps)
    ax, aty = A @ x, A.T @ y
    if S > 0:
        xsum, ysum = S * xa, S * ya
        if pending:
            xsum, ysum = xsum - w * x, ysum - w * y
    else:
        xsum, ysum = xa, ya
    v = dict(x=x, y=y, ax=ax, aty=aty, xsum=xsum, ysum=ysum, xlr=x.copy() if xlr_equal else nx(bx, lr_eps), ylr=nx(by, lr_eps))
    if light:
        axs, atys = A @ xa, A.T @ ya
        if S > 0:
            axs, atys = S * axs, S * atys
            if pending:
                axs, atys = axs - w * ax, atys - w * aty
        v["axsum"], v["atysum"] = axs, atys
    return v


def averages(v, sc, light):
    """C1 (and the light sweeps): flushed sums and averages"""
    w, S, pend = sc["w_pending"], sc["sum_step"], sc["pending"]
    scale = 1.0 / S if S > 0.0 else 1.0
    out = {}
    for s_, cur in (("xsum", "x"), ("ysum", "y")) + ((("axsum", "ax"), ("atysum", "aty")) if light else ()):
        s = v[s_] + w * v[cur] if pend else v[s_].copy()
        out[s_] = s
        out[s_ + "_avg"] = s * scale
    return out


def pre_residuals(f, A, v, sc, light, sense, offset):
    """the residuals of the inputs from exact sums (products by scipy): what a case needs to place its memo"""
    av = averages(v, sc, light)
    xa, ya = av["xsum_avg"], av["ysum_avg"]
    axa, atya = (av["axsum_avg"], av["atysum_avg"]) if light else (A @ xa, A.T @ ya)
    ex, _ = sums_with_bounds(all_terms(f, v["x"], v["aty"], xa, atya, v["y"], v["ax"], ya, axa))
    return residuals_from_sums(ex, sense, offset)


def verify(f, v, sc, memo, got, sense, offset, light, measured):
    """every assertion of one case; returns the branch the reference took"""
    from test_gpu_hipdlp_kernels import check_spmv
    eq = lambda a, b, what: np.array_equal(a, b) or pytest.fail(f"{what}: {np.flatnonzero(a != b)[:5]} "
                                                                  f"{a[np.flatnonzero(a != b)[:3]]} vs {b[np.flatnonzero(a != b)[:3]]}")
    kept = False
    av = averages(v, sc, light)
    eq(got["xavg"], av["xsum_avg"], "xbar")
    eq(got["yavg"], av["ysum_avg"], "ybar")
    if light:
        eq(got["axavg"], av["axsum_avg"], "A xbar (light)")
        eq(got["atyavg"], av["atysum_avg"], "A'ybar (light)")
    else:
        check_spmv(got["axavg"], f["rbeg"].astype(np.int64), f["ridx"], f["rval"], got["xavg"], "A xbar")
        check_spmv(got["atyavg"], f["cbeg"].astype(np.int64), f["cidx"], f["cval"], got["yavg"], "A'ybar")
    terms = all_terms(f, v["x"], v["aty"], got["xavg"], got["atyavg"], v["y"], v["ax"], got["yavg"], got["axavg"])
    ex, bd = sums_with_bounds(terms)
    for q in range(28):
        assert abs(got["sums"][q] - ex[q]) <= bd[q], ("sum", q, got["sums"][q], ex[q], bd[q])
    # residuals: bit for bit from the device's sums, within the propagated bound of the exact ones
    R = residuals_from_sums([float(s) for s in got["sums"]], sense, offset)
    Rx = residuals_from_sums(ex, sense, offset)
    B = residual_bounds(ex, bd, Rx, offset)
    for t in range(2):
        for k, val in got["res"][t].items():
            assert val == R[t][k] or (math.isnan(val) and math.isnan(R[t][k])), ("residual", t, k, val, R[t][k])
            assert abs(val - Rx[t][k]) <= B[t][k], ("residual bound", t, k, val, Rx[t][k], B[t][k])
    # the verdict: the same from the device's and from the exact residuals, no comparison near its threshold
    mg = Margins()
    term, ti, choice, memo_after, branch = decide(R, sc, memo, mg)
    assert decide(Rx, sc, memo)[:3] == (term, ti, choice), ("exact residuals decide otherwise", branch)
    near = [(w, d) for w, d in mg.items if d < MARGIN]
    assert not near, ("deciding comparisons within MARGIN of their thresholds", near)
    assert (got["term"], got["term_iterate"], got["restart_choice"]) == (term, ti if term == 0 else 0, choice), \
        ("verdict", got["term"], got["term_iterate"], got["restart_choice"], term, ti, choice, branch)
    assert got["checks"] == 1 and got["trace_len"] == 1 and got["done"] == (1 if term >= 0 else 0)
    assert got["pending"] == 0
    trace = got["trace"]
    # vectors after the check
    new = dict(x=v["x"], y=v["y"], ax=v["ax"], aty=v["aty"], xsum=av["xsum"], ysum=av["ysum"], xlr=v["xlr"], ylr=v["ylr"])
    if light:
        new["axsum"], new["atysum"] = av["axsum"], av["atysum"]
    out = dict(beta=sc["beta"], tau=sc["tau"], sigma=sc["sigma"], sum_step=sc["sum_step"])
    if choice:
        if choice == 1:
            new.update(x=got["xavg"], y=got["yavg"], ax=got["axavg"], aty=got["atyavg"])
        for k in ("xsum", "ysum") + (("axsum", "atysum") if light else ()):
            new[k] = np.zeros_like(new[k])
        new["xlr"], new["ylr"] = new["x"], new["y"]
        d2 = []
        for cur, lr in (("x", "xlr"), ("y", "ylr")):
            d = new[cur] + -1.0 * v[lr]
            t = d * d
            s, e = exact_sum(t)
            lim = t.size * U / (1 - t.size * U) * float(np.sum(t.astype(np.longdouble))) * (1 + 2.0 ** -40) + e + 2 * U * s
            d2.append(s)
            assert abs(got["restart_sq"][len(d2) - 1] - s) <= lim, ("restart |d|^2", cur, got["restart_sq"], s, lim)
        upd, kept, bound = beta_update(sc["beta"], sc["tau"], sc["sigma"], *got["restart_sq"], sc["adaptive"])
        for k, rv in upd.items():
            lim = 0.0 if kept else ((bound if k == "beta" else bound + 8 * EPS) * abs(rv))
            assert abs(got[k] - rv) <= lim, ("step sizes", k, got[k], rv, lim, kept)
            if not kept:
                measured["beta_ulps"] = max(measured.get("beta_ulps", 0.0), abs(got[k] - rv) / (EPS * abs(rv)))
        out.update(upd)
        out["sum_step"] = 0.0
        Rc = R[1] if choice == 1 else R[0]
        memo_after.update(pf_lr=Rc["pfeas"], df_lr=Rc["dfeas"], gap_lr=Rc["gap"], last_restart_iter=sc["iter"])
        assert got["restarts"] == 1
    else:
        assert got["restarts"] == 0
        for k in ("beta", "tau", "sigma", "sum_step"):
            assert got[k] == sc[k], k
        assert all(math.isnan(got[k]) for k in ("eta", "tau_try", "sigma_try"))
    for k, val in new.items():
        eq(got[k], val, f"{k} after the check")
    for k in ("pf_lr", "df_lr", "gap_lr", "pf_lc", "df_lc", "gap_lc", "last_restart_iter"):
        assert got[k] == memo_after[k], ("memo", k, got[k], memo_after[k])
    # trace row, next check, power tables
    if term >= 0:
        Lr = R[0]
        assert got["stop_iter"] == sc["iter"] and np.isnan(got["pow_red"]).all() and np.isnan(got["pow_grow"]).all()
    else:
        Lr = R[1] if choice == 1 else R[0]
        assert got["stop_iter"] == next_check_iter(sc["iter"], sc["interval"], sc["iter_limit"]), got["stop_iter"]
        assert got["pow_base"] == sc["step_iter"]
        k = (sc["step_iter"] + 1 + np.arange(128)).astype(np.float64) + 1.0
        for name, e in (("pow_red", -0.3), ("pow_grow", -0.6)):
            ref = np.power(k, e)
            d = np.abs(got[name] - ref) / (EPS * ref)
            measured["pow_ulps"] = max(measured.get("pow_ulps", 0.0), float(d.max()))
            assert (d <= POW_ULPS).all(), (name, float(d.max()))
    A_ = R[1]
    want = [sc["iter"], Lr["pobj"], Lr["dobj"], Lr["pfeas"], Lr["dfeas"], A_["pobj"], A_["dobj"], A_["pfeas"], A_["dfeas"],
            got["tau"], got["sigma"], got["beta"], choice, sc["step_iter"], out["sum_step"], 0.0]
    assert np.array_equal(trace, np.array(want)), ("trace row", trace.tolist(), want)
    if choice and kept:
        return branch, True
    return branch, False


# ========================================================================================================== the cases
def scalars(**kw):
    sc = dict(iter=100, step_iter=117, adaptive=1, pending=0, beta=1.7, tau=0.31, sigma=0.52, sum_step=3.25, w_pending=0.4,
              tol_p=1e-6, tol_d=1e-6, tol_gap=1e-6, iter_limit=100000, interval=40, restart_on=1, time_flag=0, light=0)
    sc.update(kw)
    return sc


# (name, iterates (cur_eps, avg_eps), scalar changes, memo rule, expected branch); memo rule "lr k / lc q": the memo is k (q)
# times the candidate's residuals, so that mu_lr = k mu_cand (mu_lc = q mu_cand)
SPLIT_CASES = [
    ("opt_current", (0.0, 1e-2), dict(sum_step=0.0), None, "term0_current"),
    ("opt_average", (1e-1, 0.0), dict(pending=1), None, "term0_average"),
    ("time_flag", (1e-2, 1e-1), dict(time_flag=1), None, "term4_time"),
    ("iter_limit", (1e-2, 1e-1), dict(iter=399, iter_limit=400), None, "term4_iter_limit"),
    ("iter_limit_minus_2", (1e-2, 1e-1), dict(iter=398, iter_limit=400, restart_on=0, pending=1), None, "restart_off"),
    ("first_after_restart", (1e-2, 1e-1), dict(iter=80), dict(last=80, lr=3.0, lc=3.0), "first_after_restart"),
    ("artificial_exact", (1e-2, 1e-1), dict(iter=100, pending=1, adaptive=0), dict(last=64, lr=1.0, lc=1.0), "artificial_2"),
    ("artificial_avg", (1e-1, 1e-2), dict(iter=25), dict(last=16, lr=1.0, lc=1.0), "artificial_1"),
    ("sufficient_cur", (1e-3, 1e-1), dict(iter=120, pending=1), dict(last=100, lr=10.0, lc=1.0), "sufficient_2"),
    ("sufficient_avg", (1e-1, 1e-3), dict(iter=120, adaptive=0), dict(last=100, lr=10.0, lc=1.0), "sufficient_1"),
    ("necessary_cur", (1e-3, 1e-1), dict(iter=120), dict(last=100, lr=1.5, lc=0.5), "necessary_2"),
    ("necessary_avg", (1e-1, 1e-3), dict(iter=120, pending=1, adaptive=0), dict(last=100, lr=1.5, lc=0.5), "necessary_1"),
    ("no_progress", (1e-3, 1e-1), dict(iter=120), dict(last=100, lr=1.5, lc=2.0), "no_restart"),
    ("below_artificial", (1e-3, 1e-1), dict(iter=200, pending=1), dict(last=129, lr=1.0, lc=0.5), "no_restart"),
    ("beta_kept", (1e-3, 1e-1), dict(iter=120, xlr_equal=True), dict(last=100, lr=10.0, lc=1.0), "sufficient_2"),
    ("restart_off", (1e-3, 1e-1), dict(iter=120, restart_on=0), dict(last=100, lr=10.0, lc=1.0), "restart_off"),
]
LIGHT_CASES = [
    ("light_opt_current", (0.0, 1e-2), dict(iter=5, pending=1), None, "term0_current"),
    ("light_opt_average", (1e-1, 0.0), dict(iter=6), None, "term0_average"),
    ("light_iter_limit", (1e-2, 1e-1), dict(iter=9, iter_limit=10), None, "term4_iter_limit"),
    ("light_first", (1e-2, 1e-1), dict(iter=0, sum_step=0.0), dict(last=0, lr=2.0, lc=2.0), "first_after_restart"),
    ("light_artificial_cur", (1e-2, 1e-1), dict(iter=9, pending=1), dict(last=5, lr=1.0, lc=1.0), "artificial_2"),
    ("light_artificial_avg", (1e-1, 1e-2), dict(iter=9, pending=1, adaptive=0), dict(last=5, lr=1.0, lc=1.0), "artificial_1"),
    ("light_sufficient_avg", (1e-1, 1e-3), dict(iter=8, pending=1), dict(last=7, lr=10.0, lc=1.0), "sufficient_1"),
    ("light_no_progress", (1e-3, 1e-1), dict(iter=8, iter_limit=11), dict(last=7, lr=1.5, lc=2.0), "no_restart"),
]
BIG_CASES = ("opt_average", "iter_limit", "artificial_exact", "sufficient_avg", "necessary_cur", "below_artificial",
             "light_artificial_cur", "light_sufficient_avg")


def run_case(prob, f, A, base, case, rng, sense, offset, measured, base_is_ray=None):
    name, (ce, ae), ch, memo_rule, expect = case
    ch = dict(ch)
    light = name.startswith("light")
    xlr_equal = ch.pop("xlr_equal", False)
    sc = scalars(light=int(light), **ch)
    v = build_inputs(f, A, base, rng, ce, ae, sc["sum_step"], sc["pending"], sc["w_pending"], light, xlr_equal=xlr_equal)
    memo = dict(pf_lr=0.0, df_lr=0.0, gap_lr=0.0, pf_lc=0.0, df_lc=0.0, gap_lc=0.0, last_restart_iter=0)
    if memo_rule:
        R = pre_residuals(f, A, v, sc, light, sense, offset)
        L, Av = R
        C = L if score(sc["beta"], L["pfeas"], L["dfeas"], L["gap"]) < score(sc["beta"], Av["pfeas"], Av["dfeas"], Av["gap"]) else Av
        for k, rk in (("pf", "pfeas"), ("df", "dfeas"), ("gap", "gap")):
            memo[k + "_lr"] = memo_rule["lr"] * C[rk]
            memo[k + "_lc"] = memo_rule["lc"] * C[rk]
        memo["last_restart_iter"] = memo_rule["last"]
    kw = {k: v_ for k, v_ in sc.items()}
    kw.update(memo)
    got = prob.check_device(**{k: v[k] for k in ("x", "y", "ax", "aty", "xsum", "ysum", "xlr", "ylr")},
                            axsum=v.get("axsum"), atysum=v.get("atysum"), **kw)
    branch, kept = verify(f, v, sc, memo, got, sense, offset, light, measured)
    assert branch == expect, (name, branch, expect)
    hit = {branch, "light" if light else "split", f"pending{sc['pending']}", f"adaptive{sc['adaptive']}"}
    if sc["sum_step"] == 0.0:
        hit.add("sum_step0")
    if branch == "restart_off" and sc["iter"] == sc["iter_limit"] - 2:
        hit.add("go_on")
    if name.endswith("artificial_exact"):
        assert sc["iter"] - memo["last_restart_iter"] == 0.36 * sc["iter"]
        hit.add("artificial_exact")
    if kept:
        hit.add("beta_kept")
    return hit


def ray_case(prob, f, A, lp, x0, y0, ray, which, where, rng, measured):
    """a Farkas ray y (which = "primal") or a recession direction x (which = "dual") of size 1e14, in the current iterate or
    in the average; the other iterate is a perturbed planted point"""
    rs, cs = f["row_scale"], f["col_scale"]
    lam = 1e14
    sc = scalars(iter=160, pending=0, sum_step=2.0)
    bx, by = x0 * cs, y0 * rs
    xr, yr = bx + 1e-2 * rng.standard_normal(bx.size), by + 1e-2 * rng.standard_normal(by.size)
    if which == "primal":
        yr = lam * ray * rs
    else:
        xr = bx + lam * ray * cs
    xo, yo = bx + 1e-1 * rng.standard_normal(bx.size), by + 1e-1 * rng.standard_normal(by.size)
    (x, y), (xa, ya) = ((xr, yr), (xo, yo)) if where == "current" else ((xo, yo), (xr, yr))
    v = dict(x=x, y=y, ax=A @ x, aty=A.T @ y, xsum=2.0 * xa, ysum=2.0 * ya, xlr=x.copy(), ylr=y.copy())
    memo = dict(pf_lr=1.0, df_lr=1.0, gap_lr=1.0, pf_lc=1.0, df_lc=1.0, gap_lc=1.0, last_restart_iter=100)
    got = prob.check_device(**v, **sc, **memo)
    branch, _ = verify(f, v, sc, memo, got, lp.sense_, lp.offset_, False, measured)
    assert branch == f"term3_{which}", (which, where, branch)
    return {branch}


# shapes: (m, n, neq, sense, offset, cases); every grid reaches its cap and wraps somewhere, lengths odd and even
SHAPES = {
    "one_block": (200, 151, 60, -1, 2.5, "all"),
    "caps_160002x80001": (160_002, 80_001, 20_000, 1, -1.25, "all"),
    "tall_1300001x40000": (1_300_001, 40_000, 1_300_001, 1, 0.0, "big"),      # neq = m
    "wide_30000x1250001": (30_000, 1_250_001, 0, -1, 3.0, "big"),            # neq = 0
}


def _child_shape(name):
    from highs_b200 import engine
    from oracle import binding as ob
    m, n, neq, sense, offset, which = SHAPES[name]
    lp, x0, y0, _ = check_lp(m, n, neq, sense=sense, offset=offset, seed=len(name) + m % 97,
                             per_row=(1, 4) if max(m, n) > 1_000_000 else (1, 6))
    f = ob.formulate_and_scale(lp)
    assert (f["n"], f["m"], f["neq"]) == (n, m, neq) and np.array_equal(f["row_new_idx"], np.arange(m))
    A = _matrix(f)
    base = (x0 * f["col_scale"], y0 * f["row_scale"])
    cases = SPLIT_CASES + LIGHT_CASES
    if which == "big":
        cases = [c for c in cases if c[0] in BIG_CASES]
    out, hits, measured = {}, set(), {}
    prob = engine.Problem(lp, ordered_max=-1)
    try:
        assert (prob.n, prob.m) == (n, m)
        rng = np.random.default_rng(5)
        for case in cases:
            key = f"{name}#{case[0]}"
            try:
                hits |= run_case(prob, f, A, base, case, rng, sense, offset, measured)
                out[key] = "ok"
            except BaseException as e:   # noqa: BLE001  (pytest.fail raises a BaseException)
                out[key] = f"{type(e).__name__}: {e}"[:700]
    finally:
        prob.close()
    out["_hits"] = json.dumps(sorted(hits))
    out["_measured"] = json.dumps(measured)
    return out


RAY_LPS = {   # name: (m, n, neq, kind, sense, offset)
    "farkas_160002x80001": (160_002, 80_001, 5_000, "farkas", -1, 1.5),
    "recession_min": (30_000, 30_001, 2_000, "recession", 1, -2.0),
    "recession_max": (30_001, 30_000, 0, "recession", -1, 4.0),
}


def _child_rays():
    from highs_b200 import engine
    from oracle import binding as ob
    out, hits, measured = {}, set(), {}
    for name, (m, n, neq, kind, sense, offset) in RAY_LPS.items():
        lp, x0, y0, ray = check_lp(m, n, neq, kind=kind, sense=sense, offset=offset, seed=17)
        f = ob.formulate_and_scale(lp)
        assert np.array_equal(f["row_new_idx"], np.arange(m))
        A = _matrix(f)
        prob = engine.Problem(lp, ordered_max=-1)
        try:
            rng = np.random.default_rng(9)
            for where in ("current", "average"):
                key = f"{name}#{where}"
                try:
                    hits |= ray_case(prob, f, A, lp, x0, y0, ray, "primal" if kind == "farkas" else "dual", where, rng, measured)
                    out[key] = "ok"
                except BaseException as e:   # noqa: BLE001
                    out[key] = f"{type(e).__name__}: {e}"[:700]
        finally:
            prob.close()
    out["_hits"] = json.dumps(sorted(hits))
    out["_measured"] = json.dumps(measured)
    return out


def _child_rejections():
    """ordered problems, light checks past the dense phase: B200PDLP_ERR_ARG with nothing written"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    out = {}
    L = engine.lib()
    for name, lp, prm, sc in (("ordered", synthetic_lp(900, 700, 5, 2), {}, scalars(iter=5)),
                              ("light_past_dense", synthetic_lp(9000, 7000, 5, 2), dict(ordered_max=-1), scalars(iter=10, light=1)),
                              ("interval0", synthetic_lp(9000, 7000, 5, 2), dict(ordered_max=-1), scalars(interval=0))):
        prob = engine.Problem(lp, **prm)
        try:
            cin = engine.CCheckIn(**{k: v for k, v in sc.items() if hasattr(engine.CCheckIn, k)})
            vs = [np.full(max(prob.n, prob.m), 7.0) for _ in engine.CHECK_VECTORS]
            cout = engine.CCheckOut()
            engine.C.memset(engine.C.byref(cout), 0x5A, engine.C.sizeof(cout))
            before = bytes(cout)
            rc = L.b200pdlp_check_device(prob._h, engine.C.byref(cin), *(engine._p(v, engine._dp) for v in vs), engine.C.byref(cout))
            ok = rc == -1 and bytes(cout) == before and all((v == 7.0).all() for v in vs)
            out[name] = "ok" if ok else f"rc {rc}: {L.b200pdlp_last_error().decode()}"
        finally:
            prob.close()
    return out


def _child_e2e(env_name):
    """the ordered goldens that end INFEASIBLE_OR_UNBOUNDED, solved in tree mode (device checks, light or split as the
    environment says): the golden's model status.  The `unbounded` golden's status (10, Unbounded) is HiGHS's own verdict, which no
    PDLP term code maps to; there the status must be the one the oracle's PDLP verdict maps to (9)."""
    from conftest import golden_lp, load_golden, options_to_params, term_to_model_status
    from highs_b200 import engine
    from oracle import binding as ob
    out = {}
    for case in load_golden():
        if case["name"] not in ("infeasible", "unbounded", "woodinfe", "galenet") or case["tag"] not in ("kkt1e-4",):
            continue
        key = f"{env_name}#{case['name']}"
        try:
            prm = options_to_params(case["options"])
            lp = golden_lp(case)
            res = engine.solve(lp, ordered_max=-1, **prm)
            st = term_to_model_status(res["term_code"], res["iters"], prm.get("iter_limit", 2147483647))
            want = case["model_status_code"]
            if want == 10:
                ref = ob.solve(lp, **prm)
                want = term_to_model_status(ref["term_code"], ref["iters"], prm.get("iter_limit", 2147483647))
                assert want == 9, ref["term_name"]
            assert st == want, (st, want, res["term_name"], res["iters"])
            out[key] = "ok"
        except BaseException as e:   # noqa: BLE001
            out[key] = f"{type(e).__name__}: {e}"[:500]
    return out


def synthetic_verdict_lps():
    """tree-size LPs with a planted Farkas certificate / recession direction"""
    return {"farkas_30000": check_lp(30_000, 30_001, 3_000, kind="farkas", sense=1, offset=0.5, seed=41)[0],
            "recession_30000": check_lp(30_001, 30_000, 1_000, kind="recession", sense=-1, offset=1.0, seed=43)[0]}


def _child_synthetic(name):
    from highs_b200 import engine
    from oracle import binding as ob
    lp = synthetic_verdict_lps()[name]
    prm = dict(tol_primal=1e-4, tol_dual=1e-4, tol_gap=1e-4, iter_limit=40000)
    ref = ob.solve(lp, **prm)
    res = engine.solve(lp, ordered_max=-1, **prm)
    try:
        assert ref["term_code"] == 3, ("oracle", ref["term_name"], ref["iters"])
        assert res["term_code"] == ref["term_code"], (res["term_name"], ref["term_name"])
        assert ref["iters"] / 2 <= res["iters"] <= 2 * ref["iters"] + 1, (res["iters"], ref["iters"])
        r = "ok"
    except BaseException as e:   # noqa: BLE001
        r = f"{type(e).__name__}: {e}"[:500]
    return {name: r, "_iters": json.dumps(dict(engine=res["iters"], oracle=ref["iters"]))}


def child_main(case):
    kind, _, arg = case.partition(":")
    out = {"shape": _child_shape, "e2e": _child_e2e, "synthetic": _child_synthetic}[kind](arg) if arg else \
        {"rays": _child_rays, "rejections": _child_rejections}[kind]()
    print(json.dumps(out), flush=True)
    return 0


# ======================================================================================================== parent side
_HITS = set()


def _run_child(case, env=None, timeout=900):
    from test_gpu_spmv_shapes import _ENV
    e = {k: v for k, v in os.environ.items() if k not in _ENV + ("B200PDLP_TIMING", "B200PDLP_LIGHT_CHECK")}
    e.update(env or {})
    try:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "child", case], capture_output=True, text=True,
                           timeout=timeout, cwd=ROOT, env=e)
    except subprocess.TimeoutExpired:
        pytest.fail(f"child {case} did not finish in {timeout} s (killed)")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert lines and r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-3000:])
    out = json.loads(lines[-1])
    info = {k: v for k, v in out.items() if k.startswith("_")}
    if "_hits" in info:
        _HITS.update(json.loads(info["_hits"]))
    if info:
        print(case, info)
    return {k: v for k, v in out.items() if not k.startswith("_")}


def _assert_all_ok(out, at_least):
    bad = {k: v for k, v in out.items() if v != "ok"}
    assert len(out) >= at_least and not bad, (len(out), bad)


pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", list(SHAPES))
def test_check_device_shapes(shape):
    _assert_all_ok(_run_child(f"shape:{shape}"), len(BIG_CASES) if SHAPES[shape][5] == "big" else len(SPLIT_CASES))


def test_check_device_infeasibility_rays():
    _assert_all_ok(_run_child("rays"), 6)


def test_check_device_rejections():
    _assert_all_ok(_run_child("rejections"), 3)


def test_every_branch_was_hit():
    """every verdict and restart branch of BRANCHES was reached by the cases above (which run first, in file order; run
    alone, this test runs them itself)"""
    if not BRANCHES <= _HITS:
        for case in [f"shape:{s}" for s in SHAPES] + ["rays"]:
            _run_child(case)
    assert BRANCHES <= _HITS, sorted(BRANCHES - _HITS)


@pytest.mark.parametrize("env_name,env", [("device_checks", {}), ("split_only", {"B200PDLP_LIGHT_CHECK": "0"})],
                         ids=["device_checks-env0", "split_only-env2"])   # (the ids these two cases have always had)
def test_tree_mode_verdicts_of_the_goldens(env_name, env):
    _assert_all_ok(_run_child(f"e2e:{env_name}", env=env), 4)


@pytest.mark.parametrize("name", ["farkas_30000", "recession_30000"])
def test_tree_mode_verdicts_of_synthetic_lps(name):
    _assert_all_ok(_run_child(f"synthetic:{name}", timeout=1200), 1)


if __name__ == "__main__" and len(sys.argv) >= 3 and sys.argv[1] == "child":
    sys.exit(child_main(sys.argv[2]))
