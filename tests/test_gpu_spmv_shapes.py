"""Every launch shape of the hot-path SpMV against an extended-precision reference.

The engine picks one of four shapes per matrix (engine.cu apply_spmv_grid): one slice per warp, the persistent
software-pipelined walk (spmv_sell_kernel<Epi, true>), and the tiled kernel with the input window staged by a bulk copy
(B200PDLP_TILE=1) or by cooperative loads (=2).  Each arm below forces one shape through the environment, and asserts from
the `SpMV shapes:` line that B200PDLP_TIMING=1 prints that this shape, and no other, was chosen.

Every element of A x and A'y must satisfy the a-priori bound of a floating-point dot product of length k,
|got - ref| <= gamma_k sum_j |a_ij x_j| with gamma_k = k u / (1 - k u), u = 2^-53, whatever the summation order.  A dropped,
zeroed or repeated term misses it by many orders of magnitude.  Rows of ordinary length (<= 512 entries) are summed one entry
at a time in storage order by every shape, so they must also equal that sequential sum bit for bit.  Long rows (> 512) are
cut into 2048-entry segments: the same 256-thread code in the default and the persistent shape (bit-identical there), 1024
threads in the tiled one (the bound only).
"""
import math
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
LONG = 512             # rows longer than this are long rows (host_prep.cpp build_layout)
TILE_ROWS = 8192       # rows per tile of the tiled shape (kTileSlices slices of 32)
ROWS_PER_CTA = 256     # one-slice-per-warp shape: 8 slices of 32 rows per CTA
REL_TRACE = 1e-6       # trajectories under different shapes: the block partial sums are grouped differently
# The ragged LP's trajectory amplifies rounding quickly: on an H100, two persistent grids (1 and 2 CTAs per SM, the same kernel,
# only the grouping of the partial sums differs) agree to 7e-14 at iteration 40 and to 9e-6 at iteration 79.  Its trace is
# compared up to iteration 40.
TRACE_UNTIL = {"ragged": 40}

_ENV = ("B200PDLP_TILE", "B200PDLP_TILE_A", "B200PDLP_TILE_AT", "B200PDLP_TILE_FORCE", "B200PDLP_SPMV_CTAS_PER_SM",
        "B200PDLP_SPMV_A_CTAS_PER_SM", "B200PDLP_SPMV_AT_CTAS_PER_SM")

# arm -> (environment, shape the engine must report, CTAs per SM of the persistent grid)
ARMS = {
    "default": ({"B200PDLP_TILE": "0", "B200PDLP_SPMV_A_CTAS_PER_SM": "0", "B200PDLP_SPMV_AT_CTAS_PER_SM": "0"},
                "one slice per warp", 0),
    "persistent_k1": ({"B200PDLP_TILE": "0", "B200PDLP_SPMV_A_CTAS_PER_SM": "1", "B200PDLP_SPMV_AT_CTAS_PER_SM": "1"},
                      "persistent", 1),
    "persistent_k2": ({"B200PDLP_TILE": "0", "B200PDLP_SPMV_A_CTAS_PER_SM": "2", "B200PDLP_SPMV_AT_CTAS_PER_SM": "2"},
                      "persistent", 2),
    "tiled_bulk_copy": ({"B200PDLP_TILE": "1", "B200PDLP_TILE_FORCE": "1", "B200PDLP_SPMV_A_CTAS_PER_SM": "0",
                         "B200PDLP_SPMV_AT_CTAS_PER_SM": "0"}, "tiled", 0),
    "tiled_cooperative_loads": ({"B200PDLP_TILE": "2", "B200PDLP_TILE_FORCE": "1", "B200PDLP_SPMV_A_CTAS_PER_SM": "0",
                                 "B200PDLP_SPMV_AT_CTAS_PER_SM": "0"}, "tiled", 0),
}
PASS_SHAPES = ("default", "persistent_k1", "persistent_k2", "tiled_bulk_copy", "tiled_cooperative_loads")

_SHAPE_RE = re.compile(r"SpMV shapes: A (.+?) \((\d+) CTAs, tiles staged (\d+)/(\d+)\)\s+A' (.+?) \((\d+) CTAs, "
                       r"tiles staged (\d+)/(\d+)\)")


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def forced_problem(engine, lp, arm, monkeypatch, capfd):
    """engine.Problem(lp) under the arm's environment; returns (problem, {"A": (shape, ctas, staged, tiles), "A'": ...})"""
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in ARMS[arm][0].items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("B200PDLP_TIMING", "1")
    capfd.readouterr()
    prob = engine.Problem(lp, ordered_max=-1)
    found = _SHAPE_RE.findall(capfd.readouterr().err)
    for k in _ENV + ("B200PDLP_TIMING",):
        monkeypatch.delenv(k, raising=False)
    assert found, f"{arm}: the engine printed no SpMV shape line"
    g = found[-1]
    return prob, {"A": (g[0], int(g[1]), int(g[2]), int(g[3])), "A'": (g[4], int(g[5]), int(g[6]), int(g[7]))}


def assert_shape(arm, shapes, rows, sms):
    """the intended shape was chosen for both matrices; rows = {"A": rows of A, "A'": rows of A'}"""
    want, k = ARMS[arm][1], ARMS[arm][2]
    for which, (shape, ctas, staged, tiles) in shapes.items():
        body = -(-rows[which] // ROWS_PER_CTA)
        assert shape == want, (arm, which, shapes[which])
        if want == "one slice per warp":
            assert ctas == body, (arm, which, ctas, body)
        elif want == "persistent":
            assert body > sms * k, f"{which} has {body} body CTAs: too few for a persistent grid of {k} per SM"
            assert ctas == sms * k, (arm, which, ctas)
        else:
            assert ctas == tiles == -(-rows[which] // TILE_ROWS), (arm, which, shapes[which])


# ---------------------------------------------------------------- matrix families (numpy only, deterministic)
def _planted_lp(m, n, rows, cols, rng, name):
    """min c.x  s.t.  A x >= b, x >= 0 with the pattern (rows, cols) (duplicates merged) and a planted optimal pair, as
    highs_b200.lp.synthetic_lp builds it: the standard form is A itself"""
    from highs_b200.lp import HighsLp, HighsSparseMatrix, kHighsInf
    key = np.unique(np.asarray(cols, np.int64) * m + np.asarray(rows, np.int64))   # column-major order
    c, r = key // m, key % m
    val = rng.standard_normal(key.size)
    start = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(c, minlength=n), out=start[1:])
    xs = np.where(rng.random(n) < 0.5, 0.0, rng.random(n))
    ys = np.where(rng.random(m) < 0.5, 0.0, rng.random(m))
    b = np.bincount(r, weights=val * xs[c], minlength=m) - np.where(ys > 0, 0.0, rng.random(m))
    cost = np.bincount(c, weights=val * ys[r], minlength=n) + np.where(xs > 0, 0.0, rng.random(n))
    return HighsLp(n, m, cost, np.zeros(n), np.full(n, kHighsInf), b, np.full(m, kHighsInf),
                   HighsSparseMatrix(n, m, start.astype(np.int32), r.astype(np.int32), val), 1, 0.0, name)


def _with_long_lines(m, n, rows, cols, long_rows, long_cols, row_cols, col_rows):
    """replace every entry of the rows `long_rows` / columns `long_cols` ({index: length}) by exactly that many entries:
    row_cols(i, L) gives row i's columns, col_rows(j, L) column j's rows (both avoid the other kind of long line)"""
    drop = np.isin(rows, list(long_rows)) | np.isin(cols, list(long_cols))
    rows, cols = [rows[~drop]], [cols[~drop]]
    for i, L in long_rows.items():
        c = row_cols(i, L)
        assert c.size == L and np.unique(c).size == L and not np.isin(c, list(long_cols)).any()
        rows.append(np.full(L, i)); cols.append(c)
    for j, L in long_cols.items():
        r = col_rows(j, L)
        assert r.size == L and np.unique(r).size == L and not np.isin(r, list(long_rows)).any()
        rows.append(r); cols.append(np.full(L, j))
    return np.concatenate(rows), np.concatenate(cols)


def _long_lines(m, n):
    # 512: the longest ordinary row; 513: long, one segment; 5000: long, three 2048-entry segments
    return ({int(0.2 * m): 5000, int(0.3 * m): 513, int(0.4 * m): 512},
            {int(0.6 * n): 5000, int(0.7 * n): 513, int(0.8 * n): 512})


def ragged_lp(m, n, seed=11):
    """random columns; rows of every length 0..40, columns of lengths around 0..40 (every 41st column empty), a long row and
    a long column of each kind"""
    rng = np.random.default_rng(seed)
    lr, lc = _long_lines(m, n)
    ln = rng.permutation(np.arange(m) % 41)
    ln[list(lr)] = 0
    w = (np.arange(n) % 41).astype(np.float64)
    w[list(lc)] = 0.0
    rows = np.repeat(np.arange(m), ln)
    cols = rng.choice(n, size=rows.size, p=w / w.sum())
    free_c = np.setdiff1d(np.arange(n), list(lc))
    free_r = np.setdiff1d(np.arange(m), list(lr))
    rows, cols = _with_long_lines(m, n, rows, cols, lr, lc, lambda i, L: rng.choice(free_c, L, replace=False),
                                  lambda j, L: rng.choice(free_r, L, replace=False))
    return _planted_lp(m, n, rows, cols, rng, f"ragged_{m}x{n}")


def banded_lp(m, n, band=1000, seed=12, wrap=False):
    """row i holds 0..40 entries within `band` of the diagonal column i n / m, plus a long row and a long column of each
    kind (contiguous around the diagonal).  wrap: one row also touches column 0 and column n - 1"""
    rng = np.random.default_rng(seed)
    lr, lc = _long_lines(m, n)
    ln = rng.permutation(np.arange(m) % 41)
    rows = np.repeat(np.arange(m), ln)
    cols = np.clip(rows * n // m + rng.integers(-band, band + 1, size=rows.size), 0, n - 1)
    rows, cols = _with_long_lines(m, n, rows, cols, lr, lc, lambda i, L: i * n // m - L // 2 + np.arange(L),
                                  lambda j, L: j * m // n - L // 2 + np.arange(L))
    if wrap:
        r = m // 2 + 13
        rows, cols = np.concatenate([rows, [r, r]]), np.concatenate([cols, [0, n - 1]])
    return _planted_lp(m, n, rows, cols, rng, f"banded_{m}x{n}" + ("_wrap" if wrap else ""))


def _family(name, sms):
    from highs_b200.lp import synthetic_lp
    big = 2 * ROWS_PER_CTA * sms * 2 + 999          # twice the rows a persistent grid of 2 CTAs per SM covers in one sweep
    if name == "ragged":
        return ragged_lp(big, big - 1234)
    if name == "random":
        return synthetic_lp(big + 1, big - 321, 8, seed=31)
    # about 24 tiles (8192 rows each): one or two tiles that cannot be staged leave >= 90 %, so the tiled shape is kept
    if name == "banded_staged":
        return banded_lp(24 * TILE_ROWS - 6, 24 * TILE_ROWS - 8)          # even n: the last window fits as well
    if name == "banded_mixed":
        # the wrap-around row's tile of A and the first and last tile of A' are too wide; odd n: A's last window falls back
        return banded_lp(24 * TILE_ROWS - 6, 24 * TILE_ROWS - 5, wrap=True)
    if name == "banded_synthetic":
        return synthetic_lp(60000, 50000, 7, seed=5, band=1500)          # 8 tiles, all staged; clipping makes long rows
    raise KeyError(name)


FAMILIES = {
    "ragged": ("default", "persistent_k1", "persistent_k2"),   # random patterns: no window fits, the tiled shape is never chosen
    "random": ("default", "persistent_k1", "persistent_k2"),
    "banded_staged": tuple(ARMS),
    "banded_mixed": tuple(ARMS),
    "banded_synthetic": ("default", "tiled_bulk_copy", "tiled_cooperative_loads"),   # (too few rows for a persistent grid)
}


# ---------------------------------------------------------------- references
def sequential_rows(beg, idx, val, x):
    """each row's sum added one entry at a time in storage order, from 0.0 (what every shape does for an ordinary row)"""
    ln = np.diff(beg)
    s = np.zeros(len(ln))
    live = np.arange(len(ln))
    for k in range(int(ln.max(initial=0))):
        live = live[ln[live] > k]
        p = beg[live] + k
        s[live] = s[live] + val[p] * x[idx[p]]
    return s


def _split(v):
    t = v * 134217729.0   # 2^27 + 1 (Dekker)
    hi = t - (t - v)
    return hi, v - hi


def _two_product(a, b):
    """p + e == a b exactly (Dekker's TwoProduct, no FMA)"""
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def extended_rows(beg, idx, val, x):
    """(ref, err): each row's exact sum within err, as extended precision numbers -- np.longdouble where it is wider than
    double, else TwoProduct terms added by math.fsum"""
    ld = np.longdouble
    ln = np.diff(beg)
    nz = np.flatnonzero(ln > 0)
    if np.finfo(ld).nmant >= 63:
        prod = val.astype(ld) * x[idx].astype(ld)
        ref = np.zeros(len(ln), ld)
        ref[nz] = np.add.reduceat(prod, beg[:-1][nz])
        mag = np.zeros(len(ln), ld)
        mag[nz] = np.add.reduceat(np.abs(prod), beg[:-1][nz])
        ul = ld(np.finfo(ld).eps) / 2
        kk = ln.astype(ld) + 1
        return ref, kk * ul / (1 - kk * ul) * mag
    p, e = _two_product(val, x[idx])
    ref = np.array([math.fsum(np.concatenate([p[beg[i]:beg[i + 1]], e[beg[i]:beg[i + 1]]])) for i in range(len(ln))])
    return ref.astype(ld), np.abs(ref).astype(ld) * U


def row_bounds(beg, idx, val, x):
    """(ref, bound): each row's extended-precision sum, and gamma_k sum |a_ij x_j| (k = its length) plus the reference's
    own error"""
    ld = np.longdouble
    ref, err = extended_rows(beg, idx, val, x)
    ln = np.diff(beg)
    mag = np.zeros(len(ln), ld)
    nz = np.flatnonzero(ln > 0)
    mag[nz] = np.add.reduceat(np.abs(val.astype(ld) * x[idx].astype(ld)), beg[:-1][nz])
    k = ln.astype(ld)
    return ref, k * ld(U) / (1 - k * ld(U)) * mag * (1 + ld(2.0 ** -40)) + err


def assert_within_bound(got, beg, idx, val, x, what, bounds=None):
    """|got - ref| <= gamma_k sum |a_ij x_j| for every row, k = its length (plus the reference's own error); bounds: the
    rows' (ref, bound) from row_bounds, when the caller has them"""
    ld = np.longdouble
    ref, bound = row_bounds(beg, idx, val, x) if bounds is None else bounds
    ln = np.diff(beg)
    dev = np.abs(got.astype(ld) - ref)
    bad = np.flatnonzero(dev > bound)
    assert bad.size == 0, (what, f"{bad.size} rows outside the bound, e.g. row {bad[0]} (length {ln[bad[0]]}): "
                                 f"got {got[bad[0]]!r}, ref {float(ref[bad[0]])!r}, bound {float(bound[bad[0]])!r}")


def assert_ordinary_rows_exact(got, seq, ln, what):
    ok = ln <= LONG
    bad = np.flatnonzero(ok & (got != seq))
    assert bad.size == 0, (what, f"{bad.size} ordinary rows differ from the sequential sum, e.g. row {bad[0]} "
                                 f"(length {ln[bad[0]]}): {got[bad[0]]!r} vs {seq[bad[0]]!r}")


# ---------------------------------------------------------------- the test
@pytest.mark.parametrize("family", list(FAMILIES))
def test_spmv_shapes(engine_lib, oracle, monkeypatch, capfd, family):
    """A x, A'y, the fused K2 (DualEpilogue) and 80-iteration trajectories under every shape the family admits"""
    from highs_b200 import engine
    sms = sm_count()
    lp = _family(family, sms)
    f = oracle.formulate_and_scale(lp)
    m, n, neq = f["m"], f["n"], f["neq"]
    assert (m, n) == (lp.num_row_, lp.num_col_)
    rbeg, ridx, rval = f["rbeg"].astype(np.int64), f["ridx"], f["rval"]
    cbeg, cidx, cval = f["cbeg"].astype(np.int64), f["cidx"], f["cval"]
    rlen, clen = np.diff(rbeg), np.diff(cbeg)
    if family in ("ragged", "banded_staged", "banded_mixed"):
        assert m % 32 and n % 32
        assert set(range(41)) <= set(rlen.tolist())
        for L in (512, 513, 5000):
            assert L in rlen.tolist() and L in clen.tolist()
    if family == "ragged":
        assert (clen == 0).any()
    rng = np.random.default_rng(7)
    x, y = rng.standard_normal(n), rng.standard_normal(m)
    ax_in, sigma = rng.standard_normal(m), 0.81
    ax_seq, aty_seq = sequential_rows(rbeg, ridx, rval, x), sequential_rows(cbeg, cidx, cval, y)
    w0 = y + sigma * f["rhs"]

    got = {}
    for arm in FAMILIES[family]:
        prob, shapes = forced_problem(engine, lp, arm, monkeypatch, capfd)
        try:
            assert_shape(arm, shapes, {"A": m, "A'": n}, sms)
            ax, aty = prob.spmv_ax(x), prob.spmv_aty(y)
            yn, axn, dy2 = prob.dual_step(x, y, ax_in, sigma)
            res = prob.solve(iter_limit=80, trace_cap=64)
        finally:
            prob.close()
        got[arm] = dict(shapes=shapes, ax=ax, aty=aty, yn=yn, axn=axn, dy2=dy2, res=res)
        # the reference: every element within the bound, ordinary rows bit for bit
        assert_within_bound(ax, rbeg, ridx, rval, x, (arm, "A x"))
        assert_within_bound(aty, cbeg, cidx, cval, y, (arm, "A'y"))
        assert_ordinary_rows_exact(ax, ax_seq, rlen, (arm, "A x"))
        assert_ordinary_rows_exact(aty, aty_seq, clen, (arm, "A'y"))
        # K2 = A x_new in the DualEpilogue and y_new = proj(y + sigma (b - 2 A x_new + A x)) (cupdlp_step.c:44-69)
        assert_within_bound(axn, rbeg, ridx, rval, x, (arm, "K2 A x"))
        assert_ordinary_rows_exact(axn, ax_seq, rlen, (arm, "K2 A x"))
        w = w0 + (-2.0 * sigma) * axn
        w = w + sigma * ax_in
        w[neq:] = np.maximum(w[neq:], 0.0)
        assert np.array_equal(yn, w), (arm, np.flatnonzero(yn != w)[:5])
        dy_ref = math.fsum((y - w) ** 2)
        assert abs(dy2 - dy_ref) <= 1e-12 * (1 + dy_ref), (arm, dy2, dy_ref)

    # agreement between shapes
    base = got["default"]
    long_a, long_at = rlen > LONG, clen > LONG
    for arm, g in got.items():
        for k, lng in (("ax", long_a), ("aty", long_at), ("axn", long_a)):
            u, v = base[k], g[k]
            if ARMS[arm][1] == "tiled":   # long rows: 1024-thread segment sums instead of 256-thread ones
                u, v = u[~lng], v[~lng]
            assert np.array_equal(u, v), (arm, k, np.flatnonzero(u != v)[:5])
        # the staged-tile counts do not depend on the shape
        assert [s[2:] for s in g["shapes"].values()] == [s[2:] for s in base["shapes"].values()], arm
        r0, r1 = base["res"], g["res"]
        assert r0["iters"] == r1["iters"] and r0["term_code"] == r1["term_code"], (arm, r0["iters"], r1["iters"])
        t0, t1 = r0["trace"], r1["trace"]
        assert len(t0) == len(t1) >= 2 and np.array_equal(t0[:, 0], t1[:, 0]), arm
        keep = t0[:, 0] <= TRACE_UNTIL.get(family, np.inf)
        scale = 1.0 + np.abs(t0[:, 1:9]).max(axis=0)
        dev = np.abs(t0[keep, 1:9] - t1[keep, 1:9])
        assert (dev <= REL_TRACE * scale).all(), (arm, dev.max(axis=0))
        if family not in TRACE_UNTIL:
            for k in ("col_value", "row_dual"):
                assert np.abs(r0[k] - r1[k]).max() <= 1e-5 * (1 + np.abs(r0[k]).max()), (arm, k)

    # which tiles were staged: every one, or (wrap-around row, odd n) a few but >= 90 % so that the tiled shape is kept
    staged = {w: base["shapes"][w][2:] for w in ("A", "A'")}
    if family in ("banded_staged", "banded_synthetic"):
        assert all(k == t > 0 for k, t in staged.values()), staged
    if family == "banded_mixed":
        # (A' keeps every tile: the columns 0 and n - 1 are long rows of A', which the tile windows leave out)
        assert 9 * staged["A"][1] <= 10 * staged["A"][0] < 10 * staged["A"][1], staged
        assert 9 * staged["A'"][1] <= 10 * staged["A'"][0] <= 10 * staged["A'"][1], staged
