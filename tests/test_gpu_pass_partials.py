"""The partial sums of a tree-mode PDHG pass, slot by slot, under every SpMV launch shape.

K1 (primal step), K2 (A x' + dual step) and K3 (A'y' + interaction) each write one partial sum per CTA into a slot array,
and step_rule_kernel (K4) adds the slots in a fixed order.  A row longer than 2048 entries is cut into segments of 2048, one
CTA and one slot each; the segment that takes the last ticket runs the row's epilogue.  Its term must land in the slot of the
row's FIRST segment, as 0.0 + term (so a zero term is +0.0), and every other segment slot must hold +0.0, whichever segment
finished last: otherwise K4's rounding, and with it the trajectory, changes from run to run.

b200pdlp_pass_partials (engine.Problem.pass_partials) runs K1-K4 once and returns the slot arrays, where each long row's slots
are and K4's sums.  For every shape the LP admits, forced through the environment and confirmed from the B200PDLP_TIMING=1
lines (one slice per warp, persistent with 1 and 2 CTAs per SM, each with zero-skip on and off, and tiled with a bulk copy
and with cooperative loads):
  * every long row's first slot is its term bit for bit (one IEEE operation on the returned vectors), the other slots +0.0;
  * K4's dx2, dy2 and inter equal a replay of step_rule_kernel's order over the returned slots, bit for bit;
  * the body slots add up to the body rows' terms within the bound of a sum of k terms;
  * a second launch on the same inputs returns the same bytes, and two 300-iteration solves return the same results.
"""
import math

import numpy as np
import pytest

from hipdlp_batch_child import INTS, SCALARS, VECTORS, _bits
from test_gpu_spmv_shapes import (ARMS, TILE_ROWS, _ENV, _SHAPE_RE, _planted_lp, _with_long_lines, assert_shape,
                                  assert_within_bound, sm_count)
from test_gpu_zero_skip import _ZS_RE

pytestmark = pytest.mark.gpu

SEG = 2048               # entries per segment of a long row (kNnzBlk)
LONG = 512               # rows longer than this are long rows
HUGE = 66_000            # more than 32 segments
STEP_THREADS = 1024      # step_rule_kernel's block

# arm -> (arm of test_gpu_spmv_shapes, B200PDLP_ZERO_SKIP)
SHAPES = {
    "warp": ("default", 0), "warp_zero_skip": ("default", 1),
    "persistent_k1": ("persistent_k1", 0), "persistent_k1_zero_skip": ("persistent_k1", 1),
    "persistent_k2": ("persistent_k2", 0), "persistent_k2_zero_skip": ("persistent_k2", 1),
    "tiled_bulk_copy": ("tiled_bulk_copy", 1), "tiled_cooperative_loads": ("tiled_cooperative_loads", 1),
}


def long_lines_lp(m=72 * TILE_ROWS - 6, n=72 * TILE_ROWS - 8, band=500, seed=21):
    """a banded LP (72 tiles of rows, so the tiled shape is admitted while a few windows miss) with long rows and long
    columns of 513, 2048, 2049, 4097, 5000 and HUGE entries, and 50 rows and 50 columns of 3 to 8 segments each, every long
    line contiguous around the diagonal.  Returns (lp, the column of length 4097)."""
    rng = np.random.default_rng(seed)
    fixed = [513, 2048, 2049, 4097, 5000, HUGE]
    rlens = fixed + rng.integers(2 * SEG + 1, 8 * SEG + 1, size=50).tolist()
    clens = fixed + rng.integers(2 * SEG + 1, 8 * SEG + 1, size=50).tolist()
    ri = (np.linspace(0.01, 0.99, len(rlens)) * m).astype(np.int64)
    ci = (np.linspace(0.015, 0.985, len(clens)) * n).astype(np.int64)
    lr = dict(zip(ri.tolist(), rng.permutation(rlens).tolist()))
    lc = dict(zip(ci.tolist(), rng.permutation(clens).tolist()))
    ln = rng.integers(0, 17, size=m)
    ln[list(lr)] = 0
    rows = np.repeat(np.arange(m), ln)
    cols = np.clip(rows * n // m + rng.integers(-band, band + 1, size=rows.size), 0, n - 1)
    free_c, free_r = np.setdiff1d(np.arange(n), list(lc)), np.setdiff1d(np.arange(m), list(lr))

    def around(free, centre, L):
        k = min(max(int(np.searchsorted(free, centre)) - L // 2, 0), free.size - L)
        return free[k:k + L]

    rows, cols = _with_long_lines(m, n, rows, cols, lr, lc, lambda i, L: around(free_c, i * n // m, L),
                                  lambda j, L: around(free_r, j * m // n, L))
    j4097 = next(j for j, L in lc.items() if L == 4097)
    return _planted_lp(m, n, rows, cols, rng, f"long_lines_{m}x{n}"), j4097


@pytest.fixture(scope="module")
def family():
    return long_lines_lp()


def create(engine, lp, arm, monkeypatch, capfd):
    """engine.Problem(lp) in tree mode under the arm's environment; asserts the SpMV shapes and zero-skip the engine took"""
    shape, zs = SHAPES[arm]
    for k in _ENV + ("B200PDLP_ZERO_SKIP",):
        monkeypatch.delenv(k, raising=False)
    for k, v in ARMS[shape][0].items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("B200PDLP_ZERO_SKIP", str(zs))
    monkeypatch.setenv("B200PDLP_TIMING", "1")
    capfd.readouterr()
    prob = engine.Problem(lp, ordered_max=-1)
    err = capfd.readouterr().err
    for k in _ENV + ("B200PDLP_ZERO_SKIP", "B200PDLP_TIMING"):
        monkeypatch.delenv(k, raising=False)
    found, zsk = _SHAPE_RE.findall(err), _ZS_RE.findall(err)
    try:
        assert found and zsk, f"{arm}: the engine printed no SpMV shape or zero-skip line"
        g = found[-1]
        shapes = {"A": (g[0], int(g[1]), int(g[2]), int(g[3])), "A'": (g[4], int(g[5]), int(g[6]), int(g[7]))}
        assert_shape(shape, shapes, {"A": prob.m, "A'": prob.n}, sm_count())
        a, at = (int(v) for v in zsk[-1])
        on = zs and ARMS[shape][1] != "tiled"
        assert (a > 0 and at > 0) if on else (a == 0 and at == 0), (arm, a, at)
    except BaseException:
        prob.close()
        raise
    return prob


# ---------------------------------------------------------------- references
def k4_sum(slots):
    """step_rule_kernel's sum of one slot array: thread t adds slots t, t + 1024, ... from +0.0, a __shfl_down tree (16, 8,
    4, 2, 1) in each warp, then warp 0 applies the same tree to the 32 warp sums"""
    s = np.zeros(STEP_THREADS)
    for i0 in range(0, slots.size, STEP_THREADS):
        c = slots[i0:i0 + STEP_THREADS]
        s[:c.size] = s[:c.size] + c

    def tree(v):   # lanes on the last axis; lane l reads lane l + o before anything changes
        v = v.copy()
        for o in (16, 8, 4, 2, 1):
            v[..., :32 - o] = v[..., :32 - o] + v[..., o:]
        return v[..., 0]
    return tree(tree(s.reshape(32, 32)))


def check_long_slots(slots, recs, terms, lengths, what):
    """each record (row, first, segments): slots[first] == 0.0 + term bit for bit, the other segment slots +0.0; the
    records tile the end of the slot array.  Returns the number of body slots."""
    assert recs.shape[0] == int((lengths > LONG).sum()), (what, "long rows", recs.shape[0])
    assert np.array_equal(np.sort(recs[:, 0]), np.flatnonzero(lengths > LONG)), (what, "long rows are not the rows > 512")
    assert np.array_equal(recs[:, 2], -(-lengths[recs[:, 0]] // SEG)), (what, "segment counts")
    order = np.argsort(recs[:, 1])
    first, nseg = recs[order, 1], recs[order, 2]
    nb = slots.size - int(nseg.sum())
    assert first[0] == nb and np.array_equal(first[1:], first[:-1] + nseg[:-1]), (what, "segment slots are not contiguous")
    bad = []
    for r, f, s in recs:
        seg = _bits(slots[f:f + s])
        want = _bits(np.float64(terms[r]) + 0.0)
        if seg[0] != want or (seg[1:] != 0).any():
            held = np.flatnonzero(seg != 0).tolist()
            bad.append(f"row {r} ({s} segments): term {terms[r]!r} expected in segment 0, nonzero segments {held}")
    assert not bad, (what, f"{len(bad)} of {len(recs)} long rows have their term outside the first slot", bad[:8])
    return nb


def check_body(slots, nb, terms, body, what):
    """the body slots add up to the body rows' terms within gamma_k sum |term| (k = number of terms)"""
    t = terms[body]
    got = np.array([math.fsum(slots[:nb])])
    assert_within_bound(got, np.array([0, t.size]), np.arange(t.size), t, np.ones(t.size), what)


def pass_inputs(prob, j0, seed=3):
    """x >= 0 with many exact zeros; column j0 at its lower bound 0 with aty[j0] = -1e6, so that x'[j0] = 0 and its
    interaction term (x - x')(aty - aty') is -0.0"""
    rng = np.random.default_rng(seed)
    n, m = prob.n, prob.m
    x = np.where(rng.random(n) < 0.5, 0.0, rng.random(n))
    y, ax, aty = rng.standard_normal(m), rng.standard_normal(m), rng.standard_normal(n)
    x[j0], aty[j0] = 0.0, -1e6
    return x, y, ax, aty


# ---------------------------------------------------------------- the tests
@pytest.mark.parametrize("arm", list(SHAPES))
def test_pass_partials(engine_lib, monkeypatch, capfd, family, arm):
    """K2's and K3's long-row slots, K4's sums and the body sums of one pass, and a repeat launch"""
    from highs_b200 import engine
    lp, j0 = family
    prob = create(engine, lp, arm, monkeypatch, capfd)
    try:
        assert (prob.m, prob.n) == (lp.num_row_, lp.num_col_)   # the standard form is A itself
        x, y, ax, aty = pass_inputs(prob, j0)
        tau, sigma = 0.37, 0.61
        r = prob.pass_partials(x, y, ax, aty, tau, sigma)
        again = prob.pass_partials(x, y, ax, aty, tau, sigma)
    finally:
        prob.close()
    rlen = np.bincount(lp.a_matrix_.index_, minlength=lp.num_row_)
    clen = np.diff(lp.a_matrix_.start_).astype(np.int64)
    assert (rlen > 32 * SEG).any() and (clen > 32 * SEG).any() and clen[j0] == 4097
    for L in (2048, 2049, 4097, 5000):
        assert L in rlen.tolist() and L in clen.tolist()
    assert ((rlen > 2 * SEG) & (rlen <= 8 * SEG)).sum() >= 50 and ((clen > 2 * SEG) & (clen <= 8 * SEG)).sum() >= 50

    dx, d = x - r["x_new"], y - r["y_new"]
    dy_terms, dx_terms = d * d, dx * dx
    inter_terms = dx * (aty - r["aty_new"])
    assert r["x_new"][j0] == 0.0 and np.signbit(inter_terms[j0]), "the zero-movement column's term is not -0.0"
    nb2 = check_long_slots(r["k2"], r["long_a"], dy_terms, rlen, (arm, "K2 |dy|^2"))
    nb3 = check_long_slots(r["k3"], r["long_at"], inter_terms, clen, (arm, "K3 interaction"))

    # K4, bit for bit
    for k, key in (("k1", "dx2"), ("k2", "dy2"), ("k3", "inter")):
        assert _bits(k4_sum(r[k])) == _bits(r[key]), (arm, key, r[key], k4_sum(r[k]))

    # the body slots against the extended-precision sum of the body rows' terms
    check_body(r["k1"], r["k1"].size, dx_terms, np.arange(prob.n), (arm, "K1 |dx|^2"))
    check_body(r["k2"], nb2, dy_terms, rlen <= LONG, (arm, "K2 body"))
    check_body(r["k3"], nb3, inter_terms, clen <= LONG, (arm, "K3 body"))

    # a second launch on the same inputs: the same bytes
    for k, v in r.items():
        if isinstance(v, np.ndarray):
            assert v.shape == again[k].shape and v.tobytes() == again[k].tobytes(), (arm, k, "differs between two launches")
        else:
            assert _bits(v) == _bits(again[k]), (arm, k, v, again[k])


@pytest.mark.parametrize("arm", list(SHAPES))
def test_solve_repeats(engine_lib, monkeypatch, capfd, family, arm):
    """two 300-iteration solves of the LP with multi-segment long rows and columns return the same bytes"""
    from highs_b200 import engine
    lp, _ = family
    prob = create(engine, lp, arm, monkeypatch, capfd)
    try:
        a = prob.solve(iter_limit=300, trace_cap=64)
        b = prob.solve(iter_limit=300, trace_cap=64)
    finally:
        prob.close()
    for k in INTS:
        assert a[k] == b[k], (arm, k, a[k], b[k])
    for k in SCALARS:
        assert _bits(a[k]) == _bits(b[k]), (arm, k, a[k], b[k])
    for k in VECTORS:
        assert np.array_equal(_bits(a[k]), _bits(b[k])), (arm, k)
    assert a["trace"].shape == b["trace"].shape and len(a["trace"]) >= 2, (arm, a["trace"].shape, b["trace"].shape)
    assert np.array_equal(_bits(a["trace"]), _bits(b["trace"])), (arm, "trace")
