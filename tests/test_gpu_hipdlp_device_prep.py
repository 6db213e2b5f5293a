"""The HiPDLP mode's device-resident prologue, initial point and postsolve (device_prep.cu, DevicePrologue::hipdlp) against
the host path it replaces (host_prep_hipdlp.cpp + the host boundary steps of engine_hipdlp.cu solve_hipdlp_on_device).

1. Prologue parity: b200pdlp_debug_prep_compare_hipdlp reports no mismatch in any array -- the scaled standard form, the row
   upper bounds, both orderings and layouts, the row-major copy of the caller's matrix, and both unscaled norms bit for bit --
   on every instance fixture under five scaling options, and on synthetic LPs that reach the special cases: a large LP, a
   column of 15 000 entries (long rows in A'), columns stored with shuffled rows, and every row class (EQ, LEQ, GEQ, ranged,
   free, and a row bound of 1e25, which is finite for HiPDLP).
2. Solve parity: the default (device prologue) and device_prep=-1 (host prologue) return the same iteration count,
   termination and the four solution vectors byte for byte, both iteration-limited (the zero solution) and converged.
3. Every SpMV launch shape (one slice per warp, persistent, tiled by bulk copy, tiled by cooperative loads), forced through the
   environment and read back from the `SpMV shapes:` line, gives the host path's bits -- except rows longer than 512 entries
   under the tiled shape, whose segments that kernel groups differently (tests/test_gpu_spmv_shapes.py): there 1e-12.

The GPU work runs in child processes (this file with `child <case>`): a faulting kernel must not poison the test session.
"""
import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

_SHAPE_ENV = ("B200PDLP_TILE", "B200PDLP_TILE_A", "B200PDLP_TILE_AT", "B200PDLP_TILE_FORCE", "B200PDLP_SPMV_CTAS_PER_SM",
              "B200PDLP_SPMV_A_CTAS_PER_SM", "B200PDLP_SPMV_AT_CTAS_PER_SM", "B200PDLP_DEVICE_PREP", "B200PDLP_TIMING")
# arm -> (environment, shape the engine must report for A and A')
SHAPES = {
    "one_slice_per_warp": ({"B200PDLP_TILE": "0", "B200PDLP_SPMV_CTAS_PER_SM": "0"}, "one slice per warp"),
    "persistent": ({"B200PDLP_TILE": "0", "B200PDLP_SPMV_CTAS_PER_SM": "1"}, "persistent"),
    "tiled_bulk_copy": ({"B200PDLP_TILE": "1", "B200PDLP_TILE_FORCE": "1"}, "tiled"),
    "tiled_cooperative_loads": ({"B200PDLP_TILE": "2", "B200PDLP_TILE_FORCE": "1"}, "tiled"),
}
_SHAPE_RE = re.compile(r"SpMV shapes: A (.+?) \((\d+) CTAs, tiles staged (\d+)/(\d+)\)\s+A' (.+?) \((\d+) CTAs, "
                       r"tiles staged (\d+)/(\d+)\)")
VECS = ("col_value", "col_dual", "row_value", "row_dual")
SCALINGS = [(5, 10), (7, 3), (0, 10), (2, 10), (4, 10)]   # (scaling_mode, ruiz_iterations)


# ----------------------------------------------------------------------------------------------------------- LP families
def mixed_rows_lp(m=6000, n=5000, seed=7):
    """Every row class: EQ, LEQ, GEQ, ranged, free, and GEQ with an upper bound of 1e25 (finite for HiPDLP, infinite for
    cuPDLP); boxed, free-below and fixed columns; maximised with an offset.  Feasible at a planted x* in [0, 1]."""
    from highs_b200.lp import HighsLp, HighsSparseMatrix, kHighsInf, synthetic_lp
    base = synthetic_lp(m, n, 6, seed)
    rng = np.random.default_rng(seed)
    A = base.a_matrix_.to_scipy()
    xs = rng.random(n)
    ax = A @ xs
    cls = np.arange(m) % 6
    lo = np.where(cls == 1, -kHighsInf, ax - np.where(cls == 2, rng.random(m), 0.0))
    lo = np.where(cls == 3, ax - 1.0, lo)
    lo = np.where(cls == 4, -kHighsInf, lo)
    up = np.where(cls == 0, ax, kHighsInf)
    up = np.where(cls == 1, ax + rng.random(m), up)
    up = np.where(cls == 3, ax + 1.0, up)
    up = np.where(cls == 5, 1e25, up)
    cl = np.zeros(n)
    cu = np.full(n, 10.0)
    cl[1::7] = -5.0
    cl[3::11] = cu[3::11] = xs[3::11]
    cost = rng.standard_normal(n)
    a = base.a_matrix_
    return HighsLp(n, m, cost, cl, cu, lo, up, HighsSparseMatrix(n, m, a.start_.copy(), a.index_.copy(), a.value_.copy()),
                   -1, 3.5, "mixed_rows")


def long_rows_lp(m=60000, n=60000, seed=3):
    """Banded (every tile of either layout fits the staging buffer) plus a column of 15 000 entries and a row of 15 000
    entries, so that both A and A' have rows longer than 512 entries.  60 000 rows: more CTAs than an H100 has SMs, so that
    a persistent grid of one CTA per SM walks several slices per warp."""
    from highs_b200.lp import HighsLp, HighsSparseMatrix, synthetic_lp
    base = synthetic_lp(m, n, 5, seed, band=64)
    A = base.a_matrix_.to_scipy().tolil()
    rng = np.random.default_rng(seed)
    A[0, :15000] = 0.1 * rng.standard_normal(15000)[None, :]
    A[:15000, 0] = 0.1 * rng.standard_normal(15000)[:, None]
    A = A.tocsc()
    A.sort_indices()
    # a planted strictly complementary pair, as synthetic_lp plants one
    xs = np.where(rng.random(n) < 0.5, 0.0, rng.random(n))
    ys = np.where(rng.random(m) < 0.5, 0.0, rng.random(m))
    b = A @ xs - np.where(ys > 0, 0.0, rng.random(m))
    c = A.T @ ys + np.where(xs > 0, 0.0, rng.random(n))
    return HighsLp(n, m, c, base.col_lower_, base.col_upper_, b, base.row_upper_,
                   HighsSparseMatrix(n, m, A.indptr, A.indices, A.data), 1, 0.0, "long_rows")


def shuffled_lp(seed=5):
    """Columns stored with their rows in random order, a few of them repeated (cols_sorted == 0)."""
    from highs_b200.lp import HighsLp, HighsSparseMatrix
    lp = mixed_rows_lp(3000, 2500, seed)
    a = lp.a_matrix_
    rng = np.random.default_rng(seed)
    index, value = a.index_.copy(), a.value_.copy()
    for j in range(lp.num_col_):
        s, e = a.start_[j], a.start_[j + 1]
        p = rng.permutation(e - s)
        index[s:e], value[s:e] = index[s:e][p], value[s:e][p]
    # a repeated row in a few columns (same row, two values): the host sorts such pairs by value
    for j in range(0, lp.num_col_, 97):
        s, e = a.start_[j], a.start_[j + 1]
        if e - s >= 2:
            index[s + 1] = index[s]
    return HighsLp(lp.num_col_, lp.num_row_, lp.col_cost_, lp.col_lower_, lp.col_upper_, lp.row_lower_, lp.row_upper_,
                   HighsSparseMatrix(lp.num_col_, lp.num_row_, a.start_.copy(), index, value), 1, 0.0, "shuffled")


def solve_lps():
    from highs_b200.lp import synthetic_lp
    return {"synthetic_12k_9k": synthetic_lp(12000, 9000, 6, 21),
            "mixed_rows_max_offset": mixed_rows_lp(),
            "s2_banded": synthetic_lp(100_000, 100_000, 10, 12345, band=2048),
            "s2_multidiagonal": synthetic_lp(100_000, 100_000, 10, 12345, band=-2048)}


# ----------------------------------------------------------------------------------------------------------- child side
def _child_prep():
    import glob
    from highs_b200 import engine
    from highs_b200.lp import read_b2lp, synthetic_lp
    out = {}

    def check(key, lp, mode, ruiz):
        rep = engine.prep_compare_hipdlp(lp, mode, ruiz)
        bad = {k: v for k, v in rep.items() if k != "cols_sorted" and v != 0}
        out[key] = "ok" if not bad else str(bad)[:300]
        return rep

    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "instances", "*.b2lp"))):
        lp = read_b2lp(path)
        for mode, ruiz in SCALINGS:
            check(f"{os.path.basename(path)[:-5]}#{mode}/{ruiz}", lp, mode, ruiz)
    check("synthetic_100k_80k", synthetic_lp(100_000, 80_000, 8, 9), 5, 10)
    check("long_column_30k", synthetic_lp(30_000, 30_000, 6, 4, dense_col_nnz=15_000), 5, 10)
    rep = check("shuffled", shuffled_lp(), 5, 10)
    out["shuffled_is_unsorted"] = "ok" if rep["cols_sorted"] == 0 else "the shuffled LP was reported sorted"
    for mode, ruiz in SCALINGS:
        check(f"mixed_rows#{mode}/{ruiz}", mixed_rows_lp(), mode, ruiz)
    return out


def _solve_pair(lp, **prm):
    from highs_b200 import engine
    dev = engine.solve_hipdlp(lp, **prm)
    host = engine.solve_hipdlp(lp, device_prep=-1, **prm)
    return dev, host


def _same_bits(dev, host):
    assert dev["iters"] == host["iters"], ("iterations", dev["iters"], host["iters"])
    assert dev["term_code"] == host["term_code"], ("termination", dev["term_code"], host["term_code"])
    for k in VECS:
        assert dev[k].tobytes() == host[k].tobytes(), (k, float(np.max(np.abs(dev[k] - host[k]))))


def _child_solve():
    out = {}
    for name, lp in solve_lps().items():
        for tag, prm in (("iter_limit", dict(iter_limit=400)), ("converged", dict(tolerance=1e-4, iter_limit=100_000))):
            key = f"{name}#{tag}"
            try:
                dev, host = _solve_pair(lp, **prm)
                _same_bits(dev, host)
                if tag == "iter_limit":
                    assert dev["term_code"] != 0, "converged within the iteration limit"
                    assert not any(np.any(dev[k]) for k in ("col_value", "row_dual")), "an iteration-limited run returns x = y = 0"
                else:
                    assert dev["term_code"] == 0, ("did not converge", dev["iters"])
                out[key] = "ok"
            except Exception as e:   # noqa: BLE001
                out[key] = f"{type(e).__name__}: {e}"[:300]
    return out


def _child_shape(lp_name):
    """One LP under the shape the environment forces: the host path's result (saved by the parent's first call) against the
    device path's, plus the parsed shape line (stderr)."""
    from highs_b200.lp import synthetic_lp
    from highs_b200 import engine
    lp = long_rows_lp() if lp_name == "long_rows" else synthetic_lp(60_000, 60_000, 6, 17, band=256)
    res = engine.solve_hipdlp(lp, tolerance=1e-4, iter_limit=100_000)
    dump = os.environ["HIPDLP_SHAPE_DUMP"]
    np.savez(dump, iters=res["iters"], term=res["term_code"], **{k: res[k] for k in VECS})
    return {"ok": "ok"}


def child_main(case):
    if case == "prep":
        out = _child_prep()
    elif case == "solve":
        out = _child_solve()
    else:
        out = _child_shape(case.split(":", 1)[1])
    print(json.dumps(out), flush=True)
    return 0


# ----------------------------------------------------------------------------------------------------------- parent side
def _run_child(case, env_extra=None, timeout=300):
    env = {k: v for k, v in os.environ.items() if k not in _SHAPE_ENV}
    env.update(env_extra or {})
    try:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "child", case], capture_output=True, text=True,
                           timeout=timeout, cwd=ROOT, env=env)
    except subprocess.TimeoutExpired:
        pytest.fail(f"child {case} did not finish in {timeout} s (killed)")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert lines and r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-3000:])
    return json.loads(lines[-1]), r.stderr


def test_hipdlp_params_struct_matches_header():
    """sizeof(b200pdlp_hipdlp_params) from a C compile of the header against the ctypes mirror (device_prep took one of the
    reserved ints: the size is unchanged)"""
    from highs_b200 import engine
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write('#include <stdio.h>\n#include <stddef.h>\n#include "b200pdlp.h"\n'
                           'int main(){printf("%zu %zu\\n",sizeof(b200pdlp_hipdlp_params),'
                           'offsetof(b200pdlp_hipdlp_params,device_prep));return 0;}\n')
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        size, off = (int(v) for v in subprocess.check_output([exe]).split())
    assert size == ctypes.sizeof(engine.CHipdlpParams) == 56
    assert off == engine.CHipdlpParams.device_prep.offset


@pytest.mark.gpu
def test_device_prologue_matches_host_twin():
    out, _ = _run_child("prep")
    bad = {k: v for k, v in out.items() if v != "ok"}
    assert len(out) >= 74 * len(SCALINGS) + 4 and not bad, dict(list(bad.items())[:10])


@pytest.mark.gpu
def test_solve_matches_host_prologue_bit_for_bit():
    out, _ = _run_child("solve")
    bad = {k: v for k, v in out.items() if v != "ok"}
    assert len(out) == 8 and not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("lp_name", ["banded", "long_rows"])
def test_every_spmv_shape_matches_host_prologue(lp_name, tmp_path):
    host_dump = str(tmp_path / "host.npz")
    _run_child(f"shape:{lp_name}", {"HIPDLP_SHAPE_DUMP": host_dump, "B200PDLP_DEVICE_PREP": "0"})
    host = np.load(host_dump)
    assert int(host["term"]) == 0, "the host path did not converge"
    for arm, (env, want) in SHAPES.items():
        dump = str(tmp_path / f"{arm}.npz")
        _, err = _run_child(f"shape:{lp_name}", dict(env, HIPDLP_SHAPE_DUMP=dump, B200PDLP_TIMING="1"))
        m = _SHAPE_RE.search(err)
        assert m, (arm, err[-2000:])
        assert m.group(1) == want and m.group(5) == want, (arm, m.group(0))
        if want == "tiled":
            assert int(m.group(3)) == int(m.group(4)) > 0 and int(m.group(7)) == int(m.group(8)) > 0, (arm, m.group(0))
        dev = np.load(dump)
        assert int(dev["iters"]) == int(host["iters"]) and int(dev["term"]) == int(host["term"]), (arm, int(dev["iters"]), int(host["iters"]))
        for k in VECS:
            if lp_name == "long_rows" and want == "tiled":
                np.testing.assert_allclose(dev[k], host[k], rtol=1e-12, atol=1e-12 * (1 + np.abs(host[k]).max()), err_msg=f"{arm} {k}")
            else:
                assert dev[k].tobytes() == host[k].tobytes(), (arm, k, float(np.max(np.abs(dev[k] - host[k]))))


if __name__ == "__main__" and len(sys.argv) >= 3 and sys.argv[1] == "child":
    sys.exit(child_main(sys.argv[2]))
