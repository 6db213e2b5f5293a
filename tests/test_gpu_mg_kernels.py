"""The fused multi-GPU PDHG pass, rank by rank, on G logical shards of one device (b200pdlp_pass_partials_mg).

One C call runs the solve's pass on every linked rank: the primal kernel that adds the ranks' partial A_g'y (the
reduce-scatter folded into its loads) and stores x' into every peer's xfull (the all-gather), barrier 0 with |dx|^2 in the
tail slot of the pass's parity, A_g x' with the dual step and its two accumulators, the partial A_g'y', and barrier 1 with
the step rule.  tests/mg_kernels_child.py checks what it returns against numpy replays and extended-precision sums:
  * x_new: the primal expression, bit for bit, and the one-GPU pass on the same inputs; the A'y it used: the rank-order sum
    of the seeded partials from +0.0;
  * ax_new and each rank's partial A_g'y': form_layout_eval bit for bit on lines of <= 512 entries, every line within
    gamma_k sum |a_ij x_j| of an extended-precision sum (long lines: form_layout_eval adds a segment's entries in order,
    the device as a tree, so they are held to the bound only); the reduced A'y': the rank-order sum of the partials;
  * y_new: dual_update, bit for bit;
  * each rank's slots of A_g x', both accumulators: a long row's term in its first segment's slot as 0.0 + term, +0.0 in
    the others; body slots within gamma_k of the exact sum;
  * dx2, dy2, inter: the rank-order sum of every rank's 1024-thread slot sums, identical on every rank, within gamma of
    the exact sums; tau, sigma, eta, step_iter, accepted_last: the step rule replayed (glibc pow), both branches;
  * the dense-phase sums xsum, ysum, axsum, atysum: s + w v bit for bit, axsum and atysum untouched from iteration 10;
  * the parity of the tail slot alternates call by call and a repeat returns the same bytes.
LPs: long rows of 2-8 segments in every row block and one of more than 32, long columns over several row blocks, odd n
with a padded last shard and one rank without equality rows (worlds 2, 3, 4); a 100k x 80k random LP with a dense column
(2, 4); a 9-column LP whose fourth rank owns no column at world 4 (2, 4).  Argument errors on real problems are ERR_ARG,
write nothing and return at once (no barrier waits for a peer that will not come).

Each case runs in a child process with a hard timeout, as tests/test_gpu_logical_shards.py does: a stuck barrier must not
take the session along."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = os.path.join(ROOT, "tests", "mg_kernels_child.py")

pytestmark = pytest.mark.gpu


def _run(*args, timeout=600):
    try:
        r = subprocess.run([sys.executable, CHILD, *map(str, args)], capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    except subprocess.TimeoutExpired:
        pytest.fail(f"{args}: the child did not finish in {timeout} s (killed)")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert lines, (r.returncode, r.stdout[-2000:], r.stderr[-3000:])
    return json.loads(lines[-1]), r


@pytest.mark.parametrize("case,world", [("long_lines", 2), ("long_lines", 3), ("long_lines", 4), ("random", 2), ("random", 4),
                                        ("tiny", 2), ("tiny", 4)])
def test_pass_mg(case, world):
    out, r = _run(case, world)
    assert out["ok"] and r.returncode == 0, out["fails"]
    assert out["checked"] == 39, out["checked"]


@pytest.mark.parametrize("world", [2, 3])
def test_check_mg(world):
    """test_gpu_check_device's verdict scenarios on linked ranks: every split and light case and both infeasibility rays;
    every rank's b200pdlp_check_out the same bytes; the averages, and the vectors after a restart the one-GPU check also
    chose, bit for bit the one-GPU check's"""
    from test_gpu_check_device import BRANCHES
    out, r = _run("check", world, timeout=900)
    assert out["ok"] and r.returncode == 0, out["fails"]
    assert BRANCHES <= set(out["hits"]), sorted(BRANCHES - set(out["hits"]))
    assert out["compared_restarts"] >= 4, out["compared_restarts"]


def test_rejections():
    out, r = _run("rejections")
    assert out["ok"] and r.returncode == 0, out["fails"]
