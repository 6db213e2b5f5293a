"""b200pdlp_solve_hipdlp_batch on the GPU: every member returns the bits b200pdlp_solve_hipdlp returns for it alone, and the
HiPDLP oracle's iterations, termination and vectors.  The cases (tests/hipdlp_batch_child.py) run in a child process each:
a faulting kernel must not poison the CUDA context of the test session."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = os.path.join(ROOT, "tests", "hipdlp_batch_child.py")

pytestmark = pytest.mark.gpu

CASES = ([f"instances{v}" for v in range(5)] + [f"oracle{v}" for v in range(5)] +
         ["limits", "time_limit_zero", "converged_at_zero", "synthetic", "switches", "position", "twice", "largest"])


@pytest.mark.parametrize("case", CASES)
def test_hipdlp_batch(case):
    try:
        r = subprocess.run([sys.executable, CHILD, case], capture_output=True, text=True, timeout=900, cwd=ROOT)
    except subprocess.TimeoutExpired:
        pytest.fail(f"HiPDLP batch child {case} did not finish in 900 s (killed)")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert lines, (r.stdout[-2000:], r.stderr[-2000:])
    out = json.loads(lines[-1])
    assert out.get(case) == "ok" and r.returncode == 0, (out, r.stderr[-2000:])
