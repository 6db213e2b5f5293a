"""b200pdlp_solve_device and b200pdlp_solve_hipdlp_device on the GPU: an LP already in device memory returns the bits (and
trace rows) b200pdlp_solve / b200pdlp_solve_hipdlp return for host copies of its arrays, in ordered mode, in tree mode (read
in place: no copy of the LP) and for degenerate LPs, cold and warm; errors name the field and write nothing.  The cases
(tests/solve_device_child.py) run in a child process each: a faulting kernel must not poison the CUDA context of the test
session."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = os.path.join(ROOT, "tests", "solve_device_child.py")

pytestmark = pytest.mark.gpu

CASES = [f"pdlp_instances{k}" for k in range(7)] + [f"hip_instances{v}" for v in range(5)] + \
        ["hot_starts", "synthetic", "big", "degenerate", "device_prep_off", "no_upload", "errors", "kkt", "twice"]


@pytest.mark.parametrize("case", CASES)
def test_solve_device(case):
    try:
        r = subprocess.run([sys.executable, CHILD, case], capture_output=True, text=True, timeout=900, cwd=ROOT)
    except subprocess.TimeoutExpired:
        pytest.fail(f"device-array solve child {case} did not finish in 900 s (killed)")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert lines, (r.stdout[-2000:], r.stderr[-2000:])
    out = json.loads(lines[-1])
    assert out.get(case) == "ok" and r.returncode == 0, (out, r.stderr[-2000:])
