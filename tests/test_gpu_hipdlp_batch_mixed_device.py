"""b200pdlp_solve_hipdlp_batch_mixed_device on the GPU: the tree-mode device prologue equals the host's bit for bit, and every
member returns the bits (and trace rows) b200pdlp_solve_hipdlp_batch_mixed returns for it from host arrays.  The cases
(tests/hipdlp_batch_mixed_device_child.py) run in a child process each: a faulting kernel must not poison the CUDA context
of the test session."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = os.path.join(ROOT, "tests", "hipdlp_batch_mixed_device_child.py")

pytestmark = pytest.mark.gpu

CASES = ["prep_compare"] + [f"instances_tree{v}" for v in range(5)] + ["midsize", "mixed", "clusters", "limits", "errors",
                                                                          "inputs_untouched", "kkt", "twice"]


@pytest.mark.parametrize("case", CASES)
def test_hipdlp_batch_mixed_device(case):
    try:
        r = subprocess.run([sys.executable, CHILD, case], capture_output=True, text=True, timeout=900, cwd=ROOT)
    except subprocess.TimeoutExpired:
        pytest.fail(f"HiPDLP mixed device batch child {case} did not finish in 900 s (killed)")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert lines, (r.stdout[-2000:], r.stderr[-2000:])
    out = json.loads(lines[-1])
    assert out.get(case) == "ok" and r.returncode == 0, (out, r.stderr[-2000:])
