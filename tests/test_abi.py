"""The C-ABI library loads and exports every symbol include/b200pdlp.h declares (no GPU needed)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


def _declared():
    src = open(os.path.join(ROOT, "include", "b200pdlp.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200pdlp_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(engine_lib):
    from highs_b200 import engine
    names = _declared()
    assert len(names) >= 20
    for nm in names:
        assert hasattr(engine_lib, nm), f"libb200pdlp.so does not export {nm}"
    assert sorted(engine.ABI_SYMBOLS) == names, "engine.ABI_SYMBOLS out of sync with include/b200pdlp.h"


def test_version_and_defaults(engine_lib):
    from highs_b200 import engine
    assert engine_lib.b200pdlp_version() == 100
    p = engine.make_params()
    assert p.iter_limit == 2147483647 and p.tol_primal == 1e-7 and p.scaling == 1 and p.adaptive_step == 1
    assert p.restart == 1 and p.check_interval == 40 and p.device == -1


def test_struct_layout_matches_header(engine_lib):
    """sizes of the ctypes mirrors against a C compile of the header"""
    import subprocess
    import tempfile
    from highs_b200 import engine
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write('#include <stdio.h>\n#include "b200pdlp.h"\nint main(){printf("%zu %zu %zu %zu\\n",'
                           'sizeof(b200pdlp_lp),sizeof(b200pdlp_params),sizeof(b200pdlp_warm),sizeof(b200pdlp_result));return 0;}\n')
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(engine.CLp), ctypes.sizeof(engine.CParams), ctypes.sizeof(engine.CWarm),
                     ctypes.sizeof(engine.CResult)]


def test_no_cpu_fallback(engine_lib):
    """Without a CUDA device every compute entry point must fail loudly (never route to a CPU path)."""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    lp = synthetic_lp(50, 40, 3, 1)
    with pytest.raises(engine.EngineError, match="no CUDA device"):
        engine.solve(lp)
    with pytest.raises(engine.EngineError):
        engine.Problem(lp)
    with pytest.raises(engine.EngineError, match="no CUDA device"):
        engine.solve_multi(lp, 2)          # several GPUs from one process: same rule, and a clean error path
    with pytest.raises(engine.EngineError):
        engine.solve_logical_shards(lp, 2)
    with pytest.raises(engine.EngineError, match="no CUDA device"):
        engine.solve_hipdlp(lp)            # the HiPDLP mode as well


def test_bad_arguments(engine_lib):
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(50, 40, 3, 1)
    lp.sense_ = 3
    with pytest.raises(engine.EngineError, match="sense"):
        engine.host_form(lp)
    # checked with the other arguments, before any device is looked for
    with pytest.raises(engine.EngineError, match="device_scaling"):
        engine.solve(synthetic_lp(50, 40, 3, 1), device_scaling=2)


def test_product_does_not_touch_oracle():
    """The product path must not import, link or call anything under oracle/."""
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "highs_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cpp", ".hpp", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                if re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M) or "pdlp_oracle" in txt or "libhighs_ref" in txt:
                    bad.append(f)
    assert not bad, bad
    import subprocess
    from highs_b200 import engine
    ldd = subprocess.check_output(["ldd", engine.LIB_PATH], text=True)
    assert "oracle" not in ldd and "highs_ref" not in ldd
