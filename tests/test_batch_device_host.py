"""b200pdlp_solve_batch_device without a GPU: exported, argument checks before any device work, no CPU fallback, and the new
kernels compile for sm_90a without spills."""
import ctypes as C
import os
import re
import subprocess

import pytest


def _lps(k):
    from highs_b200.lp import synthetic_lp
    return [synthetic_lp(50, 40, 3, seed) for seed in range(1, k + 1)]


def _call(engine_lib, count, lps, prm, warms, outs):
    from highs_b200 import engine
    f = engine_lib.b200pdlp_solve_batch_device
    f.argtypes = [C.c_int32, C.POINTER(engine.CLp), C.POINTER(engine.CParams), C.POINTER(engine.CWarm), C.POINTER(engine.CResult)]
    return f(count, lps, prm, warms, outs)


def test_exported(engine_lib):
    from highs_b200 import engine
    for sym in ("b200pdlp_solve_batch_device", "b200pdlp_debug_batch_prep_compare"):
        assert hasattr(engine_lib, sym)
        assert sym in engine.ABI_SYMBOLS


def test_torch_is_imported_lazily():
    """importing the binding must not pull torch in (solve_batch_device imports it when it needs it)"""
    import sys
    code = "import sys; import highs_b200.engine; print('torch' in sys.modules)"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=root, timeout=120)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "False"


def test_bad_counts_and_null_arrays(engine_lib):
    from highs_b200 import engine
    prm = engine.make_params()
    clp, keep = engine.make_clp(_lps(1)[0])
    res, arrays = engine._mk_result(_lps(1)[0])
    assert _call(engine_lib, -1, C.byref(clp), C.byref(prm), None, C.byref(res)) == -1
    assert b"count < 0" in engine_lib.b200pdlp_last_error()
    assert _call(engine_lib, 1, None, C.byref(prm), None, C.byref(res)) == -1
    assert _call(engine_lib, 1, C.byref(clp), None, None, C.byref(res)) == -1
    assert _call(engine_lib, 1, C.byref(clp), C.byref(prm), None, None) == -1
    assert b"null argument" in engine_lib.b200pdlp_last_error()
    assert _call(engine_lib, 0, None, None, None, None) == 0
    assert engine.solve_batch_device([]) == []


def test_rejections_before_device_work(engine_lib):
    """ordered_max < 0, a bad device_scaling, a sense other than +-1 and a malformed member fail with ERR_ARG, naming the
    member, whether or not a device is visible"""
    from highs_b200 import engine
    lps = _lps(3)
    clps, cres, keep = (engine.CLp * 3)(), (engine.CResult * 3)(), []
    for i, lp in enumerate(lps):
        clps[i], k = engine.make_clp(lp)
        cres[i], a = engine._mk_result(lp)
        keep += [k, a]
    assert _call(engine_lib, 3, clps, C.byref(engine.make_params(ordered_max=-1)), None, cres) == -1
    assert re.search(rb"member 0: ordered_max < 0", engine_lib.b200pdlp_last_error())
    assert _call(engine_lib, 3, clps, C.byref(engine.make_params(device_scaling=2)), None, cres) == -1
    assert b"device_scaling" in engine_lib.b200pdlp_last_error()
    clps[2].sense = 3.0
    assert _call(engine_lib, 3, clps, C.byref(engine.make_params()), None, cres) == -1
    assert re.search(rb"member 2: .*sense", engine_lib.b200pdlp_last_error())
    clps[2].sense = 1.0
    clps[1].col_cost = None
    assert _call(engine_lib, 3, clps, C.byref(engine.make_params()), None, cres) == -1
    assert re.search(rb"member 1: .*malformed", engine_lib.b200pdlp_last_error())


def test_no_device_is_a_cuda_error(engine_lib):
    from highs_b200 import engine
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    lps = _lps(2)
    clps, cres, keep = (engine.CLp * 2)(), (engine.CResult * 2)(), []
    for i, lp in enumerate(lps):
        clps[i], k = engine.make_clp(lp)
        cres[i], a = engine._mk_result(lp)
        keep += [k, a]
    assert _call(engine_lib, 2, clps, C.byref(engine.make_params()), None, cres) == -2
    assert b"no CUDA device" in engine_lib.b200pdlp_last_error()


def test_warm_list_length(engine_lib):
    from highs_b200 import engine
    with pytest.raises(ValueError, match="2 warm starts for 3 LPs"):
        engine.solve_batch_device([{}, {}, {}], warms=[None, None])


def test_kernels_compile_without_spills(tmp_path):
    """batch_prep.cu for sm_90a, with the build's flags: every kernel without spills and without a stack frame"""
    from highs_b200 import build
    out = tmp_path / "batch_prep.o"
    r = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "batch_prep.cu"), "-o", str(out)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", r.stderr)
    assert {k for k in ("batch_size_kernel", "batch_prep_kernel", "batch_post_kernel") if any(k in e for e in kernels)} == \
        {"batch_size_kernel", "batch_prep_kernel", "batch_post_kernel"}
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == len(kernels)
    assert all(p == ("0", "0", "0") for p in props), props
