"""b200pdlp_solve_hipdlp_batch_mixed_device without a GPU: exported, argument checks before any device work, no CPU fallback,
and the tree-mode prologue kernels compile for sm_90a without spills."""
import ctypes as C
import os
import re
import subprocess

import pytest


def _lps(k):
    from highs_b200.lp import synthetic_lp
    return [synthetic_lp(50, 40, 3, seed) for seed in range(1, k + 1)]


def _call(engine_lib, count, lps, prm, outs):
    from highs_b200 import engine
    f = engine_lib.b200pdlp_solve_hipdlp_batch_mixed_device
    f.argtypes = [C.c_int32, C.POINTER(engine.CLp), C.POINTER(engine.CHipdlpParams), C.POINTER(engine.CResult)]
    return f(count, lps, prm, outs)


def _batch(k):
    from highs_b200 import engine
    lps = _lps(k)
    clps, cres, keep = (engine.CLp * k)(), (engine.CResult * k)(), []
    for i, lp in enumerate(lps):
        clps[i], kk = engine.make_clp(lp)
        cres[i], a = engine._mk_result(lp)
        keep += [kk, a]
    for i in range(k):   # sentinels: nothing may be written on an error
        cres[i].term_code, cres[i].iters, cres[i].setup_seconds, cres[i].trace_len = -7, -7, -7.0, -7
    return clps, cres, keep


def _untouched(cres, k):
    for i in range(k):
        assert (cres[i].term_code, cres[i].iters, cres[i].setup_seconds, cres[i].trace_len) == (-7, -7, -7.0, -7), i


def test_exported(engine_lib):
    from highs_b200 import engine
    for sym in ("b200pdlp_solve_hipdlp_batch_mixed_device", "b200pdlp_debug_hipdlp_tree_prep_compare"):
        assert hasattr(engine_lib, sym)
        assert sym in engine.ABI_SYMBOLS
    assert len(engine.HIPDLP_TREE_PREP_ITEMS) == 31


def test_bad_counts_and_null_arrays(engine_lib):
    from highs_b200 import engine
    prm = engine._hipdlp_params({})
    clps, cres, keep = _batch(1)
    assert _call(engine_lib, -1, clps, C.byref(prm), cres) == -1
    assert b"b200pdlp_solve_hipdlp_batch_mixed_device: count < 0" in engine_lib.b200pdlp_last_error()
    assert _call(engine_lib, 1, None, C.byref(prm), cres) == -1
    assert b"null argument" in engine_lib.b200pdlp_last_error()
    assert _call(engine_lib, 1, clps, None, cres) == -1
    assert _call(engine_lib, 1, clps, C.byref(prm), None) == -1
    _untouched(cres, 1)
    assert _call(engine_lib, 0, None, None, None) == 0
    assert engine.solve_hipdlp_batch_mixed_device([]) == []


def test_rejections_before_device_work(engine_lib):
    """a sense other than +-1 and a member without its arrays fail with ERR_ARG, naming the member, whether or not a device
    is visible; nothing is written"""
    from highs_b200 import engine
    clps, cres, keep = _batch(3)
    clps[2].sense = 0.5
    assert _call(engine_lib, 3, clps, C.byref(engine._hipdlp_params({})), cres) == -1
    assert re.search(rb"b200pdlp_solve_hipdlp_batch_mixed_device: member 2: .*sense", engine_lib.b200pdlp_last_error())
    clps[2].sense = 1.0
    clps[1].col_cost = None
    assert _call(engine_lib, 3, clps, C.byref(engine._hipdlp_params({})), cres) == -1
    assert re.search(rb"member 1: .*malformed", engine_lib.b200pdlp_last_error())
    clps[1].col_cost = clps[0].col_cost
    clps[0].a_start = None
    assert _call(engine_lib, 3, clps, C.byref(engine._hipdlp_params({})), cres) == -1
    assert re.search(rb"member 0: .*malformed", engine_lib.b200pdlp_last_error())
    _untouched(cres, 3)


def test_ordered_max_negative_is_not_an_argument_error(engine_lib):
    """ordered_max < 0 makes every member a tree member: the call gets past the argument checks (to the device check, or to
    the host pointers' rejection when a GPU is visible)"""
    from highs_b200 import engine
    clps, cres, keep = _batch(2)
    rc = _call(engine_lib, 2, clps, C.byref(engine._hipdlp_params(dict(ordered_max=-1))), cres)
    msg = engine_lib.b200pdlp_last_error()
    assert b"ordered_max" not in msg, msg
    if engine.device_count() > 0:
        assert rc == -1 and b"member 0: a_start is not device memory" in msg, msg
    else:
        assert rc == -2 and b"no CUDA device" in msg, msg
    _untouched(cres, 2)


def test_no_device_is_a_cuda_error(engine_lib):
    from highs_b200 import engine
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    clps, cres, keep = _batch(2)
    assert _call(engine_lib, 2, clps, C.byref(engine._hipdlp_params({})), cres) == -2
    assert b"no CUDA device" in engine_lib.b200pdlp_last_error()
    _untouched(cres, 2)


def test_prep_compare_rejects_bad_arguments(engine_lib):
    from highs_b200 import engine
    f = engine_lib.b200pdlp_debug_hipdlp_tree_prep_compare
    f.argtypes = [C.c_int32, C.POINTER(engine.CLp), C.c_int32, C.c_int32, engine._dp]
    assert f(-1, None, 5, 10, None) == -1
    assert b"b200pdlp_debug_hipdlp_tree_prep_compare: bad arguments" in engine_lib.b200pdlp_last_error()
    assert f(0, None, 5, 10, None) == 0


def test_unknown_parameter_is_a_type_error():
    from highs_b200 import engine
    with pytest.raises(TypeError, match="unknown parameter"):
        engine.solve_hipdlp_batch_mixed_device([], not_a_parameter=1)


def test_kernels_compile_without_spills(tmp_path):
    """batch_tree_prep.cu for sm_90a, with the build's flags: every kernel without spills and without a stack frame"""
    from highs_b200 import build
    out = tmp_path / "batch_tree_prep.o"
    r = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "batch_tree_prep.cu"), "-o", str(out)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    blocks = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'\s*\n(?:.*\n)*?.*?(\d+) bytes stack frame, (\d+) bytes "
                        r"spill stores, (\d+) bytes spill loads", r.stderr)
    props = {name: vals for name, *vals in blocks}
    for k in ("hip_tree_plan_kernel", "hip_tree_form_kernel", "hip_tree_fill_kernel", "hip_tree_post_kernel"):
        hits = [v for name, v in props.items() if k in name]
        assert len(hits) == 1, (k, list(props))
        assert hits[0] == ["0", "0", "0"], (k, hits[0])
