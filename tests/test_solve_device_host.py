"""b200pdlp_solve_device and b200pdlp_solve_hipdlp_device without a GPU: exported, the ctypes mirrors of the structs they take
against the header, argument rejections before any device work that write nothing, no CPU fallback, and the sizing kernel
compiles for sm_90a without spills or a stack frame."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT

ERR_ARG, ERR_CUDA = -1, -2
SENTINEL = (-7, -7, -7.0, -7)


def _lp():
    from highs_b200.lp import synthetic_lp
    return synthetic_lp(50, 40, 3, 1)


def _result(lp):
    from highs_b200 import engine
    res, arrays = engine._mk_result(lp)
    for a in arrays:
        a[:] = 7.0
    res.term_code, res.iters, res.setup_seconds, res.trace_len = SENTINEL
    return res, arrays


def _untouched(res, arrays):
    assert (res.term_code, res.iters, res.setup_seconds, res.trace_len) == SENTINEL
    assert all((a == 7.0).all() for a in arrays)


def _pdlp(engine_lib, clp, prm, warm, res):
    from highs_b200 import engine
    f = engine_lib.b200pdlp_solve_device
    f.argtypes = [C.POINTER(engine.CLp), C.POINTER(engine.CParams), C.POINTER(engine.CWarm), C.POINTER(engine.CResult)]
    return f(clp, prm, warm, res)


def _hip(engine_lib, clp, prm, res):
    from highs_b200 import engine
    f = engine_lib.b200pdlp_solve_hipdlp_device
    f.argtypes = [C.POINTER(engine.CLp), C.POINTER(engine.CHipdlpParams), C.POINTER(engine.CResult)]
    return f(clp, prm, res)


def test_exported(engine_lib):
    from highs_b200 import engine
    for sym in ("b200pdlp_solve_device", "b200pdlp_solve_hipdlp_device"):
        assert hasattr(engine_lib, sym)
        assert sym in engine.ABI_SYMBOLS
    assert callable(engine.solve_device) and callable(engine.solve_hipdlp_device)


def test_structs_match_header():
    """sizeof and every field offset of the structs the two calls take, from a C compile of the header"""
    from highs_b200 import engine
    fields = {"b200pdlp_lp": engine.CLp, "b200pdlp_params": engine.CParams, "b200pdlp_hipdlp_params": engine.CHipdlpParams,
              "b200pdlp_warm": engine.CWarm, "b200pdlp_result": engine.CResult}
    body = "".join(f'printf("{s} %zu\\n", sizeof({s}));' + "".join(
        f'printf("{s}.{k} %zu\\n", offsetof({s}, {k}));' for k, _ in cls._fields_) for s, cls in fields.items())
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write('#include <stdio.h>\n#include <stddef.h>\n#include "b200pdlp.h"\nint main(){' + body + "return 0;}\n")
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = dict(ln.split() for ln in subprocess.check_output([exe], text=True).splitlines())
    for s, cls in fields.items():
        assert int(got[s]) == C.sizeof(cls), s
        for k, _ in cls._fields_:
            assert int(got[f"{s}.{k}"]) == getattr(cls, k).offset, (s, k)


def test_rejections_before_device_work(engine_lib):
    """NULL arguments, a bad device_scaling, a malformed b200pdlp_lp and a sense other than +-1 are ERR_ARG naming the call,
    whether or not a device is visible; nothing is written"""
    from highs_b200 import engine
    lp = _lp()
    clp, keep = engine.make_clp(lp)
    res, arrays = _result(lp)
    prm, hprm = engine.make_params(), engine._hipdlp_params({})
    for rc in (_pdlp(engine_lib, None, C.byref(prm), None, C.byref(res)), _pdlp(engine_lib, C.byref(clp), None, None, C.byref(res)),
               _pdlp(engine_lib, C.byref(clp), C.byref(prm), None, None)):
        assert rc == ERR_ARG and b"b200pdlp_solve_device: null argument" in engine_lib.b200pdlp_last_error()
    for rc in (_hip(engine_lib, None, C.byref(hprm), C.byref(res)), _hip(engine_lib, C.byref(clp), None, C.byref(res)),
               _hip(engine_lib, C.byref(clp), C.byref(hprm), None)):
        assert rc == ERR_ARG and b"b200pdlp_solve_hipdlp_device: null argument" in engine_lib.b200pdlp_last_error()
    bad = engine.make_params(device_scaling=3)
    assert _pdlp(engine_lib, C.byref(clp), C.byref(bad), None, C.byref(res)) == ERR_ARG
    assert b"device_scaling" in engine_lib.b200pdlp_last_error()
    clp.sense = 0.5
    assert _pdlp(engine_lib, C.byref(clp), C.byref(prm), None, C.byref(res)) == ERR_ARG
    assert re.search(rb"b200pdlp_solve_device: .*sense must be", engine_lib.b200pdlp_last_error())
    assert _hip(engine_lib, C.byref(clp), C.byref(hprm), C.byref(res)) == ERR_ARG
    assert re.search(rb"b200pdlp_solve_hipdlp_device: .*sense must be", engine_lib.b200pdlp_last_error())
    clp.sense = 1.0
    clp.col_cost = None
    assert _pdlp(engine_lib, C.byref(clp), C.byref(prm), None, C.byref(res)) == ERR_ARG
    assert b"malformed" in engine_lib.b200pdlp_last_error()
    assert _hip(engine_lib, C.byref(clp), C.byref(hprm), C.byref(res)) == ERR_ARG
    assert b"malformed" in engine_lib.b200pdlp_last_error()
    _untouched(res, arrays)


def test_host_pointers_or_no_device(engine_lib):
    """host arrays: with a GPU, ERR_ARG naming the first field that is not device memory; without one, ERR_CUDA (no CPU
    fallback).  Nothing is written either way."""
    from highs_b200 import engine
    lp = _lp()
    clp, keep = engine.make_clp(lp)
    res, arrays = _result(lp)
    rcs = (_pdlp(engine_lib, C.byref(clp), C.byref(engine.make_params()), None, C.byref(res)),
           _hip(engine_lib, C.byref(clp), C.byref(engine._hipdlp_params({})), C.byref(res)))
    msg = engine_lib.b200pdlp_last_error()
    if engine.device_count() > 0:
        assert rcs == (ERR_ARG, ERR_ARG) and b"b200pdlp_solve_hipdlp_device: a_start is not device memory" in msg, msg
    else:
        assert rcs == (ERR_CUDA, ERR_CUDA) and b"no CUDA device" in msg, msg
    _untouched(res, arrays)


def test_no_device_is_a_cuda_error(engine_lib):
    from highs_b200 import engine
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    lp = _lp()
    clp, keep = engine.make_clp(lp)
    res, arrays = _result(lp)
    warm = engine.CWarm(*(engine._p(np.zeros(k), engine._dp) for k in (50, 40, 40)))
    assert _pdlp(engine_lib, C.byref(clp), C.byref(engine.make_params(ordered_max=-1)), C.byref(warm), C.byref(res)) == ERR_CUDA
    assert _hip(engine_lib, C.byref(clp), C.byref(engine._hipdlp_params(dict(ordered_max=-1))), C.byref(res)) == ERR_CUDA
    assert b"no CUDA device" in engine_lib.b200pdlp_last_error()
    _untouched(res, arrays)


def test_sizing_kernel_compiles_without_spills(tmp_path):
    """batch_prep.cu for sm_90a, with the build's flags: both lp_size_kernel instances without spills and without a stack frame"""
    from highs_b200 import build
    out = tmp_path / "batch_prep.o"
    r = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "batch_prep.cu"), "-o", str(out)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    blocks = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'\s*\n(?:.*\n)*?.*?(\d+) bytes stack frame, (\d+) bytes "
                        r"spill stores, (\d+) bytes spill loads", r.stderr)
    hits = [vals for name, *vals in blocks if "lp_size_kernel" in name]
    assert len(hits) == 2, [name for name, *_ in blocks]
    assert all(h == ["0", "0", "0"] for h in hits), hits
