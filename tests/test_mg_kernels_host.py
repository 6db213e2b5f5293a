"""b200pdlp_pass_partials_mg and b200pdlp_check_device_mg without a GPU: exported, its structs against the header, the argument errors that need no
problem rejected before anything is written, and no CPU fallback.  The rejections that need real problems (rank order,
unlinked ranks, HiPDLP problems, caps) run in tests/test_gpu_mg_kernels.py."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT

ERR_ARG = -1


def test_exported(engine_lib):
    from highs_b200 import engine
    for name in ("b200pdlp_pass_partials_mg", "b200pdlp_check_device_mg"):
        assert hasattr(engine_lib, name) and name in engine.ABI_SYMBOLS, name
    assert callable(engine.pass_partials_mg) and callable(engine.check_device_mg) and callable(engine.linked_shards)


def test_structs_match_header():
    """sizeof and every field offset of b200pdlp_pass_in / b200pdlp_pass_mg_out, from a C compile of the header"""
    from highs_b200 import engine
    fields = {"b200pdlp_pass_in": engine.CPassIn, "b200pdlp_pass_mg_out": engine.CPassMgOut}
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


def _args(engine, probs, world, vs, slots, lr, out, cin):
    return ([probs, world, C.byref(cin)] + [engine._p(v, engine._dp) for v in vs] + [engine._p(slots, engine._dp), 8,
            engine._p(lr, engine._ip), 4, out])


def test_rejections_write_nothing(engine_lib):
    """every NULL pointer but part_in, a NULL problem, and a world outside 2..16: ERR_ARG naming the call, nothing written"""
    from highs_b200 import engine
    L = engine.lib()
    vs = [np.full(64, 7.0) for _ in range(15)]
    slots, lr = np.full(64, 7.0), np.full(64, 7, dtype=np.int32)
    out = (engine.CPassMgOut * 2)()
    C.memset(out, 0x5A, C.sizeof(out))
    before = bytes(out)
    cin = engine.CPassIn(tau=0.5, sigma=0.5, beta=1.0, eta=1.0)
    nulls = (C.c_void_p * 2)(None, None)
    fake = (C.c_void_p * 2)(1, 2)   # never dereferenced: the NULL checks come first
    args = _args(engine, fake, 2, vs, slots, lr, out, cin)
    for i in [0, 2] + list(range(3, 7)) + list(range(8, 18)) + [18, 20, 22]:
        a = list(args)
        a[i] = None
        assert L.b200pdlp_pass_partials_mg(*a) == ERR_ARG, i
        assert b"b200pdlp_pass_partials_mg: null argument" in L.b200pdlp_last_error(), i
    assert L.b200pdlp_pass_partials_mg(*_args(engine, nulls, 2, vs, slots, lr, out, cin)) == ERR_ARG
    assert b"null argument" in L.b200pdlp_last_error()
    for w in (-1, 0, 1, 17):
        assert L.b200pdlp_pass_partials_mg(*_args(engine, fake, w, vs, slots, lr, out, cin)) == ERR_ARG, w
        assert b"world must be 2 .. 16" in L.b200pdlp_last_error(), w
    assert all((v == 7.0).all() for v in vs) and (slots == 7.0).all() and (lr == 7).all() and bytes(out) == before


def test_check_rejections_write_nothing(engine_lib):
    """b200pdlp_check_device_mg: every NULL pointer (axsum / atysum only for a light check), a NULL problem, and a world
    outside 2..16: ERR_ARG naming the call, nothing written"""
    from highs_b200 import engine
    L = engine.lib()
    vs = [np.full(64, 7.0) for _ in engine.CHECK_VECTORS]
    out = (engine.CCheckOut * 2)()
    C.memset(out, 0x5A, C.sizeof(out))
    before = bytes(out)
    cin = engine.CCheckIn(interval=40, light=1)
    fake = (C.c_void_p * 2)(1, 2)
    args = [fake, 2, C.byref(cin)] + [engine._p(v, engine._dp) for v in vs] + [out]
    for i in [0, 2] + list(range(3, 17)) + [17]:
        a = list(args)
        a[i] = None
        assert L.b200pdlp_check_device_mg(*a) == ERR_ARG, i
        assert b"b200pdlp_check_device_mg: null argument" in L.b200pdlp_last_error(), i
    args[0] = (C.c_void_p * 2)(None, None)
    assert L.b200pdlp_check_device_mg(*args) == ERR_ARG and b"null argument" in L.b200pdlp_last_error()
    args[0] = fake
    for w in (-1, 1, 17):
        args[1] = w
        assert L.b200pdlp_check_device_mg(*args) == ERR_ARG and b"world must be 2 .. 16" in L.b200pdlp_last_error(), w
    assert all((v == 7.0).all() for v in vs) and bytes(out) == before


def test_no_cpu_fallback(engine_lib):
    """no device: the ranks the entry point takes cannot be created (B200PDLP_ERR_CUDA)"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(engine.EngineError, match=r"\(-2\)"):
        with engine.linked_shards(synthetic_lp(500, 400, 3, 1), 2, ordered_max=-1):
            pass
