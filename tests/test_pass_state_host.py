"""b200pdlp_pass_state without a GPU: exported, its two structs against the header, and NULL arguments and an out-of-range
state rejected before any device work, with nothing written."""
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
    assert hasattr(engine_lib, "b200pdlp_pass_state")
    assert "b200pdlp_pass_state" in engine.ABI_SYMBOLS
    assert callable(engine.Problem.pass_state)


def test_structs_match_header():
    """sizeof and every field offset of b200pdlp_pass_state_in / b200pdlp_pass_state_out, from a C compile of the header"""
    from highs_b200 import engine
    fields = {"b200pdlp_pass_state_in": engine.CPassStateIn, "b200pdlp_pass_state_out": engine.CPassStateOut}
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


def _call(engine, cin, null=None, problem=C.c_void_p(1)):
    """the call on a fake problem (never dereferenced: these rejections come first); argument `null` replaced by NULL.
    Returns (rc, error text, nothing written)"""
    L = engine.lib()
    v = [np.full(8, 7.0) for _ in range(9)]
    lr = np.full(12, 7, dtype=np.int32)
    nz = [np.full(4, 7, dtype=np.uint8) for _ in range(2)]
    out = engine.CPassStateOut()
    C.memset(C.byref(out), 0x5A, C.sizeof(out))
    before = bytes(out)
    args = ([problem, C.byref(cin)] + [engine._p(a, engine._dp) for a in v] + [4, engine._p(lr, engine._ip), 4] +
            [engine._p(a, engine._u8p) for a in nz] + [C.byref(out)])
    if null is not None:
        args[null] = None
    rc = L.b200pdlp_pass_state(*args)
    clean = all((a == 7.0).all() for a in v) and (lr == 7).all() and all((a == 7).all() for a in nz) and bytes(out) == before
    return rc, L.b200pdlp_last_error(), clean


def test_null_arguments(engine_lib):
    """every NULL pointer argument is ERR_ARG naming the call, with or without a device; nothing is written"""
    from highs_b200 import engine
    cin = engine.CPassStateIn(tau=0.5, sigma=0.5, beta=1.0, adaptive=1, stop_iter=100)
    pointer_args = [0, 1] + list(range(2, 11)) + [12, 14, 15, 16]
    for i in pointer_args:
        rc, msg, clean = _call(engine, cin, null=i)
        assert rc == ERR_ARG and b"b200pdlp_pass_state: null argument" in msg and clean, (i, rc, msg)


@pytest.mark.parametrize("field,value", [("cur", 2), ("cur", -1), ("iter", -1), ("step_iter", -1)])
def test_state_out_of_range(engine_lib, field, value):
    """a buffer half other than 0 or 1, and a negative iteration count: ERR_ARG before the problem is looked at"""
    from highs_b200 import engine
    cin = engine.CPassStateIn(tau=0.5, sigma=0.5, beta=1.0, adaptive=1, stop_iter=100)
    setattr(cin, field, value)
    rc, msg, clean = _call(engine, cin)
    assert rc == ERR_ARG and b"cur must be 0 or 1, iter and step_iter >= 0" in msg and clean, (field, value, rc, msg)
