"""b200pdlp_pass_partials without a GPU: exported, its output struct against the header, NULL arguments rejected before any
device work, and the three SpMV kernels whose long-row segments write the pass's partial-sum slots compile for sm_90a
without spills."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np

from conftest import ROOT

ERR_ARG = -1


def test_exported(engine_lib):
    from highs_b200 import engine
    assert hasattr(engine_lib, "b200pdlp_pass_partials")
    assert "b200pdlp_pass_partials" in engine.ABI_SYMBOLS
    assert callable(engine.Problem.pass_partials)


def test_struct_matches_header():
    """sizeof and every field offset of b200pdlp_pass_out, from a C compile of the header"""
    from highs_b200 import engine
    s, cls = "b200pdlp_pass_out", engine.CPassOut
    body = f'printf("{s} %zu\\n", sizeof({s}));' + "".join(f'printf("{s}.{k} %zu\\n", offsetof({s}, {k}));'
                                                          for k, _ in cls._fields_)
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write('#include <stdio.h>\n#include <stddef.h>\n#include "b200pdlp.h"\nint main(){' + body + "return 0;}\n")
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = dict(ln.split() for ln in subprocess.check_output([exe], text=True).splitlines())
    assert int(got[s]) == C.sizeof(cls)
    for k, _ in cls._fields_:
        assert int(got[f"{s}.{k}"]) == getattr(cls, k).offset, k


def test_null_arguments(engine_lib):
    """every NULL pointer argument is ERR_ARG naming the call, with or without a device; nothing is written"""
    from highs_b200 import engine
    L = engine.lib()
    v = [np.full(4, 7.0) for _ in range(9)]
    lr = np.full(12, 7, dtype=np.int32)
    out = engine.CPassOut()
    out.dx2, out.long_a = 7.0, 7
    fake = C.c_void_p(1)   # never dereferenced: the NULL checks come first
    args = [fake] + [engine._p(a, engine._dp) for a in v[:4]] + [0.5, 0.5] + [engine._p(a, engine._dp) for a in v[4:9]] + \
           [4, engine._p(lr, engine._ip), 4, C.byref(out)]
    pointer_args = [0, 1, 2, 3, 4, 7, 8, 9, 10, 11, 13, 15]
    for i in pointer_args:
        a = list(args)
        a[i] = None
        assert L.b200pdlp_pass_partials(*a) == ERR_ARG, i
        assert b"b200pdlp_pass_partials: null argument" in L.b200pdlp_last_error(), i
    assert all((a == 7.0).all() for a in v) and (lr == 7).all() and (out.dx2, out.long_a) == (7.0, 7)


def test_segment_kernels_compile_without_spills(tmp_path):
    """pdhg_kernels.cu for sm_90a, with the build's flags: every instance of spmv_sell_kernel, spmv_sell_tile_kernel and
    spmv_sell_zskip_kernel without spills"""
    from highs_b200 import build
    out = tmp_path / "pdhg_kernels.o"
    r = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "pdhg_kernels.cu"),
                                                            "-o", str(out)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    blocks = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'\s*\n(?:.*\n)*?.*?(\d+) bytes stack frame, (\d+) bytes "
                        r"spill stores, (\d+) bytes spill loads", r.stderr)
    hits = {name: vals for name, *vals in blocks if re.search(r"spmv_sell_(tile_|zskip_)?kernel", name)}
    for k in ("spmv_sell_kernel", "spmv_sell_tile_kernel", "spmv_sell_zskip_kernel"):
        assert any(k in name for name in hits), (k, sorted(hits))
    spills = {name: v for name, v in hits.items() if v[1:] != ["0", "0"]}
    assert not spills, spills
