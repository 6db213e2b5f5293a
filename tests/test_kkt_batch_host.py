"""b200pdlp_kkt_check_batch / _device without a GPU: exported, the struct mirror, argument and array checks before any device
work with nothing written, no CPU fallback, the Python length checks, and the new kernels compile for sm_90a without spills."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

SENTINEL = -12345


def _lps(k):
    from highs_b200.lp import synthetic_lp
    return [synthetic_lp(50, 40, 3, seed) for seed in range(1, k + 1)]


def _sol(lp, seed=0):
    rng = np.random.default_rng(seed)
    n, m = lp.num_col_, lp.num_row_
    return dict(col_value=rng.standard_normal(n), col_dual=rng.standard_normal(n), row_value=rng.standard_normal(m),
                row_dual=rng.standard_normal(m))


class _Batch:
    """ctypes arrays of `lps` and solutions, and an inout array filled with a sentinel"""

    def __init__(self, lps):
        from highs_b200 import engine
        k = len(lps)
        self.clps, self.csols, self.infos, self.keep = (engine.CLp * k)(), (engine.CSolution * k)(), (engine.CKktInfo * k)(), []
        for i, lp in enumerate(lps):
            self.clps[i], kp = engine.make_clp(lp)
            arrs = [np.ascontiguousarray(v) for v in _sol(lp, i).values()]
            self.csols[i] = engine.CSolution(*(engine._p(a, engine._dp) for a in arrs))
            self.keep += [kp, arrs]
        C.memset(self.infos, 0x5A, C.sizeof(self.infos))
        for i in range(k):
            self.infos[i].model_status = SENTINEL
        self.snapshot = bytes(self.infos)
        tol = engine.CKktTolerances()
        for f, _ in engine.CKktTolerances._fields_:
            setattr(tol, f, 1e-7)
        self.tol = tol

    def untouched(self):
        return bytes(self.infos) == self.snapshot


def _call(engine_lib, name, count, lps, sols, tol, inout, device=-1):
    from highs_b200 import engine
    f = getattr(engine_lib, name)
    f.argtypes = [C.c_int32, C.POINTER(engine.CLp), C.POINTER(engine.CSolution), C.POINTER(engine.CKktTolerances), C.c_int32,
                  C.POINTER(engine.CKktInfo)]
    return f(count, lps, sols, tol, device, inout)


NAMES = ("b200pdlp_kkt_check_batch", "b200pdlp_kkt_check_batch_device")


def test_exported(engine_lib):
    from highs_b200 import engine
    for sym in NAMES:
        assert hasattr(engine_lib, sym)
        assert sym in engine.ABI_SYMBOLS


def test_solution_struct_matches_the_header(tmp_path):
    """sizeof and offsets of b200pdlp_solution from a C compile of the header equal the ctypes mirror's"""
    from highs_b200 import engine
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "s.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200pdlp.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(b200pdlp_solution), offsetof(b200pdlp_solution, col_value),\n'
                   '         offsetof(b200pdlp_solution, col_dual), offsetof(b200pdlp_solution, row_value),\n'
                   '         offsetof(b200pdlp_solution, row_dual));\n  return 0;\n}\n')
    exe = tmp_path / "s"
    r = subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    S = engine.CSolution
    assert got == [C.sizeof(S), S.col_value.offset, S.col_dual.offset, S.row_value.offset, S.row_dual.offset]


@pytest.mark.parametrize("name", NAMES)
def test_bad_arguments_write_nothing(engine_lib, name):
    b = _Batch(_lps(3))
    assert _call(engine_lib, name, -1, b.clps, b.csols, C.byref(b.tol), b.infos) == -1
    assert b"count < 0" in engine_lib.b200pdlp_last_error()
    for args in ((None, b.csols, C.byref(b.tol), b.infos), (b.clps, None, C.byref(b.tol), b.infos),
                 (b.clps, b.csols, None, b.infos), (b.clps, b.csols, C.byref(b.tol), None)):
        assert _call(engine_lib, name, 3, *args) == -1
        assert b"null argument" in engine_lib.b200pdlp_last_error()
    assert _call(engine_lib, name, 0, None, None, None, None) == 0
    b.clps[2].num_row = -1
    assert _call(engine_lib, name, 3, b.clps, b.csols, C.byref(b.tol), b.infos) == -1
    assert re.search(rb"member 2: num_col < 0 or num_row < 0", engine_lib.b200pdlp_last_error())
    b.clps[2].num_row = 40
    b.csols[1].row_dual = None
    assert _call(engine_lib, name, 3, b.clps, b.csols, C.byref(b.tol), b.infos) == -1
    assert re.search(rb"member 1: NULL array", engine_lib.b200pdlp_last_error())
    assert b.untouched()


def test_null_arrays_of_length_zero_are_allowed_before_device_work(engine_lib):
    """an LP without rows may pass NULL row arrays: the call gets past the argument checks (to the device lookup)"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lp = synthetic_lp(5, 4, 2, 1)
    b = _Batch([lp])
    b.clps[0].num_row = 0
    b.clps[0].a_start = engine._p(np.zeros(lp.num_col_ + 1, dtype=np.int32), engine._ip)
    b.keep.append(b.clps[0].a_start)
    for f in ("row_lower", "row_upper"):
        setattr(b.clps[0], f, None)
    for f in ("row_value", "row_dual"):
        setattr(b.csols[0], f, None)
    rc = _call(engine_lib, "b200pdlp_kkt_check_batch", 1, b.clps, b.csols, C.byref(b.tol), b.infos)
    assert rc in (0, -2), engine_lib.b200pdlp_last_error()
    if rc == -2:
        assert b"no CUDA device" in engine_lib.b200pdlp_last_error()


def test_malformed_arrays_are_rejected_on_the_host(engine_lib):
    """the host variant checks a_start / a_index on the host, before any device lookup, naming the lowest failing member"""
    from highs_b200 import engine
    lps = _lps(6)
    b = _Batch(lps)
    bad_start = np.array(lps[2].a_matrix_.start_, dtype=np.int32)
    bad_start[5], bad_start[6] = bad_start[6], bad_start[5] - 1          # decreasing
    bad_index = np.array(lps[4].a_matrix_.index_, dtype=np.int32)
    bad_index[3] = lps[4].num_row_                                        # out of range
    first = np.array(lps[1].a_matrix_.start_, dtype=np.int32) + 1         # a_start[0] != 0
    b.keep += [bad_start, bad_index, first]
    b.clps[4].a_index = engine._p(bad_index, engine._ip)
    assert _call(engine_lib, "b200pdlp_kkt_check_batch", 6, b.clps, b.csols, C.byref(b.tol), b.infos) == -1
    assert re.search(rb"member 4: .*a_index entry outside", engine_lib.b200pdlp_last_error())
    b.clps[2].a_start = engine._p(bad_start, engine._ip)
    assert _call(engine_lib, "b200pdlp_kkt_check_batch", 6, b.clps, b.csols, C.byref(b.tol), b.infos) == -1
    assert re.search(rb"member 2: .*non-decreasing", engine_lib.b200pdlp_last_error())
    b.clps[1].a_start = engine._p(first, engine._ip)
    assert _call(engine_lib, "b200pdlp_kkt_check_batch", 6, b.clps, b.csols, C.byref(b.tol), b.infos) == -1
    assert re.search(rb"member 1: .*a_start\[0\] must be 0", engine_lib.b200pdlp_last_error())
    assert b.untouched()


@pytest.mark.parametrize("name", NAMES)
def test_no_device_is_a_cuda_error(engine_lib, name):
    from highs_b200 import engine
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    b = _Batch(_lps(2))
    assert _call(engine_lib, name, 2, b.clps, b.csols, C.byref(b.tol), b.infos) == -2
    assert b"no CUDA device" in engine_lib.b200pdlp_last_error()
    assert b.untouched()


def test_python_length_checks():
    from highs_b200 import engine
    lps = _lps(3)
    sols = [_sol(lp) for lp in lps]
    with pytest.raises(ValueError, match="2 solutions for 3 LPs"):
        engine.kkt_check_batch(lps, sols[:2])
    with pytest.raises(ValueError, match="2 model statuses for 3 LPs"):
        engine.kkt_check_batch(lps, sols, model_status=[7, 15])
    with pytest.raises(ValueError, match="1 solutions for 2 LPs"):
        engine.kkt_check_batch_device([{}, {}], [{}])
    with pytest.raises(ValueError, match="3 model statuses for 2 LPs"):
        engine.kkt_check_batch_device([{}, {}], [{}, {}], model_status=[7, 7, 7])


def test_torch_is_imported_lazily():
    """importing the binding must not pull torch in (kkt_check_batch_device imports it when it needs it)"""
    code = "import sys; import highs_b200.engine; print('torch' in sys.modules)"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=root, timeout=120)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "False"


def test_kernels_compile_without_spills(tmp_path):
    """kkt_batch.cu for sm_90a, with the build's flags: both kernels without spills and without a stack frame"""
    from highs_b200 import build
    out = tmp_path / "kkt_batch.o"
    r = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "kkt_batch.cu"), "-o", str(out)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'", r.stderr)
    names = sorted(m.group(1) for m in (re.search(r"(kkt_batch_(?:check_)?kernel)E", e) for e in kernels) if m)
    assert names == ["kkt_batch_check_kernel", "kkt_batch_kernel"]
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(props) == len(kernels) == 2
    assert all(p == ("0", "0", "0") for p in props), props
