"""b200pdlp_solve_hipdlp_batch_device without a GPU: exported, argument checks before any device work, no CPU fallback, and the
new kernels compile for sm_90a without spills."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest


def _lps(k):
    from highs_b200.lp import synthetic_lp
    return [synthetic_lp(50, 40, 3, seed) for seed in range(1, k + 1)]


def _call(engine_lib, count, lps, prm, outs):
    from highs_b200 import engine
    f = engine_lib.b200pdlp_solve_hipdlp_batch_device
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
    return clps, cres, keep


def test_exported(engine_lib):
    from highs_b200 import engine
    for sym in ("b200pdlp_solve_hipdlp_batch_device", "b200pdlp_debug_hipdlp_batch_prep_compare"):
        assert hasattr(engine_lib, sym)
        assert sym in engine.ABI_SYMBOLS


def test_torch_is_imported_lazily():
    """importing the binding must not pull torch in (solve_hipdlp_batch_device imports it when it needs it)"""
    code = "import sys; import highs_b200.engine; print('torch' in sys.modules)"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=root, timeout=120)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "False"


def test_bad_counts_and_null_arrays(engine_lib):
    from highs_b200 import engine
    prm = engine._hipdlp_params({})
    clps, cres, keep = _batch(1)
    assert _call(engine_lib, -1, clps, C.byref(prm), cres) == -1
    assert b"b200pdlp_solve_hipdlp_batch_device: count < 0" in engine_lib.b200pdlp_last_error()
    assert _call(engine_lib, 1, None, C.byref(prm), cres) == -1
    assert b"null argument" in engine_lib.b200pdlp_last_error()
    assert _call(engine_lib, 1, clps, None, cres) == -1
    assert _call(engine_lib, 1, clps, C.byref(prm), None) == -1
    assert _call(engine_lib, 0, None, None, None) == 0
    assert engine.solve_hipdlp_batch_device([]) == []


def test_rejections_before_device_work(engine_lib):
    """ordered_max < 0, a sense other than +-1 and a member without its arrays fail with ERR_ARG, naming the member, whether
    or not a device is visible; nothing is written"""
    from highs_b200 import engine
    clps, cres, keep = _batch(3)
    for i in range(3):
        cres[i].term_code, cres[i].iters = -7, -7
    assert _call(engine_lib, 3, clps, C.byref(engine._hipdlp_params(dict(ordered_max=-1))), cres) == -1
    assert re.search(rb"b200pdlp_solve_hipdlp_batch_device: member 0: ordered_max < 0", engine_lib.b200pdlp_last_error())
    clps[2].sense = 0.5
    assert _call(engine_lib, 3, clps, C.byref(engine._hipdlp_params({})), cres) == -1
    assert re.search(rb"member 2: .*sense", engine_lib.b200pdlp_last_error())
    clps[2].sense = 1.0
    clps[1].col_cost = None
    assert _call(engine_lib, 3, clps, C.byref(engine._hipdlp_params({})), cres) == -1
    assert re.search(rb"member 1: .*malformed", engine_lib.b200pdlp_last_error())
    clps[1].col_cost = clps[0].col_cost
    clps[1].a_start = None
    assert _call(engine_lib, 3, clps, C.byref(engine._hipdlp_params({})), cres) == -1
    assert re.search(rb"member 1: .*malformed", engine_lib.b200pdlp_last_error())
    for i in range(3):
        assert cres[i].term_code == -7 and cres[i].iters == -7


def test_no_device_is_a_cuda_error(engine_lib):
    from highs_b200 import engine
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    clps, cres, keep = _batch(2)
    assert _call(engine_lib, 2, clps, C.byref(engine._hipdlp_params({})), cres) == -2
    assert b"no CUDA device" in engine_lib.b200pdlp_last_error()


def test_non_cuda_tensors_are_a_type_error(engine_lib):
    """an LP whose arrays are CPU tensors is refused in Python, before the library is called"""
    torch = pytest.importorskip("torch")
    import numpy as np
    from highs_b200 import engine
    lp = _lps(1)[0]
    names = engine._LP_INDEX_ARRAYS + engine._LP_VALUE_ARRAYS
    d = {k: torch.as_tensor(np.ascontiguousarray(v, dtype=np.int32 if k in engine._LP_INDEX_ARRAYS else np.float64))
         for k, v in zip(names, engine.lp_arrays(lp))}
    d.update(num_col=int(lp.num_col_), num_row=int(lp.num_row_), sense=1.0, offset=0.0)
    with pytest.raises(TypeError, match="a_start must be a contiguous CUDA tensor"):
        engine.solve_hipdlp_batch_device([d])


def test_kernels_compile_without_spills(tmp_path):
    """batch_prep.cu for sm_90a, with the build's flags: the HiPDLP kernels without spills and without a stack frame"""
    from highs_b200 import build
    out = tmp_path / "batch_prep.o"
    r = subprocess.run([build._nvcc()] + build.NVCC_FLAGS + ["-c", os.path.join(build.CSRC, "batch_prep.cu"), "-o", str(out)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    blocks = re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'\s*\n(?:.*\n)*?.*?(\d+) bytes stack frame, (\d+) bytes "
                        r"spill stores, (\d+) bytes spill loads", r.stderr)
    props = {name: vals for name, *vals in blocks}
    for k in ("hip_batch_size_kernel", "hip_batch_prep_kernel", "hip_batch_post_kernel"):
        hits = [v for name, v in props.items() if k in name]
        assert len(hits) == 1, (k, list(props))
        assert hits[0] == ["0", "0", "0"], (k, hits[0])
