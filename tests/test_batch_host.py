"""b200pdlp_solve_batch without a GPU: exported, argument checks before any device work, no CPU fallback."""
import ctypes as C

import pytest


def _lps(k):
    from highs_b200.lp import synthetic_lp
    return [synthetic_lp(50, 40, 3, seed) for seed in range(1, k + 1)]


def test_exported(engine_lib):
    from highs_b200 import engine
    assert hasattr(engine_lib, "b200pdlp_solve_batch")
    assert "b200pdlp_solve_batch" in engine.ABI_SYMBOLS


def test_no_device_is_a_cuda_error(engine_lib):
    from highs_b200 import engine
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(engine.EngineError, match=r"\(-2\).*no CUDA device"):
        engine.solve_batch(_lps(3))


def test_bad_counts_and_null_arrays(engine_lib):
    from highs_b200 import engine
    prm = engine.make_params()
    clp, keep = engine.make_clp(_lps(1)[0])
    res, arrays = engine._mk_result(_lps(1)[0])
    assert engine_lib.b200pdlp_solve_batch(-1, C.byref(clp), C.byref(prm), None, C.byref(res)) == -1
    assert b"count < 0" in engine_lib.b200pdlp_last_error()
    assert engine_lib.b200pdlp_solve_batch(1, None, C.byref(prm), None, C.byref(res)) == -1
    assert engine_lib.b200pdlp_solve_batch(1, C.byref(clp), None, None, C.byref(res)) == -1
    assert engine_lib.b200pdlp_solve_batch(1, C.byref(clp), C.byref(prm), None, None) == -1
    assert engine_lib.b200pdlp_solve_batch(0, None, None, None, None) == 0
    assert engine.solve_batch([]) == []


def test_rejections_name_the_member(engine_lib):
    """a member too large for ordered mode, or a malformed one, fails the call with its index, before any device work"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lps = _lps(2) + [synthetic_lp(5000, 4000, 3, 1)]
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 2: .*exceeds ordered_max = 4096"):
        engine.solve_batch(lps)
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 1: .*exceeds ordered_max = 30"):
        engine.solve_batch([synthetic_lp(20, 20, 3, 1), synthetic_lp(50, 40, 3, 1)], ordered_max=30)
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 0: ordered_max < 0"):
        engine.solve_batch(_lps(1), ordered_max=-1)
    bad = _lps(2)
    bad[1].sense_ = 3
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 1: .*sense"):
        engine.solve_batch(bad)
    with pytest.raises(engine.EngineError, match="device_scaling"):
        engine.solve_batch(_lps(1), device_scaling=2)


def test_warm_list_length(engine_lib):
    from highs_b200 import engine
    with pytest.raises(ValueError, match="2 warm starts for 3 LPs"):
        engine.solve_batch(_lps(3), warms=[None, None])
