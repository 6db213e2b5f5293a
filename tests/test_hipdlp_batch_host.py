"""b200pdlp_solve_hipdlp_batch without a GPU: exported, argument checks before any device work, no CPU fallback."""
import ctypes as C

import numpy as np
import pytest


def _lps(k):
    from highs_b200.lp import synthetic_lp
    return [synthetic_lp(50, 40, 3, seed) for seed in range(1, k + 1)]


def _args(engine, lp):
    engine.lib().b200pdlp_solve_hipdlp_batch.argtypes = [C.c_int32, C.POINTER(engine.CLp), C.POINTER(engine.CHipdlpParams),
                                                         C.POINTER(engine.CResult)]
    prm = engine._hipdlp_params({})
    clp, keep = engine.make_clp(lp)
    res, arrays = engine._mk_result(lp)
    return prm, clp, res, (keep, arrays)


def test_exported(engine_lib):
    from highs_b200 import engine
    assert hasattr(engine_lib, "b200pdlp_solve_hipdlp_batch")
    assert "b200pdlp_solve_hipdlp_batch" in engine.ABI_SYMBOLS


def test_no_device_is_a_cuda_error(engine_lib):
    from highs_b200 import engine
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(engine.EngineError, match=r"\(-2\).*no CUDA device"):
        engine.solve_hipdlp_batch(_lps(3))


def test_bad_counts_and_null_arrays(engine_lib):
    from highs_b200 import engine
    prm, clp, res, keep = _args(engine, _lps(1)[0])
    f = engine_lib.b200pdlp_solve_hipdlp_batch
    assert f(-1, C.byref(clp), C.byref(prm), C.byref(res)) == -1
    assert b"count < 0" in engine_lib.b200pdlp_last_error()
    assert f(1, None, C.byref(prm), C.byref(res)) == -1
    assert b"null argument" in engine_lib.b200pdlp_last_error()
    assert f(1, C.byref(clp), None, C.byref(res)) == -1
    assert f(1, C.byref(clp), C.byref(prm), None) == -1
    assert f(0, None, None, None) == 0
    assert engine.solve_hipdlp_batch([]) == []


def test_rejections_name_the_member(engine_lib):
    """a member too large for ordered mode, or a malformed one, fails the call with its index, before any device work"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    with pytest.raises(engine.EngineError, match=r"\(-1\).*b200pdlp_solve_hipdlp_batch: member 2: .*exceeds ordered_max = 4096"):
        engine.solve_hipdlp_batch(_lps(2) + [synthetic_lp(5000, 4000, 3, 1)])
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 1: .*exceeds ordered_max = 30"):
        engine.solve_hipdlp_batch([synthetic_lp(20, 20, 3, 1), synthetic_lp(50, 40, 3, 1)], ordered_max=30)
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 0: ordered_max < 0"):
        engine.solve_hipdlp_batch(_lps(1), ordered_max=-1)
    bad = _lps(3)
    bad[1].sense_ = 3
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 1: .*sense"):
        engine.solve_hipdlp_batch(bad)
    bad = _lps(3)
    bad[2].a_matrix_.index_[0] = 10 ** 6
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 2: .*a_index"):
        engine.solve_hipdlp_batch(bad)


def test_hipdlp_classification_decides(engine_lib):
    """1e25 row bounds are finite for HiPDLP: 100 rows with one finite bound and 1e25 become ranged rows with a slack column
    each, so 4000 columns give a 4100-column standard form, over ordered_max; pdlp's 1e20 rule sees >= rows and 4000 columns"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    big = synthetic_lp(100, 4000, 3, 1)
    big.row_upper_ = np.full(100, 1e25)
    assert engine.host_form(big, 1)["n"] == 4000
    assert engine.host_form_hipdlp(big)["n"] == 4100
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 1: standard form 100 x 4100 exceeds ordered_max = 4096"):
        engine.solve_hipdlp_batch([_lps(1)[0], big, _lps(1)[0]])


def test_rejection_writes_nothing(engine_lib):
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    lps = _lps(1) + [synthetic_lp(5000, 5000, 4, 3)]
    engine.lib().b200pdlp_solve_hipdlp_batch.argtypes = [C.c_int32, C.POINTER(engine.CLp), C.POINTER(engine.CHipdlpParams),
                                                         C.POINTER(engine.CResult)]
    clps, cres, keep, arrays = (engine.CLp * 2)(), (engine.CResult * 2)(), [], []
    for i, lp in enumerate(lps):
        clps[i], k = engine.make_clp(lp)
        keep.append(k)
        cres[i], a = engine._mk_result(lp)
        for v in a:
            v.fill(7.0)
        cres[i].term_code, cres[i].iters = -7, -7
        arrays.append(a)
    prm = engine._hipdlp_params({})
    assert engine_lib.b200pdlp_solve_hipdlp_batch(2, clps, C.byref(prm), cres) == -1
    assert b"member 1" in engine_lib.b200pdlp_last_error()
    for i in range(2):
        assert cres[i].term_code == -7 and cres[i].iters == -7
        assert all((v == 7.0).all() for v in arrays[i])


def test_unknown_parameter(engine_lib):
    from highs_b200 import engine
    with pytest.raises(TypeError, match="unknown parameter"):
        engine.solve_hipdlp_batch(_lps(1), tol_primal=1e-4)
