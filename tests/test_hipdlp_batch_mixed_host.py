"""b200pdlp_solve_hipdlp_batch_mixed without a GPU: exported, argument checks before any device work, no CPU fallback."""
import ctypes as C

import pytest


def _lps(k):
    from highs_b200.lp import synthetic_lp
    return [synthetic_lp(50, 40, 3, seed) for seed in range(1, k + 1)]


def _bind(engine):
    engine.lib().b200pdlp_solve_hipdlp_batch_mixed.argtypes = [C.c_int32, C.POINTER(engine.CLp),
                                                               C.POINTER(engine.CHipdlpParams), C.POINTER(engine.CResult)]
    return engine.lib().b200pdlp_solve_hipdlp_batch_mixed


def test_exported(engine_lib):
    from highs_b200 import engine
    assert hasattr(engine_lib, "b200pdlp_solve_hipdlp_batch_mixed")
    assert "b200pdlp_solve_hipdlp_batch_mixed" in engine.ABI_SYMBOLS


def test_no_device_is_a_cuda_error(engine_lib):
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(engine.EngineError, match=r"\(-2\).*no CUDA device"):
        engine.solve_hipdlp_batch_mixed(_lps(2) + [synthetic_lp(5000, 4000, 3, 1)])


def test_ordered_max_negative_is_not_an_argument_error(engine_lib):
    """ordered_max < 0 makes every member a tree member (the plain batch rejects it)"""
    from highs_b200 import engine
    if engine.device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(engine.EngineError, match=r"\(-2\)"):
        engine.solve_hipdlp_batch_mixed(_lps(2), ordered_max=-1)


def test_bad_counts_and_null_arrays(engine_lib):
    from highs_b200 import engine
    f = _bind(engine)
    lp = _lps(1)[0]
    prm = engine._hipdlp_params({})
    clp, keep = engine.make_clp(lp)
    res, arrays = engine._mk_result(lp)
    assert f(-1, C.byref(clp), C.byref(prm), C.byref(res)) == -1
    assert b"count < 0" in engine_lib.b200pdlp_last_error()
    assert f(1, None, C.byref(prm), C.byref(res)) == -1
    assert b"null argument" in engine_lib.b200pdlp_last_error()
    assert f(1, C.byref(clp), None, C.byref(res)) == -1
    assert f(1, C.byref(clp), C.byref(prm), None) == -1
    assert f(0, None, None, None) == 0
    assert engine.solve_hipdlp_batch_mixed([]) == []


def test_rejections_name_the_member(engine_lib):
    """a tree member past the cap, or a malformed member, fails the call with its index, before any device work"""
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    big = synthetic_lp(300000, 50, 1, 1)
    with pytest.raises(engine.EngineError, match=r"\(-1\).*b200pdlp_solve_hipdlp_batch_mixed: member 2: standard form "
                                                 r"300000 x \d+ exceeds max\(n, m\) = 262144 .*b200pdlp_solve_hipdlp"):
        engine.solve_hipdlp_batch_mixed(_lps(2) + [big])
    bad = _lps(3)
    bad[1].sense_ = 3
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 1: .*sense"):
        engine.solve_hipdlp_batch_mixed(bad)
    bad = _lps(3)
    bad[2].a_matrix_.index_[0] = 10 ** 6
    with pytest.raises(engine.EngineError, match=r"\(-1\).*member 2: .*a_index"):
        engine.solve_hipdlp_batch_mixed(bad)


def test_rejection_writes_nothing(engine_lib):
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    f = _bind(engine)
    lps = [synthetic_lp(5000, 4000, 3, 1), _lps(1)[0], synthetic_lp(300000, 50, 1, 2)]
    clps, cres, keep, arrays = (engine.CLp * 3)(), (engine.CResult * 3)(), [], []
    for i, lp in enumerate(lps):
        clps[i], k = engine.make_clp(lp)
        keep.append(k)
        cres[i], a = engine._mk_result(lp, 4)
        for v in a:
            v.fill(7.0)
        cres[i].term_code, cres[i].iters, cres[i].trace_len = -7, -7, -7
        arrays.append(a)
    prm = engine._hipdlp_params({})
    assert f(3, clps, C.byref(prm), cres) == -1
    assert b"member 2" in engine_lib.b200pdlp_last_error()
    for i in range(3):
        assert cres[i].term_code == -7 and cres[i].iters == -7 and cres[i].trace_len == -7
        assert all((v == 7.0).all() for v in arrays[i])


def test_unknown_parameter(engine_lib):
    from highs_b200 import engine
    with pytest.raises(TypeError, match="unknown parameter"):
        engine.solve_hipdlp_batch_mixed(_lps(1), tol_primal=1e-4)
