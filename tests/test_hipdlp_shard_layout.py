"""The layouts of the HiPDLP mode on several GPUs (host_prep.cpp plan_hipdlp_shards / build_hipdlp_shard), evaluated on the
host in the kernels' traversal order (b200pdlp_hipdlp_shard_layout_eval); no GPU needed.

Rank g of G holds device rows [R_g, R_g+1) of A and device columns [C_g, C_g+1) of A', cut from the one-GPU device orders.
Its rows of A x and its columns of A'y must be the one-GPU layout's values byte for byte
(b200pdlp_form_layout_eval, world = 1), for every G and in both ordered and tree mode; together the blocks must tile the
device rows and columns exactly.  This is what makes a G-rank solve return the one-GPU bits."""
import glob
import os

import numpy as np
import pytest

from conftest import GOLDEN
from highs_b200 import engine
from highs_b200.lp import HighsLp, HighsSparseMatrix, kHighsInf, read_b2lp, synthetic_lp
from test_gpu_hipdlp_device_prep import mixed_rows_lp, shuffled_lp

INSTANCES = sorted(glob.glob(os.path.join(GOLDEN, "instances", "*.b2lp")))
WORLDS = (1, 2, 3, 4)


def _check(lp, world, ordered_max):
    r = engine.hipdlp_shard_layout_eval(lp, world, ordered_max=ordered_max, seed=world)
    n, m = r["n"], r["m"]
    ax, aty = np.full(m, np.nan), np.full(n, np.nan)
    rows, cols = [], []
    for g in range(world):
        st = r["stats"][g]
        rows.append((int(st[0]), int(st[1])))
        cols.append((int(st[2]), int(st[3])))
        assert bool(st[4]) == r["ref_ordered"], "ordered mode is decided on the whole problem"
        mine_r, mine_c = ~np.isnan(r["ax"][g]), ~np.isnan(r["aty"][g])
        assert mine_r.sum() == st[1] - st[0] and mine_c.sum() == st[3] - st[2]
        assert not (mine_r & ~np.isnan(ax)).any() and not (mine_c & ~np.isnan(aty)).any(), "two ranks own one row / column"
        ax[mine_r] = r["ax"][g][mine_r]
        aty[mine_c] = r["aty"][g][mine_c]
    # the blocks tile the device rows and columns
    for b, total in ((rows, m), (cols, n)):
        assert b[0][0] == 0 and b[-1][1] == total
        assert all(lo <= hi for lo, hi in b) and all(b[k][1] == b[k + 1][0] for k in range(world - 1))
    assert ax.tobytes() == r["ref_ax"].tobytes()
    assert aty.tobytes() == r["ref_aty"].tobytes()
    return r


@pytest.mark.parametrize("path", INSTANCES, ids=[os.path.basename(p)[:-5] for p in INSTANCES])
def test_instances(engine_lib, path):
    lp = read_b2lp(path)
    for world in WORLDS:
        for ordered_max in (0, -1):
            _check(lp, world, ordered_max)


def _long_row_and_column_lp(m=20000, n=18000, seed=3):
    """A column of 15 000 entries and a row of 15 000 entries (long rows of A' and of A), columns stored with shuffled
    rows, and every HiPDLP row class."""
    rng = np.random.default_rng(seed)
    A = synthetic_lp(m, n, 4, seed).a_matrix_.to_scipy().tolil()
    A[1, :15000] = rng.standard_normal(15000)[None, :]
    A[:15000, 2] = rng.standard_normal(15000)[:, None]
    A = A.tocsc()
    A.sort_indices()
    index, value = A.indices.copy(), A.data.copy()
    for j in range(0, n, 3):
        s, e = A.indptr[j], A.indptr[j + 1]
        p = rng.permutation(e - s)
        index[s:e], value[s:e] = index[s:e][p], value[s:e][p]
    cls = np.arange(m) % 5
    lo = np.where(cls == 1, -kHighsInf, -1.0)
    lo = np.where(cls == 4, -kHighsInf, lo)
    up = np.where(cls == 0, -1.0, kHighsInf)
    up = np.where(cls == 1, 2.0, up)
    up = np.where(cls == 3, 3.0, up)
    return HighsLp(n, m, rng.standard_normal(n), np.zeros(n), np.full(n, 10.0), lo, up,
                   HighsSparseMatrix(n, m, A.indptr.astype(np.int32), index.astype(np.int32), value), 1, 0.0, "long_rc")


@pytest.mark.parametrize("world", WORLDS)
def test_long_rows_and_columns(engine_lib, world):
    lp = _long_row_and_column_lp()
    r = _check(lp, world, 0)
    assert not r["ref_ordered"]
    # tree mode cuts both 15 000-entry vectors into segments, on whichever rank owns them
    assert sum(st[5] for st in r["stats"]) >= 1 and sum(st[6] for st in r["stats"]) >= 1
    # ordered mode (forced up to this size) splits no row
    r = _check(lp, world, 40000)
    assert r["ref_ordered"] and all(st[5] == 0 and st[6] == 0 for st in r["stats"])


@pytest.mark.parametrize("world", WORLDS)
def test_mixed_rows_and_shuffled_columns(engine_lib, world):
    for lp in (mixed_rows_lp(), shuffled_lp()):
        for ordered_max in (0, -1):
            _check(lp, world, ordered_max)


def test_fewer_rows_and_columns_than_ranks(engine_lib):
    n, m = 3, 2
    start = np.array([0, 2, 3, 4], dtype=np.int32)
    index = np.array([0, 1, 1, 0], dtype=np.int32)
    value = np.array([1.0, -2.0, 3.0, 4.0])
    lp = HighsLp(n, m, np.ones(n), np.zeros(n), np.full(n, kHighsInf), np.array([1.0, 0.5]), np.array([kHighsInf, kHighsInf]),
                 HighsSparseMatrix(n, m, start, index, value), 1, 0.0, "tiny")
    for world in WORLDS:
        for ordered_max in (0, -1):
            r = _check(lp, world, ordered_max)
            if world == 4:
                assert any(st[1] == st[0] for st in r["stats"]) and any(st[3] == st[2] for st in r["stats"])
