"""Row-partitioned solve over 2 GPUs (one process per GPU; fused peer-memory path and NCCL variant) against the ORACLE
(the CPU restatement pinned to the reference) on the same LP: same optimum to 1e-6 (1 + |ref|), consistent row activities,
and after a fixed number of iterations the same iterate up to the summation order.  Skipped with fewer than 2 devices."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import json, os, sys
sys.path.insert(0, %r)
import numpy as np, torch, torch.distributed as dist
from highs_b200 import engine
from highs_b200.lp import synthetic_lp
rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
lp = synthetic_lp(30000, 24000, 6, 17, dense_col_nnz=9000)
prob = engine.Problem(lp, rank=rank, world=world, device=lr)
ids = [engine.nccl_unique_id() if rank == 0 else None]
dist.broadcast_object_list(ids, src=0)
prob.comm_init(ids[0])
if sys.argv[2] == "p2p":
    handles = [None] * world
    dist.all_gather_object(handles, prob.p2p_export())
    prob.p2p_import(b"".join(handles))
res = prob.solve(tol_primal=1e-7, tol_dual=1e-7, tol_gap=1e-7, iter_limit=200000)
fix = prob.solve(iter_limit=121)
if rank == 0:
    np.savez(sys.argv[1], col_value=res["col_value"], row_dual=res["row_dual"], row_value=res["row_value"],
             col_dual=res["col_dual"], iters=res["iters"], term=res["term_code"],
             fix_col_value=fix["col_value"], fix_row_dual=fix["row_dual"], fix_iters=fix["iters"])
if sys.argv[2] == "p2p":
    prob.p2p_release()
dist.barrier()
prob.close()
dist.barrier()
dist.destroy_process_group()
''' % ROOT


_ORACLE = {}


def _oracle_runs(oracle, lp):
    """the two oracle solves all variants are compared with (minutes of CPU: once per session)"""
    if not _ORACLE:
        _ORACLE["conv"] = oracle.solve(lp, tol_primal=1e-7, tol_dual=1e-7, tol_gap=1e-7, iter_limit=200000)
        _ORACLE["fix"] = oracle.solve(lp, iter_limit=121)
    return _ORACLE["conv"], _ORACLE["fix"]


@pytest.mark.parametrize("mode,devcheck", [("p2p", 1), ("nccl", 0)], ids=["p2p-device_checks", "nccl-host_checks"])
def test_two_gpu_row_partition(engine_lib, oracle, tmp_path, mode, devcheck):
    from highs_b200 import engine
    from highs_b200.lp import synthetic_lp
    if engine.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    w = tmp_path / "worker.py"
    w.write_text(WORKER)
    out = tmp_path / "res.npz"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(29611 + 2 * devcheck + (mode == "nccl")), str(w), str(out), mode]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    multi = dict(np.load(out))
    lp = synthetic_lp(30000, 24000, 6, 17, dense_col_nnz=9000)
    orc, fix = _oracle_runs(oracle, lp)
    assert int(multi["term"]) == orc["term_code"] == 0
    o1, o2 = lp.objectiveValue(multi["col_value"]), lp.objectiveValue(orc["col_value"])
    assert abs(o1 - o2) <= 1e-6 * (1 + abs(o2))     # north-star criterion: objective to 1e-6 relative
    # converged iteration counts of two runs that differ in summation order spread by tens of percent (measured on the oracle
    # itself: profiles/r02_s2_order_sensitivity.json); the trajectory itself is compared below, where it is still comparable
    assert 0.5 * orc["iters"] <= int(multi["iters"]) <= 2.0 * orc["iters"] + 80
    # 120 iterations from the same start: the multi-GPU step rule takes the interaction term on the row side
    # (DESIGN.md section 5), identical in exact arithmetic -- the iterates agree up to rounding propagation
    assert int(multi["fix_iters"]) == fix["iters"]
    for k in ("col_value", "row_dual"):
        assert np.abs(multi["fix_" + k] - fix[k]).max() <= 1e-6 * (1 + np.abs(fix[k]).max()), k
    A = lp.a_matrix_.to_scipy()
    assert np.allclose(A @ multi["col_value"], multi["row_value"], atol=1e-8 * (1 + np.abs(multi["row_value"]).max()))
