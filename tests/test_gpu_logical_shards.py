"""SURVEY.md 8(e): "the same code path must run with G logical shards on 1 device".  G problems (rank g of G) are
created in ONE process on ONE GPU, wired to each other with b200pdlp_p2p_link_local (plain pointers instead of CUDA IPC,
no NCCL), and solved by G host threads: the row/column partition, the fused peer-memory kernels, both flag barriers,
the device-side step rule, the device-side checks and the NCCL-free solution assembly all run as they do on G GPUs.
This is what lets a one-GPU box exercise the multi-GPU path (tests/test_gpu_multi.py needs two devices).

Each case runs in a child process with a hard timeout (a stuck barrier must not take the session along).

Round 2: the path deadlocked on hardware because CUDA loads kernels lazily and a load can need a context-wide synchronisation,
which never comes while a peer rank's barrier kernel spins on the same device; the kernels of the multi-GPU path are now
loaded (and the graphs instantiated) before any rank launches a kernel that waits for its peers (engine.hpp LocalGroup,
pdhg_kernels.cu preload_multi_gpu_kernels).  The check iterations run on the device, the only way tree mode runs them over
peer memory."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = os.path.join(ROOT, "tests", "logical_shards_child.py")

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("devcheck", [1], ids=["devcheck"])
@pytest.mark.parametrize("world,case,mode", [(2, "synthetic", "threads"), (3, "adlittle", "threads"), (4, "dense", "threads"),
                                             (2, "synthetic", "c_entry"), (2, "long_rows", "threads")])
def test_logical_shards(world, case, mode, devcheck):
    try:
        r = subprocess.run([sys.executable, CHILD, str(world), case, mode], capture_output=True, text=True, timeout=300, cwd=ROOT)
    except subprocess.TimeoutExpired:
        pytest.fail("logical-shard solve did not finish in 300 s (child killed)")
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert lines, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    out = json.loads(lines[-1])
    assert out["ok"] and out["ranks_identical"] and r.returncode == 0, (out.get("fails"), {k: out[k] for k in ("iters", "term", "obj", "ref_iters", "ref_obj")})
    assert out["term"][0] == out["ref_term"]
