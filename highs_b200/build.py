"""Build libb200pdlp.so (the CUDA engine + C ABI) in-tree with nvcc for sm_90a (H100).

No CPU fallback is built: the library needs a CUDA device at run time.
    python -m highs_b200.build [--force] [--verbose]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200pdlp.so")
OBJ = os.path.join(HERE, "_build")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-fmad=false", "-Xcompiler", "-fPIC,-O2,-ffp-contract=off",
                     "-Xptxas", "-v", "--expt-relaxed-constexpr"]
CXX_FLAGS = ["-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-Wall", "-Wno-sign-compare"]

SOURCES = [("host_prep.cpp", "cxx"), ("host_prep_hipdlp.cpp", "cxx"), ("pdhg_kernels.cu", "nvcc"), ("setup_kernels.cu", "nvcc"), ("device_prep.cu", "nvcc"), ("kkt_check.cu", "nvcc"), ("kkt_batch.cu", "nvcc"), ("batch_kernels.cu", "nvcc"), ("batch_prep.cu", "nvcc"), ("batch_tree_prep.cu", "nvcc"), ("engine.cu", "nvcc"), ("engine_hipdlp.cu", "nvcc"), ("engine_batch.cu", "nvcc")]
HEADERS = ["host_prep.hpp", "kernels.cuh", "pdhg_arith.cuh", "pdhg_kernels.hpp", "batch_kernels.hpp", "batch_prep.hpp", "row_index.cuh", "hip_form.cuh", "kkt_batch.hpp", "setup_kernels.hpp", "device_prep.hpp", "kkt_logic.hpp", "engine.hpp", os.path.join("..", "..", "include", "b200pdlp.h")]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _newer(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


STAMP = os.path.join(OBJ, "flags.txt")
FLAGS = " ".join(NVCC_FLAGS + CXX_FLAGS)


def _flags_changed() -> bool:
    """True when the objects in _build/ were compiled with other flags (another architecture, say): mtimes alone would
    keep them."""
    return not os.path.exists(STAMP) or open(STAMP).read() != FLAGS


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    force = _flags_changed() or force
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    objs = []
    logs = []
    for src, kind in SOURCES:
        sp = os.path.join(CSRC, src)
        op = os.path.join(OBJ, src + ".o")
        objs.append(op)
        if not force and not _newer(op, [sp] + hdrs):
            continue
        cmd = ([_nvcc()] + NVCC_FLAGS if kind == "nvcc" else ["g++"] + CXX_FLAGS) + ["-c", sp, "-o", op]
        r = subprocess.run(cmd, capture_output=True, text=True)
        logs.append((src, r.stderr))
        if verbose or r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"compile failed: {' '.join(cmd)}")
    if force or _newer(LIB, objs):
        cmd = [_nvcc()] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    with open(STAMP, "w") as f:
        f.write(FLAGS)
    ptx = os.path.join(OBJ, "ptxas.log")
    if logs:
        with open(ptx, "w") as f:
            for src, err in logs:
                f.write(f"==== {src}\n{err}\n")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
