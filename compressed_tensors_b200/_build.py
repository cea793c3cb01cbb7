"""
In-tree build of libct_b200.so (hand-written sm_90a kernels + C ABI) with nvcc.

    python -m compressed_tensors_b200._build [--force] [--verbose]

Each .cu is compiled to an object in csrc/build/ in parallel and linked into
compressed_tensors_b200/libct_b200.so.  nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "libct_b200.so")

SOURCES = [
    "runtime.cu",
    "generic.cu",
    "fp4.cu",
    "fast_fp4.cu",
    "convert.cu",
    "observe_channel.cu",
    "fast_pack.cu",
    "fast_quant.cu",
    "fast_fake.cu",
    "fake_heads.cu",
    "hadamard.cu",
    "dispatch.cu",
    "selftest.cu",
    "host_pipeline.cu",
    "sparse.cu",
    "bitmask_onepass.cu",
    "fast_sparse24q.cu",
    "observe_tensor.cu",
    "cpu_twin.cu",
    "fast_observe.cu",
    "dynamic_fake.cu",
    "observe_block_mx.cu",
]
HEADERS = sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + ["../../include/ct_b200.h"]   # every header: a stale object is a silent wrong build

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]   # H100 (Hopper); the kernels use sm_90a's TMA bulk copies and mbarriers

NVCC_FLAGS = [
    *ARCH,
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    # host code (the CPU twins of the ABI, cpu_twin.cu): OpenMP, and no fused multiply-add contraction -- every op rounds separately
    "-Xcompiler", "-fopenmp", "-Xcompiler", "-ffp-contract=off",
    "--expt-relaxed-constexpr",
    # parity: never let the compiler relax IEEE semantics
    "--fmad=true", "--prec-div=true", "--prec-sqrt=true", "--ftz=false",
]


def nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libct_b200.so cannot be built")


def _newest_header() -> float:
    return max(os.path.getmtime(os.path.join(CSRC, h)) for h in HEADERS)


def _compile(src: str, force: bool, verbose: bool) -> str:
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    srcp = os.path.join(CSRC, src)
    if not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(srcp), _newest_header()):
        return obj
    cmd = [nvcc(), *NVCC_FLAGS, "-c", srcp, "-o", obj]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    newest_src = max(max(os.path.getmtime(os.path.join(CSRC, s)) for s in SOURCES), _newest_header())
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= newest_src:
        return LIB
    with cf.ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
        objs = list(ex.map(lambda s: _compile(s, force, verbose), SOURCES))
    cmd = [nvcc(), "-shared", "-o", LIB, *objs, *ARCH, "-Xcompiler", "-fPIC", "-Xcompiler", "-fopenmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
