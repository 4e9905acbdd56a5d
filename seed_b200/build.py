"""Build libseedb200.so (sm_90a, H100) and the C oracle, in-tree.

nvcc cross-compiles without a GPU.  `python -m seed_b200.build [--force]` or `__graft_entry__.build()`.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(ROOT)
CSRC = os.path.join(ROOT, "csrc")
OBJ = os.path.join(ROOT, "_build")
LIB = os.path.join(ROOT, "libseedb200.so")
ORACLE_DIR = os.path.join(REPO, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "libvq_oracle.so")

SOURCES = ["capi.cu", "gemm_wgmma.cu", "attention.cu", "rowwise.cu", "vq.cu", "misc.cu", "sampler.cu", "encoder.cu", "llama.cu", "preprocess.cu", "int8.cu", "beam.cu", "lora.cu", "quant4.cu", "contrastive.cu"]
HEADERS = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "int8.cuh"), os.path.join(CSRC, "quant4.cuh"), os.path.join(CSRC, "wgmma.cuh"), os.path.join(CSRC, "select.cuh"), os.path.join(CSRC, "ops.h"), os.path.join(REPO, "include", "seedb200.h")]

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _newer(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps)


def _run(cmd: list[str], log: str | None = None) -> None:
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log:
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + p.stdout)
    if p.returncode != 0:
        sys.stderr.write(p.stdout)
        raise RuntimeError("command failed: " + " ".join(cmd))


def build_cuda(force: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    jobs = []
    objs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or not _newer(obj, [src] + HEADERS):
            jobs.append((NVCC_FLAGS_CMD(src, obj), obj + ".log"))
    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(lambda j: _run(*j), jobs))
    if force or jobs or not _newer(LIB, objs):
        _run([NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    return LIB


def NVCC_FLAGS_CMD(src: str, obj: str) -> list[str]:
    return [NVCC] + NVCC_FLAGS + ["-c", src, "-o", obj]


def build_oracle(force: bool = False) -> str:
    srcs = [os.path.join(ORACLE_DIR, "vq_oracle.c"), os.path.join(ORACLE_DIR, "resize_oracle.c")]
    if force or not _newer(ORACLE_LIB, srcs):
        # -ffp-contract=off: the oracle's arithmetic is pinned operation by operation
        _run(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", ORACLE_LIB] + srcs + ["-lm"])
    return ORACLE_LIB


def build(force: bool = False) -> None:
    build_cuda(force)
    build_oracle(force)


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    print("built", LIB, "and", ORACLE_LIB)
