"""Builds the sm_90a C-ABI library in-tree (tdmpc2_b200/libtdmpc2_b200.so).

nvcc cross-compiles without a GPU; the .so is git-ignored but travels with the
repo snapshot to the GPU box.  `python -m tdmpc2_b200.build` or
`__graft_entry__.build()` call this.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libtdmpc2_b200.so")
STAMP = LIB + ".stamp"
SOURCES = ["api.cu", "plan_kernels.cuh", "grad_kernels.cuh", "pixel_encoder.cuh", "pixel_grad_kernels.cuh", "buffer_kernels.cuh", "ptx.cuh", "rng.cuh",
           "draw_kernels.cuh", "model_file.cuh",
           os.path.join("..", "..", "include", "tdmpc2_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]


def _digest() -> str:
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for s in SOURCES:
        with open(os.path.join(CSRC, s), "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def find_nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found: cannot build libtdmpc2_b200.so")
    return cand


def up_to_date() -> bool:
    if not (os.path.exists(LIB) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() == _digest()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and up_to_date():
        return LIB
    cmd = [find_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["api.cu", "-o", LIB]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    with open(STAMP, "w") as f:
        f.write(_digest())
    return LIB


def build_variant(name: str, defines: list[str]) -> str:
    """Experiment build: libtdmpc2_b200_<name>.so with extra -D flags; load it through TDMPC2_B200_LIB."""
    out = os.path.join(HERE, f"libtdmpc2_b200_{name}.so")
    cmd = [find_nvcc()] + NVCC_FLAGS + [f"-D{d}" for d in defines] + ["api.cu", "-o", out]
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
