"""Builds ``bevformer_b200/lib/libbevformer_b200.so`` with plain nvcc for sm_90a (H100; no torch headers).

The shared library is the product's only native artefact; it is built IN-TREE so that it travels to
the GPU box with the repo snapshot (it is git-ignored through ``*.so``).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libbevformer_b200.so")
STAMP = os.path.join(LIB_DIR, "build.stamp")
HEADER = os.path.join(os.path.dirname(HERE), "include", "bevformer_b200.h")   # the C ABI; _lib binds from it

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "--use_fast_math", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "-shared", "-Xptxas", "-v",
]
# --use_fast_math only changes division/transcendental lowering and ftz; the sampler uses neither
# division nor transcendentals on its value path, and the softmaxes, LayerNorm and point sampling use explicitly
# rounded operations (exp_rn, __frcp_rn, __frsqrt_rn, __fdiv_rn) where fp32 results must match the reference.


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest() -> str:
    h = hashlib.sha256()
    files = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC))
    files.append(HEADER)
    for f in files:
        with open(f, "rb") as fh:
            h.update(f.encode() + b"\0" + fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def nvcc_path() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; the bevformer_b200 CUDA library cannot be built")


def build(force: bool = False, verbose: bool = False) -> str:
    digest = _digest()
    if not force and os.path.exists(LIB_PATH) and os.path.exists(STAMP):
        with open(STAMP) as f:
            if f.read().strip() == digest:
                return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    cmd = [nvcc_path(), *NVCC_FLAGS, "-o", LIB_PATH, *sources()]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(LIB_DIR, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + log[-4000:])
    if verbose:
        print(log)
    with open(STAMP, "w") as f:
        f.write(digest)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
