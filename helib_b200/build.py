"""Build helib_b200/libhelib_b200.so in-tree with nvcc for sm_90a (H100)."""
from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["csrc/hb_engine.cu", "csrc/hb_chain.cpp"]
DEPS = ["csrc/hb_engine.cu", "csrc/hb_device.cuh", "csrc/hb_device_v1.cuh", "csrc/hb_device_v2.cuh", "csrc/hb_device_gen.cuh", "csrc/hb_device_prg.cuh", "csrc/hb_chain.cpp", "../include/helib_b200.h", "../include/helib_b200_chain.h"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libhelib_b200.so")


def build_library(force: bool = False, verbose: bool = False) -> str:
    out = os.path.join(_HERE, "libhelib_b200.so")
    deps = [os.path.join(_HERE, d) for d in DEPS]
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + [os.path.join(_HERE, s) for s in SOURCES]
    subprocess.check_call(cmd)
    return out
