"""Builds one CPU development harness of tests/emu/ into a shared library with nvcc, when the library is missing or older than a source it
depends on: its own files and every product header.  Test infrastructure only."""
from __future__ import annotations

import shutil
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
EMU = ROOT / "tests" / "emu"
CSRC = ROOT / "wb_humanoid_mpc_b200" / "csrc"


def build(src, so, defines=(), deps=()):
    """tests/emu/<src> -> tests/emu/<so>, with -D<name> for every name in defines; deps: the harness files src includes"""
    src, so = EMU / src, EMU / so
    srcs = [src, *(EMU / d for d in deps), *CSRC.glob("*.cuh"), *CSRC.glob("*.inc"), ROOT / "include" / "b200sqp.h"]
    if not so.exists() or any(s.stat().st_mtime > so.stat().st_mtime for s in srcs):
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        subprocess.run([nvcc, "-O2", "-std=c++17", *(f"-D{d}" for d in defines), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler",
                        "-fPIC", "-Wno-deprecated-gpu-targets", "-diag-suppress", "177", "-o", str(so), str(src)], check=True)
    return so
