"""ctypes binding of the CPU development harness of the device-pointer I/O (tests/emu/libdevioemu.so, built from tests/emu/devio_emu.cu): the
robot-state check of b200sqp_joint_actions_dev (wb_devio.cuh) executed on the host.  Test infrastructure only -- never linked into or called
by the product library."""
from __future__ import annotations

import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
EMU = ROOT / "tests" / "emu"
CSRC = ROOT / "wb_humanoid_mpc_b200" / "csrc"
_lib = None


def build(force=False):
    so = EMU / "libdevioemu.so"
    srcs = [EMU / "devio_emu.cu"] + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.inc")) + [ROOT / "include" / "b200sqp.h"]
    if force or not so.exists() or any(s.stat().st_mtime > so.stat().st_mtime for s in srcs):
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        subprocess.run([nvcc, "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                        "-diag-suppress", "177", "-o", str(so), str(EMU / "devio_emu.cu")], check=True)
    return so


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
    return _lib


def robot_state_status(rows) -> np.ndarray:
    """wb_devio.cuh's mrtRobotStateStatus per row of rows [n, 13 + 2 nj] -> status [n]"""
    rows = np.ascontiguousarray(rows, dtype=np.float64)
    st = np.zeros(len(rows), dtype=np.int32)
    width = lib().emu_robot_state_status(rows.ctypes.data_as(C.POINTER(C.c_double)), C.c_int(len(rows)), st.ctypes.data_as(C.POINTER(C.c_int)))
    assert width == rows.shape[1], (width, rows.shape)
    return st
