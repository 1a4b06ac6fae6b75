"""ctypes binding of the CPU development harness of the device-pointer I/O (tests/emu/libdevioemu.so, built from tests/emu/devio_emu.cu): the
robot-state check of b200sqp_joint_actions_dev (wb_devio.cuh) executed on the host.  Test infrastructure only -- never linked into or called
by the product library."""
from __future__ import annotations

import ctypes as C

import numpy as np

from emu_build import build

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build("devio_emu.cu", "libdevioemu.so")))
    return _lib


def robot_state_status(rows) -> np.ndarray:
    """wb_devio.cuh's mrtRobotStateStatus per row of rows [n, 13 + 2 nj] -> status [n]"""
    rows = np.ascontiguousarray(rows, dtype=np.float64)
    st = np.zeros(len(rows), dtype=np.int32)
    width = lib().emu_robot_state_status(rows.ctypes.data_as(C.POINTER(C.c_double)), C.c_int(len(rows)), st.ctypes.data_as(C.POINTER(C.c_int)))
    assert width == rows.shape[1], (width, rows.shape)
    return st
