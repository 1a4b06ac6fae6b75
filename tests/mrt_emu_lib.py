"""ctypes binding of the CPU development harness of the MRT joint controller (tests/emu/libmrtemu.so, built from tests/emu/mrt_emu.cu): the
kernel's __host__ __device__ phases (wb_mrt.cuh) executed on the host.  Test infrastructure only -- never linked into or called by the product
library."""
from __future__ import annotations

import ctypes as C

import numpy as np

from emu_build import build
from oracle_lib import F, _p

NX, NU, NJ = 58, 35, 23
_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build("mrt_emu.cu", "libmrtemu.so")))
    return _lib


def pad(a, width, fill=0.0):
    a = F(a)
    return np.ascontiguousarray(np.concatenate([a, np.full(a.shape[:-1] + (width - a.shape[-1],), fill)], axis=-1))


def joint_action(model, t, robot_state=None, x_obs=None, plan=None, K=None, fill=0.0):
    """wb_mrt.cuh's mrtJointAction on the CPU harness for one instance, arguments as mrt_ref.joint_action.  Centroidal state rows and gains are
    padded to the device layout with `fill`.  -> dict(x, u, q_des, qd_des, tau, mode, padding = the padded entries of the observation)"""
    from wb_humanoid_mpc_b200 import abi

    cen = model.get("kind") == "centroidal"
    nx = model["nx"]
    u8p = C.POINTER(C.c_uint8)
    args = [C.c_int(0), None, None, None, None, None, None]
    if plan is not None:
        tt, xx, uu = F(plan["t_nodes"]), pad(plan["x"], NX, fill), F(plan["u"])
        ev = np.ascontiguousarray(plan["node_event"], dtype=np.uint8)
        ct = np.ascontiguousarray(plan["contact_flags"], dtype=np.uint8)
        Kc = None
        if K is not None:   # [n-1][NX][NU] = column-major (NU x NX) per stage
            Kc = np.full((len(K), NX, NU), fill)
            Kc[:, :nx, :] = np.swapaxes(np.asarray(K), -1, -2)
            Kc = F(Kc)
        keep = (tt, xx, uu, ev, ct, Kc)
        args = [C.c_int(len(tt)), _p(tt), ev.ctypes.data_as(u8p), ct.ctypes.data_as(u8p), _p(xx), _p(uu), _p(Kc)]
    rs = None if robot_state is None else F(robot_state)
    xs = None if x_obs is None else pad(x_obs, NX, fill)
    q_des, qd_des, tau, xo, uo, mode = np.zeros(NJ), np.zeros(NJ), np.zeros(NJ), np.full(NX, np.nan), np.zeros(NU), np.zeros(1, dtype=np.int32)
    cd = C.byref(abi.cen_desc(model)) if cen else None
    rc = lib().emu_joint_action(C.byref(abi.model_desc(model)), cd, *args, C.c_int(int(plan is not None)), C.c_double(t), _p(rs), _p(xs), _p(q_des),
                                _p(qd_des), _p(tau), _p(xo), _p(uo), mode.ctypes.data_as(C.POINTER(C.c_int)))
    assert rc == 0
    if plan is not None:
        del keep
    return dict(x=xo[:nx].copy(), padding=xo[nx:].copy(), u=uo, q_des=q_des, qd_des=qd_des, tau=tau, mode=int(mode[0]))
