"""ctypes binding of the CPU development harness of the policy roll-out (tests/emu/libsimemu.so, built from tests/emu/sim_emu.cu): the kernel's
__host__ __device__ integrator (wb_sim.cuh) executed on the host.  Test infrastructure only -- never linked into or called by the product library."""
from __future__ import annotations

import ctypes as C

import numpy as np

from emu_build import build
from oracle_lib import F, _p

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build("sim_emu.cu", "libsimemu.so")))
    return _lib


def rollout_policy(desc, plan, t, duration, x_start, K=None, settings=None):
    """the policy roll-out of wb_sim.cuh (simRollout) on the CPU harness for one instance.  plan = dict(t_nodes, node_event, contact_flags, x [n, nx],
    u [n-1, nu]); K [n-1, nu, nx] or None (feed-forward) -> dict(x, u, mode, accepted, rejected, calls, status)"""
    from wb_humanoid_mpc_b200 import abi

    rs = settings if settings is not None else abi.default_rollout_settings()
    u8p = C.POINTER(C.c_uint8)
    tt, xx, uu = F(plan["t_nodes"]), F(plan["x"]), F(plan["u"])
    ev = np.ascontiguousarray(plan["node_event"], dtype=np.uint8)
    ct = np.ascontiguousarray(plan["contact_flags"], dtype=np.uint8)
    Kc = None if K is None else F(np.swapaxes(np.asarray(K), -1, -2))   # [n-1][nx][nu] = column-major (nu x nx) per stage
    xe, ue, info = np.zeros(58), np.zeros(35), np.zeros(5, dtype=np.int32)
    rc = lib().emu_rollout_policy(C.byref(desc), C.c_int(len(tt)), _p(tt), ev.ctypes.data_as(u8p), ct.ctypes.data_as(u8p), _p(xx), _p(uu), _p(Kc), C.byref(rs),
                                  C.c_double(t), C.c_double(t + duration), _p(F(x_start)), _p(xe), _p(ue), info.ctypes.data_as(C.POINTER(C.c_int)))
    assert rc == 0
    return dict(x=xe, u=ue, status=int(info[0]), accepted=int(info[1]), rejected=int(info[2]), calls=int(info[3]), mode=int(info[4]))
