"""ctypes binding of the CPU development harness of the centroidal policy roll-out (tests/emu/libcensimemu.so, built from
tests/emu/cen_sim_emu.cu): the kernel's __host__ __device__ integrator (wb_sim.cuh, SimCenSystem) executed on the host.  Test infrastructure
only -- never linked into or called by the product library."""
from __future__ import annotations

import ctypes as C

import numpy as np

from emu_build import build
from oracle_lib import F, _p

NX, NU, CNX = 58, 35, 35
_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build("cen_sim_emu.cu", "libcensimemu.so")))
    return _lib


def pad(a, fill=0.0):
    """[..., CNX] -> [..., NX], the padding set to `fill` (zero on the device; NaN proves that it is never read)"""
    a = F(a)
    return np.ascontiguousarray(np.concatenate([a, np.full(a.shape[:-1] + (NX - CNX,), fill)], axis=-1))


def rollout_policy(model, plan, t, duration, x_start, K=None, settings=None, fill=0.0):
    """the centroidal policy roll-out of wb_sim.cuh on the CPU harness for one instance.  plan = dict(t_nodes, node_event, contact_flags,
    x [n, 35], u [n-1, 35]); K [n-1, 35, 35] or None (feed-forward).  The state rows and the gains are padded to the device layout with `fill`.
    -> dict(x [35], u, mode, accepted, rejected, calls, status, padding = the 23 padded entries of the output state)"""
    from wb_humanoid_mpc_b200 import abi

    rs = settings if settings is not None else abi.cen_default_rollout_settings()
    u8p = C.POINTER(C.c_uint8)
    tt, xx, uu = F(plan["t_nodes"]), pad(plan["x"], fill), F(plan["u"])
    ev = np.ascontiguousarray(plan["node_event"], dtype=np.uint8)
    ct = np.ascontiguousarray(plan["contact_flags"], dtype=np.uint8)
    Kc = None
    if K is not None:   # [n-1][NX][NU] = column-major (NU x NX) per stage, columns 35.. the padding
        Kc = np.full((len(K), NX, NU), fill)
        Kc[:, :CNX, :] = np.swapaxes(np.asarray(K), -1, -2)
        Kc = F(Kc)
    xe, ue, info = np.full(NX, np.nan), np.zeros(NU), np.zeros(5, dtype=np.int32)
    rc = lib().emu_cen_rollout_policy(C.byref(abi.model_desc(model)), C.byref(abi.cen_desc(model)), C.c_int(len(tt)), _p(tt), ev.ctypes.data_as(u8p),
                                      ct.ctypes.data_as(u8p), _p(xx), _p(uu), _p(Kc), C.byref(rs), C.c_double(t), C.c_double(t + duration),
                                      _p(pad(x_start, fill)), _p(xe), _p(ue), info.ctypes.data_as(C.POINTER(C.c_int)))
    assert rc == 0
    return dict(x=xe[:CNX].copy(), padding=xe[CNX:].copy(), u=ue, status=int(info[0]), accepted=int(info[1]), rejected=int(info[2]), calls=int(info[3]),
                mode=int(info[4]))
