"""ctypes bindings of the CPU development harness (tests/emu/libwbemu.so): the CUDA kernels' __host__ __device__ phase functions
executed on the host.  Test infrastructure only -- never linked into or called by the product library."""
from __future__ import annotations

import ctypes as C

import numpy as np

from emu_build import build
from oracle_lib import F, _p, unpack_raw_blocks

_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build("wb_emu.cu", "libwbemu.so", defines=["EMU_WITH_LQ"], deps=["wb_emu_lq.inc", "cen_emu.inc"])))
    return _lib


class EmuNodeIn(C.Structure):
    _fields_ = [("x", C.POINTER(C.c_double)), ("u", C.POINTER(C.c_double)), ("xnext", C.POINTER(C.c_double)), ("xref", C.POINTER(C.c_double)),
                ("dt", C.c_double), ("contact", C.c_int * 2), ("swing", C.c_double * 6), ("impact", C.c_double * 2), ("armPhase", C.c_double)]


def dyn(desc, x, u, deriv=True):
    xd, G = np.zeros(58), np.zeros((93, 6))
    rc = lib().emu_dyn(C.byref(desc), _p(F(x)), _p(F(u)), _p(xd), _p(G), C.c_int(int(deriv)))
    assert rc == 0
    return xd, G.T.copy()


def penalty(kind, mu, delta, h):
    """(v, d1, d2) of the device's penRelaxed (kind "relaxed") or penPwPoly (kind "pwpoly") at h"""
    out = np.zeros(3)
    rc = lib().emu_penalty(C.c_int({"relaxed": 0, "pwpoly": 1}[kind]), C.c_double(mu), C.c_double(delta), C.c_double(h), _p(out))
    assert rc == 0
    return tuple(float(v) for v in out)


def lq_node(desc, x, u, xnext, xref, dt, contact, swing, impact, arm_phase, mode=0):
    """mode 0: one-pass K1b schedule; 1 / 2: the CUDA schedules (lu + part 1 + part 2; 2 = Q accumulated in place)."""
    NX, NU, NT = 58, 35, 23
    xs, us, xn, xr = F(x), F(u), F(xnext), F(xref)
    nin = EmuNodeIn(_p(xs), _p(us), _p(xn), _p(xr), dt, (C.c_int * 2)(*[int(c) for c in contact]), (C.c_double * 6)(*np.asarray(swing, float).reshape(6)),
                    (C.c_double * 2)(*impact), arm_phase)
    A, Bt, b = np.zeros((NX, NX)), np.zeros((NT, NX)), np.zeros(NX)
    Q, St, Rt, q, rt = np.zeros((NX, NX)), np.zeros((NX, NT)), np.zeros((NT, NT)), np.zeros(NX), np.zeros(NT)
    Pu, Px, u0 = np.zeros((NT, NU)), np.zeros((NX, NU)), np.zeros(NU)
    nut = C.c_int(0)
    perf = np.zeros(4)
    per = 2 * NX * NX + 2 * NX * NU + NU * NU + 2 * NX + NU + 1 + 14 * (NX + NU + 1) + 1
    raw = np.zeros(per)
    rc = lib().emu_lq_node_mode(C.byref(desc), C.byref(nin), _p(A), _p(Bt), _p(b), _p(Q), _p(St), _p(Rt), _p(q), _p(rt), _p(Pu), _p(Px), _p(u0),
                                C.byref(nut), _p(perf), _p(raw), C.c_int(mode))
    assert rc == 0
    n = nut.value
    return dict(A=A.T.copy(), B=Bt.T[:, :n].copy(), b=b, Q=Q.T.copy(), S=St.T[:n].copy(), R=Rt.T[:n, :n].copy(), q=q, r=rt[:n].copy(),
                Pu=Pu.T[:, :n].copy(), Px=Px.T.copy(), u0=u0, nut=n, perf=perf, raw=unpack_raw_blocks(raw, NX, NU))


def cen_node(desc, cdesc, x, u, xnext, xref, dt, contact, swing, impact, arm_phase):
    """One intermediate node of the centroidal path: cen_lq_kernel + cen_proj_kernel phase schedules on the host (padded QP record)."""
    NX, NU, NT, CX = 58, 35, 23, 35
    pad = lambda v: np.concatenate([F(v), np.zeros(NX - CX)])
    xs, us, xn, xr = pad(x), F(u), pad(xnext), pad(xref)
    nin = EmuNodeIn(_p(xs), _p(us), _p(xn), _p(xr), dt, (C.c_int * 2)(*[int(c) for c in contact]), (C.c_double * 6)(*np.asarray(swing, float).reshape(6)),
                    (C.c_double * 2)(*impact), arm_phase)
    A, Bt, b = np.zeros((NX, NX)), np.zeros((NT, NX)), np.zeros(NX)
    Q, St, Rt, q, rt = np.zeros((NX, NX)), np.zeros((NX, NT)), np.zeros((NT, NT)), np.zeros(NX), np.zeros(NT)
    Pu, Px, u0 = np.zeros((NT, NU)), np.zeros((NX, NU)), np.zeros(NU)
    nut = C.c_int(0)
    perf = np.zeros(4)
    per = 2 * CX * CX + 2 * CX * NU + NU * NU + 2 * CX + NU + 1 + 14 * (CX + NU + 1) + 1
    raw = np.zeros(per)
    rc = lib().emu_cen_node(C.byref(desc), C.byref(cdesc), C.byref(nin), _p(raw), _p(A), _p(Bt), _p(b), _p(Q), _p(St), _p(Rt), _p(q), _p(rt),
                            _p(Pu), _p(Px), _p(u0), C.byref(nut), _p(perf))
    assert rc == 0
    n = nut.value
    return dict(A=A.T.copy(), B=Bt.T[:, :n].copy(), b=b, Q=Q.T.copy(), S=St.T[:n].copy(), R=Rt.T[:n, :n].copy(), q=q, r=rt[:n].copy(),
                Pu=Pu.T[:, :n].copy(), Px=Px.T.copy(), u0=u0, nut=n, perf=perf, raw=unpack_raw_blocks(raw, CX, NU))


def cen_flow(desc, cdesc, x, u):
    """cen_flow_kernel's value lane (cenFlowDual) on the host: xdot of one centroidal (x, u)"""
    xd = np.zeros(35)
    rc = lib().emu_cen_flow(C.byref(desc), C.byref(cdesc), _p(F(x)), _p(F(u)), _p(xd))
    assert rc == 0
    return xd


def joint_torques(desc, x, u):
    tau, qddb = np.zeros(23), np.zeros(6)
    rc = lib().emu_joint_torques(C.byref(desc), _p(F(x)), _p(F(u)), _p(tau), _p(qddb))
    assert rc == 0
    return tau, qddb

