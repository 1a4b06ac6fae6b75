"""ctypes binding of the CPU oracle with the joint-torque cost (tests/oracle_jt/libjtoracle.so, built from tests/oracle_jt/jt_oracle.cpp on top of
oracle/capi.cpp), and the CPU harness of the device phases of the term (tests/emu/jt_emu.cu).  Test infrastructure only."""
from __future__ import annotations

import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np

import oracle_lib as orc
from emu_build import build as build_emu
from oracle_lib import F, _p

ROOT = Path(__file__).resolve().parents[1]
SRC = ROOT / "tests" / "oracle_jt" / "jt_oracle.cpp"
SO = ROOT / "tests" / "oracle_jt" / "libjtoracle.so"
NX, NU, NJ = 58, 35, 23
_lib = None
_emu = None


def build(force=False):
    deps = [SRC, *(ROOT / "oracle").glob("*.hpp"), *(ROOT / "oracle").glob("*.cpp"), *(ROOT / "oracle").glob("*.inc"), ROOT / "include" / "b200sqp.h"]
    if force or not SO.exists() or any(s.stat().st_mtime > SO.stat().st_mtime for s in deps):
        subprocess.run(["g++", "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-pthread", "-Wall", "-Wno-unused-parameter", "-DORC_WITH_WB", "-shared",
                        "-o", str(SO), str(SRC)], check=True, stdout=sys.stderr)
    return SO


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.orc_jt_create.restype = C.c_void_p
        _lib.orc_wb_total_mass.restype = C.c_double
        _lib.orc_wb_cost.restype = C.c_double
        _lib.orc_wb_cost_quad.restype = C.c_double
        _lib.orc_jt_residual.restype = C.c_int
    return _lib


class JtOracle(orc.WbOracle):
    """orc.WbOracle whose intermediate-node cost carries the joint-torque cost with weights w [nj] (None: the term is off)."""

    def __init__(self, model: dict, weights=None):
        from wb_humanoid_mpc_b200 import abi

        self.model = model
        self.desc = abi.model_desc(model)
        self.nx, self.nu, self.nj = model["nx"], model["nu"], model["nj"]
        self.L = lib()
        self._w = None if weights is None else F(weights)
        self.h = C.c_void_p(self.L.orc_jt_create(C.byref(self.desc), _p(self._w)))
        self.n_nodes = 0

    def torques(self, x, u):
        tau = np.zeros(self.nj)
        self.L.orc_jt_torques(self.h, _p(F(x)), _p(F(u)), _p(tau))
        return tau

    def residual(self, x, u):
        """r = sqrt(w) .* tau [nj] and J = dr/d(x, u) [nj][nx + nu]"""
        r, J = np.zeros(self.nj), np.zeros((self.nj, self.nx + self.nu))
        assert self.L.orc_jt_residual(self.h, _p(F(x)), _p(F(u)), _p(r), _p(J)) == 0
        return r, J


def solve(model, inst, settings, weights, keep_raw=False):
    """the oracle's SqpSolver on one instance (references.build_instance layout) with the joint-torque cost"""
    o = JtOracle(model, weights)
    o.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
    res = o.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], settings, keep_raw=keep_raw)
    if keep_raw:
        res["raw"] = o.last_raw_blocks(len(inst["t_nodes"]))
    return res


# ---- CPU harness of the device phases (wb_torque_cost.cuh) ----------------------------------------------------------------------------------
def emu():
    global _emu
    if _emu is None:
        _emu = C.CDLL(str(build_emu("jt_emu.cu", "libjtemu.so")))
    return _emu


def emu_node(model, weights, x, u, dt, Pu=None, Px=None, u0=None):
    """jtPhaseJacobian + jtPhaseRaw (+ jtPhaseProject / jtPhaseAccumulate when the projection Pu [NU][nut], Px [NU][NX], u0 [NU] is given) on the
    CPU, work items in reverse order.  -> dict(J, r, raw = the term's raw blocks (oracle layout, zero elsewhere), and with a projection
    Q, S [nut][NX], R, q, r_t, perf)"""
    from wb_humanoid_mpc_b200 import abi

    raw = np.zeros(2 * NX * NX + 2 * NX * NU + NU * NU + 2 * NX + NU + 1 + 14 * (NX + NU + 1) + 1)
    J, r = np.zeros((NX + NU, NJ)), np.zeros(NJ)
    nut = -1 if Pu is None else Pu.shape[1]
    Q, St, Rt, q, rt, perf = np.zeros((NX, NX)), np.zeros((NX, 23)), np.zeros((23, 23)), np.zeros(NX), np.zeros(23), np.zeros(4)
    Puc = None if Pu is None else F(np.pad(np.asarray(Pu), ((0, 0), (0, 23 - nut))).T)   # column-major NU x NUT_MAX
    Pxc = None if Px is None else F(np.asarray(Px).T)
    rc = emu().emu_jt_node(C.byref(abi.model_desc(model)), _p(F(weights)), _p(F(x)), _p(F(u)), C.c_double(dt), C.c_int(nut), _p(Puc), _p(Pxc),
                           _p(None if u0 is None else F(u0)), _p(J), _p(r), _p(raw), _p(Q), _p(St), _p(Rt), _p(q), _p(rt), _p(perf))
    assert rc == 0
    out = dict(J=J.T.copy(), r=r, raw=orc.unpack_raw_blocks(raw, NX, NU))
    if Pu is not None:   # St / Rt are column-major with ld NUT_MAX
        out.update(Q=Q.T.copy(), S=St.T[:nut].copy(), R=Rt.T[:nut, :nut].copy(), q=q, r_t=rt[:nut].copy(), perf=perf)
    return out
