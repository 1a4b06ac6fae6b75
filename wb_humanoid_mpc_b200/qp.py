"""Host-side mirror of ocs2::HpipmInterface over the C ABI (batched).

Reference interface: lib/ocs2_ros2/ocs2_sqp/hpipm_catkin/include/hpipm_catkin/HpipmInterface.h
  resize(OcpSize) -> BatchedQp(batch, N, nx, nu_max)
  solve(x0, dynamics, cost, nullptr, x, u) -> solve(...)
  getRiccatiFeedback / getRiccatiFeedforward / getRiccatiCostToGo -> fields of the returned dict
Arrays use math layout [instance, stage, row, col]; conversion to the ABI's column-major records happens here.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import lib as _l


def _cm(M):
    return np.ascontiguousarray(np.swapaxes(M, -1, -2), dtype=np.float64)


def _p(a):
    return None if a is None else a.ctypes.data_as(_l.dp)


class BatchedQp:
    def __init__(self, batch: int, N: int, nx: int, nu_max: int, device: int = 0):
        self.batch, self.N, self.nx, self.nu_max = batch, N, nx, nu_max
        self._h = C.c_void_p()
        _l.check(_l.lib().b200sqp_qp_create(C.c_int(device), C.c_int(batch), C.c_int(N), C.c_int(nx), C.c_int(nu_max), C.byref(self._h)))

    def close(self):
        if self._h:
            _l.lib().b200sqp_qp_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def upload(self, A, B, b, Q, S, R, q, r, dx0, nu=None):
        Bn, N, nx, nm = self.batch, self.N, self.nx, self.nu_max
        assert A.shape == (Bn, N, nx, nx) and B.shape == (Bn, N, nx, nm) and Q.shape == (Bn, N + 1, nx, nx)
        assert S.shape == (Bn, N, nm, nx) and R.shape == (Bn, N, nm, nm) and q.shape == (Bn, N + 1, nx) and r.shape == (Bn, N, nm)
        f = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        self._keep = [_cm(A), _cm(B), f(b), _cm(Q), _cm(S), _cm(R), f(q), f(r), f(dx0)]
        nu_arr = None if nu is None else np.ascontiguousarray(nu, dtype=np.int32)
        _l.check(_l.lib().b200sqp_qp_upload(self._h, *[_p(a) for a in self._keep[:8]],
                                            None if nu_arr is None else nu_arr.ctypes.data_as(_l.ip), _p(self._keep[8])))

    def solve(self, reg_prim: float = 1e-12, keep_P: bool = True, stream=None):
        _l.check(_l.lib().b200sqp_qp_solve(self._h, C.c_double(reg_prim), C.c_int(int(keep_P)), C.c_void_p(stream or 0)))
        self._keptP = keep_P

    def last_ms(self) -> float:
        ms = C.c_float()
        _l.check(_l.lib().b200sqp_qp_last_ms(self._h, C.byref(ms)))
        return ms.value

    def download(self, raise_on_failure: bool = True):
        """A failed factorisation of some instance raises (B200SqpError -4) unless raise_on_failure = False, in which case the dict is returned
        with the per-instance `status` array (the arrays of the other instances are valid either way)."""
        Bn, N, nx, nm = self.batch, self.N, self.nx, self.nu_max
        dx, du = np.zeros((Bn, N + 1, nx)), np.zeros((Bn, N, nm))
        K, k = np.zeros((Bn, N, nx, nm)), np.zeros((Bn, N, nm))
        P = np.zeros((Bn, N + 1, nx, nx)) if self._keptP else None
        p = np.zeros((Bn, N + 1, nx)) if self._keptP else None
        status = np.zeros(Bn, dtype=np.int32)
        rc = _l.lib().b200sqp_qp_download(self._h, _p(dx), _p(du), _p(K), _p(k), _p(P), _p(p), status.ctypes.data_as(_l.ip))
        if rc != 0 and (raise_on_failure or rc != _l.EQP):   # EQP: every array has been filled, status says which instances failed
            _l.check(rc)
        out = dict(dx=dx, du=du, K=np.swapaxes(K, -1, -2).copy(), k=k, status=status)
        if self._keptP:
            out["P"] = np.swapaxes(P, -1, -2).copy()
            out["p"] = p
        return out
