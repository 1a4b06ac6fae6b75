"""Host-side mirror of ocs2::SqpSolver for a batch of whole-body MPC instances, over the C ABI (no torch types involved).

Reference interface: lib/ocs2_ros2/ocs2_sqp/ocs2_sqp/include/ocs2_sqp/SqpSolver.h:60-103
    SqpSolver(settings, optimalControlProblem, initializer)  -> B200SqpSolver(model, settings)
    run(initTime, initState, initMode, finalTime)            -> run(instances)   (instances built by references.build_instance)
    primalSolution(finalTime)                                -> primal_solution()
    getIterationsLog()                                       -> iterations_log()
    getBenchmarks()                                          -> benchmarks()
Error behaviour follows the reference: a failed QP raises (SqpSolver.cpp:306-308 throws std::runtime_error).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi
from . import lib as _l

LOG_FIELDS = ["base_merit", "base_cost", "base_dyn_sse", "base_eq_sse", "merit", "cost", "dyn_sse", "eq_sse", "step_size", "step_type",
              "dx_norm", "du_norm", "armijo", "convergence"]


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _p(a):
    return a.ctypes.data_as(_l.dp)


def stack_instances(instances: list[dict]) -> dict:
    """list of per-instance dicts (references.build_instance) -> batched arrays; all instances must share the node count."""
    n = {len(i["t_nodes"]) for i in instances}
    if len(n) != 1:
        raise ValueError(f"instances of one batch must have the same number of shooting nodes, got {sorted(n)}")
    keys = ["x0", "x_init", "u_init", "t_nodes", "node_event", "contact_flags", "swing_ref", "impact_factor", "arm_phase", "x_ref"]
    return {k: np.stack([np.asarray(i[k]) for i in instances]) for k in keys}


class B200SqpSolver:
    def __init__(self, model: dict, settings: abi.Settings | None = None, device: int = 0, capture_raw_blocks: bool = False):
        self.model = model
        self.nx, self.nu = model["nx"], model["nu"]
        self.settings = settings if settings is not None else abi.default_settings(model)
        self._desc = abi.model_desc(model)
        self._h = C.c_void_p()
        L = _l.lib()
        if model.get("kind") == "centroidal":   # CentroidalMpcInterface OCP: same solver interface, nx = nu = 12 + nj at the ABI
            self._cdesc = abi.cen_desc(model)
            _l.check(L.b200sqp_cen_create(C.byref(self._desc), C.byref(self._cdesc), C.byref(self.settings), C.c_int(device), C.byref(self._h)))
        else:
            _l.check(L.b200sqp_create(C.byref(self._desc), C.byref(self.settings), C.c_int(device), C.byref(self._h)))
        self._raw_per = 0
        if capture_raw_blocks:
            per = C.c_int64()
            _l.check(L.b200sqp_stage_doubles(self._h, C.c_int(0), C.byref(per)))
            self._raw_per = per.value
        self.batch = self.n_nodes = 0
        self._nccl = self._comm = None

    # -- global-step mode (SURVEY.md section 8e) --------------------------------------------------------------------------------
    def enable_global_step(self):
        """Cross-rank global-step mode (settings.global_step must be 1): hands the library an NCCL communicator of this rank
        (b200sqp_set_comm); the all-reduces of the per-candidate statistics then run INSIDE b200sqp_solve on its stream, exactly as for a C++
        host.  The communicator is created here with ncclCommInitRank (ctypes on the process' libnccl.so.2), its unique id broadcast through
        torch.distributed, which is only the bootstrap plumbing.  Without an initialised process group (or world size 1) nothing is
        registered: the local statistics decide."""
        import torch
        import torch.distributed as dist

        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return
        world, rank = dist.get_world_size(), dist.get_rank()
        nccl = C.CDLL("libnccl.so.2")   # the copy torch already loaded (same soname)

        class UniqueId(C.Structure):
            _fields_ = [("internal", C.c_byte * 128)]

        uid = UniqueId()
        if rank == 0:
            rc = nccl.ncclGetUniqueId(C.byref(uid))
            assert rc == 0, f"ncclGetUniqueId failed ({rc})"
        t = torch.frombuffer(bytearray(bytes(uid)), dtype=torch.uint8).clone()
        dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
        t = t.to(dev)
        dist.broadcast(t, src=0)
        C.memmove(C.byref(uid), bytes(t.cpu().numpy().tobytes()), 128)
        comm = C.c_void_p()
        nccl.ncclCommInitRank.argtypes = [C.POINTER(C.c_void_p), C.c_int, UniqueId, C.c_int]
        rc = nccl.ncclCommInitRank(C.byref(comm), world, uid, rank)
        assert rc == 0, f"ncclCommInitRank failed ({rc})"
        self._nccl, self._comm = nccl, comm
        _l.check(_l.lib().b200sqp_set_comm(self._h, comm, C.c_int(world)))

    def global_stats(self):
        """(statistics [n_evaluated, 4] = {#accept, sum of merits, max violation, #active} over all ranks, index of the applied candidate or -1)
        of the last iteration of the last solve in the global-step mode"""
        st = np.zeros((32, 4))
        n, ch = C.c_int32(), C.c_int32()
        _l.check(_l.lib().b200sqp_global_stats(self._h, _p(st), C.byref(n), C.byref(ch)))
        return st[: n.value].copy(), ch.value

    def global_ladder(self) -> np.ndarray:
        a = np.zeros(32)
        n = C.c_int32()
        _l.check(_l.lib().b200sqp_global_ladder(self._h, _p(a), C.byref(n)))
        return a[: n.value]

    def close(self):
        if self._h:
            _l.lib().b200sqp_destroy(self._h)
            self._h = C.c_void_p()
        if getattr(self, "_comm", None):
            self._nccl.ncclCommDestroy(self._comm)
            self._comm = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- SolverBase::run ------------------------------------------------------------------------------------------------
    def upload(self, batch: dict):
        B, n = batch["t_nodes"].shape
        if (B, n) != (self.batch, self.n_nodes):
            _l.check(_l.lib().b200sqp_set_batch(self._h, C.c_int(B), C.c_int(n)))
            self.batch, self.n_nodes = B, n
        u8 = lambda a: np.ascontiguousarray(a, dtype=np.uint8)
        self._keep = [_f(batch["x0"]), _f(batch["x_init"]), _f(batch["u_init"]), _f(batch["t_nodes"]), u8(batch["node_event"]),
                      u8(batch["contact_flags"]), _f(batch["swing_ref"]), _f(batch["impact_factor"]), _f(batch["arm_phase"]), _f(batch["x_ref"])]
        k = self._keep
        _l.check(_l.lib().b200sqp_upload_instances(self._h, _p(k[0]), _p(k[1]), _p(k[2]), _p(k[3]), k[4].ctypes.data_as(_l.u8p),
                                                   k[5].ctypes.data_as(_l.u8p), _p(k[6]), _p(k[7]), _p(k[8]), _p(k[9])))

    def build_instances(self, t0: float, horizon: float, x0, gaits, gait_start, cmd, warm: bool | str = False) -> int:
        """Device-side instance builder (b200sqp_build_instances): one synchronous MPC cycle of len(x0) instances over [t0, t0 + horizon] from
        x0 [B, nx], gait names (or ids) [B], gait start times [B] and velocity commands [B, 4]; warm = shift the iterate left on the device by
        the previous solve; x0 = None (with warm): the planned state at t0 is the measured state (closed loop on the device); warm = "rollout"
        (x0 = None): warm start whose measured state is the simulated state of the last roll-out (rollout_policy on a whole-body model,
        cen_rollout_policy on a centroidal one).  On a centroidal model x0 is [B, 35] and the targets follow the centroidal rule.  Returns the
        common number of shooting nodes."""
        if warm == "rollout":
            if x0 is not None:
                raise ValueError('warm="rollout" takes the measured state from the last roll-out; pass x0=None')
            warm = 2
        elif isinstance(warm, str):
            raise ValueError(f"warm must be a bool or 'rollout', got {warm!r}")
        L = _l.lib()
        if not getattr(self, "_builder_set", False):
            self._bdesc, self._gait_names = abi.builder_desc(self.model)
            _l.check(L.b200sqp_set_builder(self._h, C.byref(self._bdesc)))
            self._builder_set = True
        if x0 is None:
            B = len(gaits)
        else:
            x0 = _f(x0)
            B = x0.shape[0]
        gid = np.ascontiguousarray([g if isinstance(g, (int, np.integer)) else self._gait_names.index(g) for g in gaits], dtype=np.int32)
        gs, cm = _f(gait_start), _f(cmd)
        assert gid.shape == (B,) and gs.shape == (B,) and cm.shape == (B, 4)
        n = C.c_int32()
        _l.check(L.b200sqp_build_instances(self._h, C.c_int(B), C.c_double(t0), C.c_double(horizon), None if x0 is None else _p(x0), gid.ctypes.data_as(_l.ip), _p(gs), _p(cm),
                                           C.c_int(int(warm)), C.byref(n)))
        self.batch, self.n_nodes = B, n.value
        return n.value

    def set_gait_schedule(self, stateful: bool = True, phase_transition_stance_time: float = 0.0):
        """b200sqp_set_gait_schedule: stateful = True keeps every instance's gait schedule on the device across cycles; the gaits passed to a
        warm build_instances are then per-instance gait commands (a changed one runs the reference's updateGaitSchedule, visible in the next
        cycle's schedule), and the warm start is spread over the new schedule.  Takes effect at the next cold build."""
        _l.check(_l.lib().b200sqp_set_gait_schedule(self._h, C.c_int(int(stateful)), C.c_double(phase_transition_stance_time)))

    def mode_schedule(self, max_events: int = 192) -> list:
        """the window mode schedule of every instance that the last build_instances used: [(event_times, mode_sequence)] * B"""
        B = self.batch
        ev, modes, n = np.zeros((B, max_events)), np.zeros((B, max_events + 1), dtype=np.int32), np.zeros(B, dtype=np.int32)
        _l.check(_l.lib().b200sqp_download_mode_schedule(self._h, C.c_int(max_events), _p(ev), modes.ctypes.data_as(_l.ip), n.ctypes.data_as(_l.ip)))
        return [(ev[b, : n[b]].tolist(), modes[b, : n[b] + 1].tolist()) for b in range(B)]

    def download_instances(self) -> dict:
        """the per-instance inputs as they lie on the device (b200sqp_download_instances), in the layout of stack_instances"""
        B, n, nx, nu = self.batch, self.n_nodes, self.nx, self.nu
        out = dict(x0=np.zeros((B, nx)), x_init=np.zeros((B, n, nx)), u_init=np.zeros((B, n - 1, nu)), t_nodes=np.zeros((B, n)),
                   node_event=np.zeros((B, n), dtype=np.uint8), contact_flags=np.zeros((B, n, 2), dtype=np.uint8), swing_ref=np.zeros((B, n, 2, 3)),
                   impact_factor=np.zeros((B, n, 2)), arm_phase=np.zeros((B, n)), x_ref=np.zeros((B, n, nx)))
        u8 = lambda a: a.ctypes.data_as(_l.u8p)
        _l.check(_l.lib().b200sqp_download_instances(self._h, _p(out["x0"]), _p(out["x_init"]), _p(out["u_init"]), _p(out["t_nodes"]), u8(out["node_event"]),
                                                     u8(out["contact_flags"]), _p(out["swing_ref"]), _p(out["impact_factor"]), _p(out["arm_phase"]),
                                                     _p(out["x_ref"])))
        return out

    def reset(self):
        """SqpSolver::reset(): restore the uploaded initial guess on the device"""
        _l.check(_l.lib().b200sqp_reset(self._h))

    def solve(self, stream=None, wait: bool = True):
        """b200sqp_solve enqueues the whole solve and returns; wait = True (default) then blocks in b200sqp_wait like the reference's synchronous
        run(); wait = False leaves the work in flight (call wait() or read results later)"""
        _l.check(_l.lib().b200sqp_solve(self._h, C.c_void_p(stream or 0)))
        if wait:
            self.wait()

    def wait(self):
        _l.check(_l.lib().b200sqp_wait(self._h))

    def rollout_policy(self, t: float, duration: float, x_start=None, settings: abi.RolloutSettings | None = None, stream=None) -> dict:
        """MRT_BASE::rolloutPolicy for every instance (b200sqp_rollout_policy): simulate from time t for `duration` seconds under the policy of
        the last solve (feedback when settings.use_feedback_policy = 1) with the ODE45 roll-out.  x_start [B, nx], or None for the current
        measured state.  Waits for the result and returns {x [B, nx], u [B, nu], mode [B], n_steps [B, 3] (accepted, rejected, flow-map
        calls), status [B]}; the simulated state also stays on the device for build_instances(..., warm="rollout")."""
        return self._rollout(_l.lib().b200sqp_rollout_policy, t, duration, x_start, settings if settings is not None else abi.default_rollout_settings(), stream)

    def cen_rollout_policy(self, t: float, duration: float, x_start=None, settings: abi.RolloutSettings | None = None, stream=None) -> dict:
        """rollout_policy on a centroidal model (b200sqp_cen_rollout_policy): the ODE45 roll-out of the centroidal flow map under the policy of
        the last solve, by default with the centroidal task.info settings (abi.cen_default_rollout_settings).  x_start [B, 35] or None; returns
        the dict of rollout_policy with x [B, 35]; the simulated state stays on the device for build_instances(..., warm="rollout")."""
        return self._rollout(_l.lib().b200sqp_cen_rollout_policy, t, duration, x_start, settings if settings is not None else abi.cen_default_rollout_settings(), stream)

    def _rollout(self, fn, t, duration, x_start, rs, stream):
        B, nx, nu = self.batch, self.nx, self.nu
        xs = None if x_start is None else _f(x_start)
        if xs is not None:
            assert xs.shape == (B, nx), xs.shape
        out = dict(x=np.zeros((B, nx)), u=np.zeros((B, nu)), mode=np.zeros(B, dtype=np.int32), n_steps=np.zeros((B, 3), dtype=np.int32),
                   status=np.zeros(B, dtype=np.int32))
        _l.check(fn(self._h, C.c_double(t), C.c_double(duration), None if xs is None else _p(xs), C.byref(rs), _p(out["x"]), _p(out["u"]),
                    out["mode"].ctypes.data_as(_l.ip), out["n_steps"].ctypes.data_as(_l.ip), out["status"].ctypes.data_as(_l.ip), C.c_void_p(stream or 0)))
        self.wait()
        return out

    def run(self, instances):
        batch = stack_instances(instances) if isinstance(instances, list) else instances
        self.upload(batch)
        self.solve()
        return self.primal_solution()

    # -- results -------------------------------------------------------------------------------------------------------------
    def primal_solution(self, with_gains: bool | None = None, out: dict | None = None, raise_on_failure: bool = True):
        """out = {"x": [B, n, nx], "u": [B, n-1, nu]} lets the caller supply (page-locked) destination arrays for the download.
        A failed QP of some instance raises like the reference (SqpSolver.cpp:306-308) unless raise_on_failure = False, in which case the dict
        is returned with the per-instance `status` array (the arrays of the other instances are valid either way)."""
        B, n, nx, nu = self.batch, self.n_nodes, self.nx, self.nu
        if out is not None:
            x, u = out["x"], out["u"]
            assert x.shape == (B, n, nx) and u.shape == (B, n - 1, nu) and x.flags.c_contiguous and u.flags.c_contiguous
        else:
            x, u = np.zeros((B, n, nx)), np.zeros((B, n - 1, nu))
        with_gains = bool(self.settings.use_feedback_policy) if with_gains is None else with_gains
        K = np.zeros((B, n - 1, nx, nu)) if with_gains else None
        log = (abi.IterLog * (B * self.settings.sqp_iteration))()
        n_iter, status = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        rc = _l.lib().b200sqp_download(self._h, _p(x), _p(u), None if K is None else _p(K), log, n_iter.ctypes.data_as(_l.ip),
                                       status.ctypes.data_as(_l.ip))
        if rc != 0 and (raise_on_failure or rc != -4):   # -4 = B200SQP_EQP: every array has been filled, status says which instances failed
            _l.check(rc)
        logs = np.frombuffer(log, dtype=np.float64).reshape(B, self.settings.sqp_iteration, 16).copy()
        out = dict(x=x, u=u, n_iter=n_iter, status=status, log=logs)
        if K is not None:
            out["K"] = np.swapaxes(K, -1, -2).copy()
        return out

    def value_function(self):
        """getValueFunction data: (P [B, n, nx, nx], p [B, n, nx]) of the last iteration (needs settings.create_value_function)"""
        B, n, nx = self.batch, self.n_nodes, self.nx
        P, p = np.zeros((B, n, nx, nx)), np.zeros((B, n, nx))
        _l.check(_l.lib().b200sqp_download_value_function(self._h, _p(P), _p(p)))
        return np.swapaxes(P, -1, -2).copy(), p

    def iterations_log(self):
        return self.primal_solution(with_gains=False)["log"]

    def raw_stage_blocks(self):
        """(B, N, per) raw pre-projection blocks of the last LQ approximation (needs capture_raw_blocks=True)."""
        B, N = self.batch, self.n_nodes - 1
        out = np.zeros((B, N, self._raw_per))
        _l.check(_l.lib().b200sqp_download_stage_blocks(self._h, C.c_int(0), _p(out), C.c_int64(out.size)))
        return out

    def benchmarks(self):
        """device milliseconds of {LQ approximation, solve QP, line search, compute controller} of the last solve"""
        ms = (C.c_float * 4)()
        _l.check(_l.lib().b200sqp_get_stage_times(self._h, ms))
        return list(ms)

    def launch_count(self) -> int:
        n = C.c_int64()
        _l.check(_l.lib().b200sqp_get_launch_count(self._h, C.byref(n)))
        return n.value


def joint_torques(model: dict, x, u, device: int = 0):
    """computeJointTorques for whole-body samples through the C ABI (b200sqp_joint_torques): x [..., nx], u [..., nu] -> (tau [..., nj],
    qddb [..., 6]); e.g. x = sol["x"][:, :-1], u = sol["u"] of a batch of primal solutions."""
    x, u = _f(x), _f(u)
    lead = x.shape[:-1]
    n = int(np.prod(lead)) if lead else 1
    desc = abi.model_desc(model)
    tau, qddb = np.zeros((n, model["nj"])), np.zeros((n, 6))
    _l.check(_l.lib().b200sqp_joint_torques(C.byref(desc), C.c_int(n), _p(x.reshape(n, -1)), _p(u.reshape(n, -1)), _p(tau), _p(qddb), C.c_int(device)))
    return tau.reshape(*lead, -1), qddb.reshape(*lead, 6)
