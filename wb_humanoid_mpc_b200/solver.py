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
import weakref

import numpy as np

from . import abi
from . import lib as _l

LOG_FIELDS = ["base_merit", "base_cost", "base_dyn_sse", "base_eq_sse", "merit", "cost", "dyn_sse", "eq_sse", "step_size", "step_type",
              "dx_norm", "du_norm", "armijo", "convergence"]


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _p(a):
    return a.ctypes.data_as(_l.dp)


def _build_args(x0, gaits, gait_start, cmd, names):
    """batch size and the int / double arrays of a build; gaits = None (warm builds with a motion manager) passes NULL"""
    B = len(cmd) if x0 is None else np.asarray(x0).shape[0]
    gid = None if gaits is None else np.ascontiguousarray([g if isinstance(g, (int, np.integer)) else names.index(g) for g in gaits], dtype=np.int32)
    gs, cm = _f(gait_start), _f(cmd)
    assert (gid is None or gid.shape == (B,)) and gs.shape == (B,) and cm.shape == (B, 4)
    return B, gid, gs, cm


def _motion_state(fn, h, B):
    st, lc, fc = np.zeros(B, dtype=np.int32), np.zeros(B), np.zeros((B, 4))
    _l.check(fn(h, st.ctypes.data_as(_l.ip), _p(lc), _p(fc)))
    return dict(state=st, gait=[abi.MOTION_GAITS[s] for s in st], last_change=lc, filtered_cmd=fc)


def _set_reset_states(fn, h, x0, gaits, offsets, names):
    x0 = _f(x0)
    B = x0.shape[0]
    gid = np.ascontiguousarray([g if isinstance(g, (int, np.integer)) else names.index(g) for g in gaits], dtype=np.int32)
    off = _f(np.zeros(B) if offsets is None else offsets)
    assert gid.shape == (B,) and off.shape == (B,)
    _l.check(fn(h, C.c_int(B), _p(x0), gid.ctypes.data_as(_l.ip), _p(off)))
    return B


def _request_resets(fn, h, indices):
    idx = np.ascontiguousarray(np.atleast_1d(indices), dtype=np.int32)
    _l.check(fn(h, C.c_int(idx.size), idx.ctypes.data_as(_l.ip)))


def _episodes(fn, h, B):
    if not B:
        raise RuntimeError("episodes: no reset states (set_reset_states first)")
    ep, st, rs, rst, ll = np.zeros(B, dtype=np.int32), np.zeros(B), np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.uint8), np.zeros(B)
    _l.check(fn(h, ep.ctypes.data_as(_l.ip), _p(st), rs.ctypes.data_as(_l.ip), rst.ctypes.data_as(_l.u8p), _p(ll)))
    return dict(episode=ep, start=st, reason=rs, reason_name=[abi.RESET_REASONS[r] for r in rs], reset=rst.astype(bool), last_length=ll)


def _command_poses(fn, h, indices, deltas):
    idx = np.ascontiguousarray(np.atleast_1d(indices), dtype=np.int32)
    d = np.ascontiguousarray(np.asarray(deltas, dtype=np.float64).reshape(idx.size, 4))
    _l.check(fn(h, C.c_int(idx.size), idx.ctypes.data_as(_l.ip), _p(d)))


def _pose_targets(fn, h, B):
    act, ts, tr, tp, err = np.zeros(B, dtype=np.int32), np.zeros(B), np.zeros(B), np.zeros((B, 6)), np.zeros((B, 2))
    _l.check(fn(h, act.ctypes.data_as(_l.ip), _p(ts), _p(tr), _p(tp), _p(err)))
    return dict(active=act.astype(bool), t_start=ts, t_reach=tr, target_pose=tp, error=err)


def _is_cuda_tensor(a) -> bool:
    return getattr(a, "is_cuda", False) is True


def check_device_tensor(t, name: str, device, dtype, shape):
    """The checks of a device-pointer argument, before any ABI call: a torch tensor on `device` of `dtype`, with `shape`, C-contiguous.
    Raises ValueError naming the argument."""
    import torch

    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name}: expected a torch tensor, got {type(t).__name__}")
    if t.device != torch.device(device):
        raise ValueError(f"{name}: the tensor is on {t.device}, the handle on {torch.device(device)}")
    if t.dtype != dtype:
        raise ValueError(f"{name}: dtype {t.dtype}, expected {dtype}")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name}: shape {tuple(t.shape)}, expected {tuple(shape)}")
    if not t.is_contiguous():
        raise ValueError(f"{name}: the tensor is not C-contiguous")
    return t


def _vp(t):
    return C.c_void_p(None if t is None else t.data_ptr())


def _stream(device, stream) -> C.c_void_p:
    """stream = None: the current torch stream of the handle's device; a torch.cuda.Stream or a raw cudaStream_t (int) otherwise"""
    import torch

    if stream is None:
        stream = torch.cuda.current_stream(device)
    return C.c_void_p(getattr(stream, "cuda_stream", stream) or 0)


def _device_outputs(device, specs: dict, out: dict | None) -> dict:
    """specs {name: (shape, dtype)} -> the caller's tensors (checked) or new ones"""
    import torch

    if out is None:
        return {k: torch.empty(shape, dtype=dt, device=device) for k, (shape, dt) in specs.items()}
    return {k: check_device_tensor(out.get(k), f"out[{k!r}]", device, dt, shape) for k, (shape, dt) in specs.items()}


def _joint_actions_device(fn, h, device, B, nx, nu, nj, t, robot_state, use_policy, out, stream) -> dict:
    import torch

    rs = None if robot_state is None else check_device_tensor(robot_state, "robot_state", device, torch.float64, (B, 13 + 2 * nj))
    f64, i32 = torch.float64, torch.int32
    o = _device_outputs(device, dict(q_des=((B, nj), f64), qd_des=((B, nj), f64), tau=((B, nj), f64), x=((B, nx), f64), u=((B, nu), f64),
                                     mode=((B,), i32), status=((B,), i32)), out)
    _l.check(fn(h, C.c_double(t), _vp(rs), C.c_int(int(use_policy)), _vp(o["q_des"]), _vp(o["qd_des"]), _vp(o["tau"]), _vp(o["x"]), _vp(o["u"]),
                _vp(o["mode"]), _vp(o["status"]), _stream(device, stream)))
    return o


def _mrt_query(fn, h, wait, B, nx, nu, t, x, value, gain, stream) -> dict:
    """the host entry point of the MRT queries; dfdxx / K come back column-major and are returned as [B, nx, nx] / [B, nu, nx]"""
    xs = None if x is None or not value else _f(x)
    if xs is not None:
        assert xs.shape == (B, nx), xs.shape
    P = np.zeros((B, nx, nx)) if value else None
    p = np.zeros((B, nx)) if value else None
    K = np.zeros((B, nx, nu)) if gain else None
    opt = lambda a: None if a is None else _p(a)
    _l.check(fn(h, C.c_double(t), opt(xs), opt(P), opt(p), opt(K), C.c_void_p(stream or 0)))
    wait()
    out = {}
    if value:
        out["dfdxx"], out["dfdx"] = np.swapaxes(P, -1, -2).copy(), p
    if gain:
        out["K"] = np.swapaxes(K, -1, -2).copy()
    return out


def _mrt_query_device(fn, h, device, B, nx, nu, t, x, value, gain, stream) -> dict:
    import torch

    xs = None if x is None or not value else check_device_tensor(x, "x", device, torch.float64, (B, nx))
    f64 = torch.float64
    P = torch.empty((B, nx, nx), dtype=f64, device=device) if value else None
    p = torch.empty((B, nx), dtype=f64, device=device) if value else None
    K = torch.empty((B, nx, nu), dtype=f64, device=device) if gain else None
    _l.check(fn(h, C.c_double(t), _vp(xs), _vp(P), _vp(p), _vp(K), _stream(device, stream)))
    out = {}
    if value:
        out["dfdxx"], out["dfdx"] = P.transpose(-1, -2), p
    if gain:
        out["K"] = K.transpose(-1, -2)
    return out


def _set_gains(fn, h, indices, gains):
    idx = np.ascontiguousarray(np.atleast_1d(indices), dtype=np.int32)
    rec = None if gains is None else abi.pack_gains(gains, idx.size if np.ndim(gains["final_cost_active"]) == 0 else None)
    if rec is not None and rec.shape[0] != idx.size:
        raise ValueError(f"set_gains: {rec.shape[0]} gain records for {idx.size} instances")
    _l.check(fn(h, C.c_int(idx.size), idx.ctypes.data_as(_l.ip), None if rec is None else rec.ctypes.data_as(C.c_void_p)))


def _gains(fn, h, B) -> dict:
    rec, custom = np.zeros((B, abi.GAINS_BYTES), dtype=np.uint8), np.zeros(B, dtype=np.int32)
    _l.check(fn(h, rec.ctypes.data_as(C.c_void_p), custom.ctypes.data_as(_l.ip)))
    out = abi.unpack_gains(rec)
    out["custom"] = custom.astype(bool)
    return out


def _set_gains_device(fn, h, device, indices, gains, stream):
    import torch

    idx = np.ascontiguousarray(np.atleast_1d(indices), dtype=np.int32)
    g = check_device_tensor(gains, "gains", device, torch.uint8, (idx.size, abi.GAINS_BYTES))
    status = torch.empty(idx.size, dtype=torch.int32, device=device)
    _l.check(fn(h, C.c_int(idx.size), idx.ctypes.data_as(_l.ip), _vp(g), _vp(status), _stream(device, stream)))
    return status


def _params_target(target, mask=True) -> int:
    if target not in abi.PARAMS_TARGETS or (not mask and target == "both"):
        raise ValueError(f"robot params: target must be one of {list(abi.PARAMS_TARGETS)[:3 if mask else 2]}, got {target!r}")
    return abi.PARAMS_TARGETS[target]


def _set_robot_params(fn, h, indices, params, target):
    idx = np.ascontiguousarray(np.atleast_1d(indices), dtype=np.int32)
    rec = None if params is None else abi.pack_robot_params(params, idx.size if np.ndim(params["mass"]) == 1 else None)
    if rec is not None and rec.shape[0] != idx.size:
        raise ValueError(f"set_robot_params: {rec.shape[0]} records for {idx.size} instances")
    _l.check(fn(h, C.c_int(idx.size), idx.ctypes.data_as(_l.ip), None if rec is None else rec.ctypes.data_as(C.c_void_p),
                C.c_int(_params_target(target))))


def _robot_params(fn, h, B, target) -> dict:
    rec, custom = np.zeros((B, abi.ROBOT_PARAMS_BYTES), dtype=np.uint8), np.zeros(B, dtype=np.int32)
    _l.check(fn(h, C.c_int(_params_target(target, mask=False)), rec.ctypes.data_as(C.c_void_p), custom.ctypes.data_as(_l.ip)))
    out = abi.unpack_robot_params(rec)
    out["custom"] = custom.astype(bool)
    return out


def _set_robot_params_device(fn, h, device, indices, params, target, stream):
    import torch

    idx = np.ascontiguousarray(np.atleast_1d(indices), dtype=np.int32)
    p = check_device_tensor(params, "params", device, torch.uint8, (idx.size, abi.ROBOT_PARAMS_BYTES))
    status = torch.empty(idx.size, dtype=torch.int32, device=device)
    _l.check(fn(h, C.c_int(idx.size), idx.ctypes.data_as(_l.ip), _vp(p), C.c_int(_params_target(target)), _vp(status), _stream(device, stream)))
    return status


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
        self.device = device
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
        fleet = self._fleet() if getattr(self, "_fleet", None) else None
        if fleet is not None:   # (b200sqp_destroy would destroy it too, leaving the fleet object with a dangling pointer)
            fleet.close()
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
        common number of shooting nodes.  With a motion manager (set_motion_manager) cmd is the raw velocity command and gaits may be None on
        warm builds.  x0 may be a float64 CUDA tensor on the handle's device (b200sqp_build_instances_dev): the build reads it after the work
        enqueued so far on the current torch stream."""
        if _is_cuda_tensor(x0):
            return self._build_dev(t0, horizon, x0, gaits, gait_start, cmd, warm)
        if warm == "rollout":
            if x0 is not None:
                raise ValueError('warm="rollout" takes the measured state from the last roll-out; pass x0=None')
            warm = 2
        elif isinstance(warm, str):
            raise ValueError(f"warm must be a bool or 'rollout', got {warm!r}")
        L = _l.lib()
        self._ensure_builder()
        B, gid, gs, cm = _build_args(x0, gaits, gait_start, cmd, self._gait_names)
        x0 = None if x0 is None else _f(x0)
        n = C.c_int32()
        _l.check(L.b200sqp_build_instances(self._h, C.c_int(B), C.c_double(t0), C.c_double(horizon), None if x0 is None else _p(x0),
                                           None if gid is None else gid.ctypes.data_as(_l.ip), _p(gs), _p(cm), C.c_int(int(warm)), C.byref(n)))
        self.batch, self.n_nodes = B, n.value
        return n.value

    def _build_dev(self, t0, horizon, x0, gaits, gait_start, cmd, warm):
        import torch

        if isinstance(warm, str):
            raise ValueError(f"warm must be a bool with a device x0 (warm='rollout' takes the simulated state), got {warm!r}")
        self._ensure_builder()
        B, gid, gs, cm = _build_args(None, gaits, gait_start, cmd, self._gait_names)
        check_device_tensor(x0, "x0", torch.device("cuda", self.device), torch.float64, (B, self.nx))
        n = C.c_int32()
        _l.check(_l.lib().b200sqp_build_instances_dev(self._h, C.c_int(B), C.c_double(t0), C.c_double(horizon), _vp(x0),
                                                      None if gid is None else gid.ctypes.data_as(_l.ip), _p(gs), _p(cm), C.c_int(int(warm)), C.byref(n),
                                                      _stream(torch.device("cuda", self.device), None)))
        self.batch, self.n_nodes = B, n.value
        return n.value

    def set_gait_schedule(self, stateful: bool = True, phase_transition_stance_time: float = 0.0):
        """b200sqp_set_gait_schedule: stateful = True keeps every instance's gait schedule on the device across cycles; the gaits passed to a
        warm build_instances are then per-instance gait commands (a changed one runs the reference's updateGaitSchedule, visible in the next
        cycle's schedule), and the warm start is spread over the new schedule.  Takes effect at the next cold build."""
        _l.check(_l.lib().b200sqp_set_gait_schedule(self._h, C.c_int(int(stateful)), C.c_double(phase_transition_stance_time)))

    def set_joint_torque_cost(self, weights=None):
        """b200sqp_set_joint_torque_cost: the reference's JointTorqueCostCppAd on every intermediate node, weights [nj] in MPC joint order
        (model_loader.joint_torque_weights reads them from a task.info); None or all zeros turns the term off.  Whole-body models only; takes
        effect at the next solve."""
        w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float64)
        if w is not None and w.shape != (self.model["nj"],):
            raise ValueError(f"set_joint_torque_cost: {w.shape} weights for {self.model['nj']} joints")
        _l.check(_l.lib().b200sqp_set_joint_torque_cost(self._h, None if w is None else w.ctypes.data_as(_l.dp)))

    def set_motion_manager(self, enable: bool = True, filter_origin: float = 0.0):
        """b200sqp_set_motion_manager: the reference's ProceduralMpcMotionManager per instance on the device (stateful gait schedule needed).
        The velocity scales come from model["reference"], the gait ids of its seven states from the builder's gait table.  The cmd of every
        build is then the raw velocity command (clamped, scaled, filtered); the gaits of a cold build are the starting states (one of
        abi.MOTION_GAITS), those of warm builds are ignored (may be None).  enable = False switches it off.  Takes effect at the next cold build."""
        self._ensure_builder()
        md = abi.motion_desc(self.model, self._gait_names, filter_origin) if enable else None
        _l.check(_l.lib().b200sqp_set_motion_manager(self._h, None if md is None else C.byref(md)))

    def cen_set_gait_schedule(self, stateful: bool = True, phase_transition_stance_time: float = 0.0):
        """set_gait_schedule on a centroidal model (b200sqp_cen_set_gait_schedule): the same stateful schedule, gait commands and spread"""
        _l.check(_l.lib().b200sqp_cen_set_gait_schedule(self._h, C.c_int(int(stateful)), C.c_double(phase_transition_stance_time)))

    def cen_set_motion_manager(self, enable: bool = True, filter_origin: float = 0.0):
        """set_motion_manager on a centroidal model (b200sqp_cen_set_motion_manager): the manager of the reference's centroidal MPC node, with
        the centroidal target rule, transitions on the normalized momentum x0[:6] and the scales of the centroidal reference.info (needs
        cen_set_gait_schedule(True))"""
        self._ensure_builder()
        md = abi.motion_desc(self.model, self._gait_names, filter_origin) if enable else None
        _l.check(_l.lib().b200sqp_cen_set_motion_manager(self._h, None if md is None else C.byref(md)))

    def _ensure_builder(self):
        if not getattr(self, "_builder_set", False):
            self._bdesc, self._gait_names = abi.builder_desc(self.model)
            _l.check(_l.lib().b200sqp_set_builder(self._h, C.byref(self._bdesc)))
            self._builder_set = True

    def motion_state(self) -> dict:
        """b200sqp_download_motion_state: {state [B] (index into abi.MOTION_GAITS), gait [B] (names), last_change [B], filtered_cmd [B, 4]}"""
        return _motion_state(_l.lib().b200sqp_download_motion_state, self._h, self.batch)

    # -- per-instance resets (the episode loop of MpcnetRolloutBase) ---------------------------------------------------------------
    def set_reset_states(self, x0, gaits, offsets=None):
        """b200sqp_set_reset_states: the row every instance restarts from when it is reset: x0 [B, nx], gait names (or ids) [B], gait offsets
        [B] (<= 0.5; the gait is tiled from the reset time + offset; None: zeros).  Needs the stateful gait schedule; may be replaced any time."""
        self._ensure_builder()
        self._reset_batch = _set_reset_states(_l.lib().b200sqp_set_reset_states, self._h, x0, gaits, offsets, self._gait_names)

    def set_auto_reset(self, enable: bool = True, on_solve_failure: bool = False, on_rollout_failure: bool = False, max_height_deviation: float = 0.0,
                       max_pitch_deviation: float = 0.0, max_roll_deviation: float = 0.0):
        """b200sqp_set_auto_reset: reset an instance at a warm build when its measured state is not finite, or (when enabled) its last solve or
        roll-out failed, or its height / pitch / roll deviates from its reset row's by more than the bound (0: that test off).  Set it before
        creating a fleet."""
        d = abi.AutoResetDesc(int(on_solve_failure), int(on_rollout_failure), max_height_deviation, max_pitch_deviation, max_roll_deviation)
        _l.check(_l.lib().b200sqp_set_auto_reset(self._h, C.byref(d) if enable else None))

    def request_resets(self, indices):
        """b200sqp_request_resets: reset these instances at the next warm build"""
        _request_resets(_l.lib().b200sqp_request_resets, self._h, indices)

    def episodes(self) -> dict:
        """b200sqp_download_episodes: {episode [B], start [B], reason [B] (codes of abi.RESET_REASONS), reason_name [B], reset [B] (bool, at the
        last build), last_length [B] (the length of the episode the last reset ended)}"""
        return _episodes(_l.lib().b200sqp_download_episodes, self._h, getattr(self, "_reset_batch", 0))

    # -- pose commands (commandedPositionToTargetTrajectories, latched per instance on the device) ----------------------------------
    def set_pose_commands(self, enable: bool = True):
        """b200sqp_set_pose_commands with the reference.info values of model["reference"] (enable = False: off, every instance follows its
        velocity command again).  Refused with a motion manager; set it before creating a fleet."""
        pd = abi.pose_desc(self.model) if enable else None
        _l.check(_l.lib().b200sqp_set_pose_commands(self._h, None if pd is None else C.byref(pd)))

    def command_poses(self, indices, deltas):
        """b200sqp_command_poses: deltas [len(indices), 4] = (dx, dy, dz, dyaw in degrees) in the pelvis frame, latched from each instance's
        measured state at the next build (see references.pose_command_targets)"""
        _command_poses(_l.lib().b200sqp_command_poses, self._h, indices, deltas)

    def clear_poses(self, indices):
        """b200sqp_clear_poses: these instances follow their velocity command again from the next build"""
        _request_resets(_l.lib().b200sqp_clear_poses, self._h, indices)

    def pose_targets(self) -> dict:
        """b200sqp_download_pose_targets: {active [B] (bool), t_start [B], t_reach [B], target_pose [B, 6], error [B, 2] (planar distance and
        |yaw error| of the last build's measured state)}"""
        return _pose_targets(_l.lib().b200sqp_download_pose_targets, self._h, self.batch)

    # -- per-instance gains (the reference's GainsReceiver, per instance on the device) ---------------------------------------------
    def default_gains(self) -> dict:
        """b200sqp_default_gains: the model's cost weights and penalties, every term active, as {field of abi.Gains: value}"""
        g = abi.Gains()
        _l.check(_l.lib().b200sqp_default_gains(self._h, C.byref(g)))
        return {k: v[0] for k, v in abi.unpack_gains(np.frombuffer(bytes(g), dtype=np.uint8)).items()}

    def set_gains(self, indices, gains: dict | None):
        """b200sqp_set_gains: gains {field: array with a leading len(indices) axis} (a default_gains()-shaped dict applies to every listed
        instance), or None to restore the model's values; takes effect at each instance's next solve"""
        _set_gains(_l.lib().b200sqp_set_gains, self._h, indices, gains)

    def gains(self) -> dict:
        """b200sqp_download_gains: {field: [B, ...]} and custom [B] (bool: set by set_gains)"""
        return _gains(_l.lib().b200sqp_download_gains, self._h, self.batch)

    def set_gains_device(self, indices, gains, stream=None):
        """b200sqp_set_gains_dev: gains a uint8 CUDA tensor [len(indices), abi.GAINS_BYTES] in the b200sqp_gains layout (abi.pack_gains),
        checked and applied per row on the device on `stream` (None: the current torch stream); returns the int32 status tensor (0 applied,
        1 an entry is not finite, 2 out of range)"""
        import torch

        return _set_gains_device(_l.lib().b200sqp_set_gains_dev, self._h, torch.device("cuda", self.device), indices, gains, stream)

    # -- per-instance robot parameters: the inertial parameters of each instance's model and of its simulated plant ----------------
    def default_robot_params(self) -> dict:
        """b200sqp_default_robot_params: the handle's masses, coms and inertias (and SRBD nominal fields) as {field of abi.RobotParams: value}"""
        p = abi.RobotParams()
        _l.check(_l.lib().b200sqp_default_robot_params(self._h, C.byref(p)))
        return {k: v[0] for k, v in abi.unpack_robot_params(np.frombuffer(bytes(p), dtype=np.uint8)).items()}

    def set_robot_params(self, indices, params: dict | None, target: str = "both"):
        """b200sqp_set_robot_params: params {field: array with a leading len(indices) axis} (a default_robot_params()-shaped dict applies to
        every listed instance), or None to restore the handle's values, for target "model" (the OCP, builder and joint actions), "plant" (the
        policy roll-out) or "both"; takes effect at each instance's next build, solve, roll-out or joint-action call"""
        _set_robot_params(_l.lib().b200sqp_set_robot_params, self._h, indices, params, target)

    def robot_params(self, target: str = "model") -> dict:
        """b200sqp_download_robot_params: {field: [B, ...]} and custom [B] (bool: set) of target "model" or "plant"."""
        return _robot_params(_l.lib().b200sqp_download_robot_params, self._h, self.batch, target)

    def set_robot_params_device(self, indices, params, target: str = "both", stream=None):
        """b200sqp_set_robot_params_dev: params a uint8 CUDA tensor [len(indices), abi.ROBOT_PARAMS_BYTES] (abi.pack_robot_params), checked
        and applied per row on the device on `stream`; returns the int32 status tensor (0 applied, 1 not finite, 2 out of range)"""
        import torch

        return _set_robot_params_device(_l.lib().b200sqp_set_robot_params_dev, self._h, torch.device("cuda", self.device), indices, params, target,
                                        stream)

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

    def joint_actions(self, t: float, robot_state=None, use_policy: bool = True, stream=None) -> dict:
        """computeJointControlAction of the MRT joint controller for every instance (b200sqp_joint_actions), whole-body or centroidal.
        robot_state [B, 13 + 2 nj] (position, quaternion x y z w, local linear and angular velocity, joint positions, joint velocities) or None
        for the end state of the last roll-out; t is the policy time (the reference passes the robot time + 0.005).  use_policy = False is the
        weight-compensation branch.  Waits for the result and returns {q_des, qd_des, tau [B, nj], x [B, nx] (the observation), u [B, nu],
        mode [B]}; kp / kd are the reference's constants (see include/b200sqp.h)."""
        B, nx, nu, nj = self.batch, self.nx, self.nu, self.model["nj"]
        rs = None if robot_state is None else _f(robot_state)
        if rs is not None:
            assert rs.shape == (B, 13 + 2 * nj), rs.shape
        out = dict(q_des=np.zeros((B, nj)), qd_des=np.zeros((B, nj)), tau=np.zeros((B, nj)), x=np.zeros((B, nx)), u=np.zeros((B, nu)),
                   mode=np.zeros(B, dtype=np.int32))
        _l.check(_l.lib().b200sqp_joint_actions(self._h, C.c_double(t), None if rs is None else _p(rs), C.c_int(int(use_policy)), _p(out["q_des"]),
                                                _p(out["qd_des"]), _p(out["tau"]), _p(out["x"]), _p(out["u"]), out["mode"].ctypes.data_as(_l.ip),
                                                C.c_void_p(stream or 0)))
        self.wait()
        return out

    def joint_actions_device(self, t: float, robot_state=None, use_policy: bool = True, out: dict | None = None, stream=None) -> dict:
        """joint_actions in device memory (b200sqp_joint_actions_dev): robot_state a float64 CUDA tensor [B, 13 + 2 nj] on the handle's device,
        or None for the end state of the last roll-out.  Enqueued on `stream` (default: the current torch stream) without waiting; returns CUDA
        tensors {q_des, qd_des, tau [B, nj], x [B, nx], u [B, nu], mode [B], status [B]} (int32 mode / status), or fills `out`, a dict of such
        tensors.  status: 0 accepted, 1 a non-finite entry, 2 a quaternion norm off 1 by more than 1e-6; a rejected row gets NaN and mode -1."""
        import torch

        return _joint_actions_device(_l.lib().b200sqp_joint_actions_dev, self._h, torch.device("cuda", self.device), self.batch, self.nx, self.nu,
                                     self.model["nj"], t, robot_state, use_policy, out, stream)

    def mrt_query(self, t: float, x=None, value: bool = True, gain: bool = True, stream=None) -> dict:
        """MPC_MRT_Interface::getValueFunction(t, x) and getLinearFeedbackGain(t) of the last solve for every instance (b200sqp_mrt_query):
        value -> dfdxx [B, nx, nx], dfdx [B, nx] (the cost-to-go interpolated at t, re-centred at x [B, nx]; x = None: the end state of the
        last roll-out), gain -> K [B, nu, nx].  Needs settings.create_value_function / use_feedback_policy for what is asked.  Waits."""
        return _mrt_query(_l.lib().b200sqp_mrt_query, self._h, self.wait, self.batch, self.nx, self.nu, t, x, value, gain, stream)

    def mrt_query_device(self, t: float, x=None, value: bool = True, gain: bool = True, stream=None) -> dict:
        """mrt_query in device memory (b200sqp_mrt_query_dev): x a float64 CUDA tensor [B, nx] or None, enqueued on `stream` (default: the
        current torch stream) without waiting; CUDA tensors dfdxx [B, nx, nx] and K [B, nu, nx] (transposed views) and dfdx [B, nx]"""
        import torch

        return _mrt_query_device(_l.lib().b200sqp_mrt_query_dev, self._h, torch.device("cuda", self.device), self.batch, self.nx, self.nu, t, x,
                                 value, gain, stream)

    def primal_solution_device(self, with_gains: bool | None = None, stream=None) -> dict:
        """primal_solution in device memory (b200sqp_download_dev), enqueued on `stream` without waiting: CUDA tensors {x [B, n, nx],
        u [B, n-1, nu], status [B] (int32, the per-instance solve status; nothing is raised), K [B, n-1, nu, nx] (a transposed view) with gains}"""
        import torch

        dev = torch.device("cuda", self.device)
        B, n, nx, nu = self.batch, self.n_nodes, self.nx, self.nu
        with_gains = bool(self.settings.use_feedback_policy) if with_gains is None else with_gains
        o = _device_outputs(dev, dict(x=((B, n, nx), torch.float64), u=((B, n - 1, nu), torch.float64), status=((B,), torch.int32)), None)
        K = torch.empty((B, n - 1, nx, nu), dtype=torch.float64, device=dev) if with_gains else None
        _l.check(_l.lib().b200sqp_download_dev(self._h, _vp(o["x"]), _vp(o["u"]), _vp(K), _vp(o["status"]), _stream(dev, stream)))
        if K is not None:
            o["K"] = K.transpose(-1, -2)
        return o

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


class B200SqpFleet:
    """A batch whose instances may differ in node count, run through the device-resident MPC loop (b200sqp_fleet_*): attached to a
    B200SqpSolver (whole-body or centroidal), whose builder, gait-schedule and motion-manager configuration it takes over.  The instances are
    regrouped by node count on the device every cycle; every array here is in the caller's instance order, node arrays padded to the largest
    node count with zeros, with the per-instance node counts `n_nodes` beside them.  While the fleet lives, the solver's own methods are refused."""

    def __init__(self, solver: B200SqpSolver):
        self.solver = solver
        self.model, self.settings, self.nx, self.nu = solver.model, solver.settings, solver.nx, solver.nu
        L = _l.lib()
        solver._ensure_builder()
        self._f = C.c_void_p()
        _l.check(L.b200sqp_fleet_create(solver._h, C.byref(self._f)))
        solver._fleet = weakref.ref(self)
        self.batch, self.n_nodes, self.n_groups = 0, np.zeros(0, dtype=np.int32), 0

    def close(self):
        if self._f:
            # a destroyed handle has destroyed its fleet already (garbage collection may finalize the solver first: its weak reference to
            # this fleet is cleared by then)
            if self.solver._h:
                _l.lib().b200sqp_fleet_destroy(self._f)
            self._f = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def build_instances(self, t0: float, horizon: float, x0, gaits, gait_start, cmd, warm: bool | str = False) -> np.ndarray:
        """B200SqpSolver.build_instances for instances of any node count; returns n_nodes [B] (self.n_groups: the distinct counts).  x0 may be a
        float64 CUDA tensor (b200sqp_fleet_build_instances_dev)."""
        if _is_cuda_tensor(x0):
            return self._build_dev(t0, horizon, x0, gaits, gait_start, cmd, warm)
        if warm == "rollout":
            if x0 is not None:
                raise ValueError('warm="rollout" takes the measured state from the last roll-out; pass x0=None')
            warm = 2
        elif isinstance(warm, str):
            raise ValueError(f"warm must be a bool or 'rollout', got {warm!r}")
        B, gid, gs, cm = _build_args(x0, gaits, gait_start, cmd, self.solver._gait_names)
        x0 = None if x0 is None else _f(x0)
        n, G = np.zeros(B, dtype=np.int32), C.c_int32()
        _l.check(_l.lib().b200sqp_fleet_build_instances(self._f, C.c_int(B), C.c_double(t0), C.c_double(horizon), None if x0 is None else _p(x0),
                                                        None if gid is None else gid.ctypes.data_as(_l.ip), _p(gs), _p(cm), C.c_int(int(warm)),
                                                        n.ctypes.data_as(_l.ip), C.byref(G)))
        self.batch, self.n_nodes, self.n_groups = B, n, G.value
        return n.copy()

    def _build_dev(self, t0, horizon, x0, gaits, gait_start, cmd, warm):
        import torch

        if isinstance(warm, str):
            raise ValueError(f"warm must be a bool with a device x0 (warm='rollout' takes the simulated state), got {warm!r}")
        dev = torch.device("cuda", self.solver.device)
        B, gid, gs, cm = _build_args(None, gaits, gait_start, cmd, self.solver._gait_names)
        check_device_tensor(x0, "x0", dev, torch.float64, (B, self.nx))
        n, G = np.zeros(B, dtype=np.int32), C.c_int32()
        _l.check(_l.lib().b200sqp_fleet_build_instances_dev(self._f, C.c_int(B), C.c_double(t0), C.c_double(horizon), _vp(x0),
                                                            None if gid is None else gid.ctypes.data_as(_l.ip), _p(gs), _p(cm), C.c_int(int(warm)),
                                                            n.ctypes.data_as(_l.ip), C.byref(G), _stream(dev, None)))
        self.batch, self.n_nodes, self.n_groups = B, n, G.value
        return n.copy()

    def solve(self, stream=None, wait: bool = True):
        _l.check(_l.lib().b200sqp_fleet_solve(self._f, C.c_void_p(stream or 0)))
        if wait:
            self.wait()

    def wait(self):
        _l.check(_l.lib().b200sqp_fleet_wait(self._f))

    def motion_state(self) -> dict:
        """B200SqpSolver.motion_state of the fleet's instances (caller order); the manager is set on the solver before the fleet is created"""
        return _motion_state(_l.lib().b200sqp_fleet_download_motion_state, self._f, self.batch)

    def set_reset_states(self, x0, gaits, offsets=None):
        """B200SqpSolver.set_reset_states for the fleet's instances (caller order)"""
        self._reset_batch = _set_reset_states(_l.lib().b200sqp_fleet_set_reset_states, self._f, x0, gaits, offsets, self.solver._gait_names)

    def request_resets(self, indices):
        """B200SqpSolver.request_resets for the fleet's instances; the automatic predicate is set on the solver before the fleet is created"""
        _request_resets(_l.lib().b200sqp_fleet_request_resets, self._f, indices)

    def episodes(self) -> dict:
        """B200SqpSolver.episodes of the fleet's instances (caller order)"""
        return _episodes(_l.lib().b200sqp_fleet_download_episodes, self._f, getattr(self, "_reset_batch", 0) or getattr(self.solver, "_reset_batch", 0))

    def command_poses(self, indices, deltas):
        """B200SqpSolver.command_poses for the fleet's instances (caller order); pose commands are enabled on the solver before the fleet is
        created"""
        _command_poses(_l.lib().b200sqp_fleet_command_poses, self._f, indices, deltas)

    def clear_poses(self, indices):
        """B200SqpSolver.clear_poses for the fleet's instances (caller order)"""
        _request_resets(_l.lib().b200sqp_fleet_clear_poses, self._f, indices)

    def pose_targets(self) -> dict:
        """B200SqpSolver.pose_targets of the fleet's instances (caller order)"""
        return _pose_targets(_l.lib().b200sqp_fleet_download_pose_targets, self._f, self.batch)

    def default_gains(self) -> dict:
        return self.solver.default_gains()

    def set_gains(self, indices, gains: dict | None):
        """B200SqpSolver.set_gains for the fleet's instances (caller order)"""
        _set_gains(_l.lib().b200sqp_fleet_set_gains, self._f, indices, gains)

    def gains(self) -> dict:
        """B200SqpSolver.gains of the fleet's instances (caller order)"""
        return _gains(_l.lib().b200sqp_fleet_download_gains, self._f, self.batch)

    def set_gains_device(self, indices, gains, stream=None):
        """B200SqpSolver.set_gains_device for the fleet's instances (caller order)"""
        import torch

        return _set_gains_device(_l.lib().b200sqp_fleet_set_gains_dev, self._f, torch.device("cuda", self.solver.device), indices, gains, stream)

    def default_robot_params(self) -> dict:
        return self.solver.default_robot_params()

    def set_robot_params(self, indices, params: dict | None, target: str = "both"):
        """B200SqpSolver.set_robot_params for the fleet's instances (caller order)"""
        _set_robot_params(_l.lib().b200sqp_fleet_set_robot_params, self._f, indices, params, target)

    def robot_params(self, target: str = "model") -> dict:
        """B200SqpSolver.robot_params of the fleet's instances (caller order)"""
        return _robot_params(_l.lib().b200sqp_fleet_download_robot_params, self._f, self.batch, target)

    def set_robot_params_device(self, indices, params, target: str = "both", stream=None):
        """B200SqpSolver.set_robot_params_device for the fleet's instances (caller order)"""
        import torch

        return _set_robot_params_device(_l.lib().b200sqp_fleet_set_robot_params_dev, self._f, torch.device("cuda", self.solver.device), indices,
                                        params, target, stream)

    def mode_schedule(self, max_events: int = 192) -> list:
        B = self.batch
        ev, modes, n = np.zeros((B, max_events)), np.zeros((B, max_events + 1), dtype=np.int32), np.zeros(B, dtype=np.int32)
        _l.check(_l.lib().b200sqp_fleet_download_mode_schedule(self._f, C.c_int(max_events), _p(ev), modes.ctypes.data_as(_l.ip), n.ctypes.data_as(_l.ip)))
        return [(ev[b, : n[b]].tolist(), modes[b, : n[b] + 1].tolist()) for b in range(B)]

    def download_instances(self) -> dict:
        """the per-instance inputs as they lie on the device, padded to max(n_nodes) rows, plus n_nodes [B]"""
        B, m, nx, nu = self.batch, int(self.n_nodes.max()), self.nx, self.nu
        out = dict(x0=np.zeros((B, nx)), x_init=np.zeros((B, m, nx)), u_init=np.zeros((B, m - 1, nu)), t_nodes=np.zeros((B, m)),
                   node_event=np.zeros((B, m), dtype=np.uint8), contact_flags=np.zeros((B, m, 2), dtype=np.uint8), swing_ref=np.zeros((B, m, 2, 3)),
                   impact_factor=np.zeros((B, m, 2)), arm_phase=np.zeros((B, m)), x_ref=np.zeros((B, m, nx)), n_nodes=np.zeros(B, dtype=np.int32))
        u8 = lambda a: a.ctypes.data_as(_l.u8p)
        _l.check(_l.lib().b200sqp_fleet_download_instances(self._f, C.c_int(m), _p(out["x0"]), _p(out["x_init"]), _p(out["u_init"]), _p(out["t_nodes"]),
                                                           u8(out["node_event"]), u8(out["contact_flags"]), _p(out["swing_ref"]), _p(out["impact_factor"]),
                                                           _p(out["arm_phase"]), _p(out["x_ref"]), out["n_nodes"].ctypes.data_as(_l.ip)))
        return out

    def primal_solution(self, with_gains: bool | None = None, raise_on_failure: bool = True) -> dict:
        """x [B, m, nx], u [B, m - 1, nu] (m = max(n_nodes), rows past an instance's n_nodes zero), n_nodes, n_iter, status, log (and K)"""
        B, m, nx, nu = self.batch, int(self.n_nodes.max()), self.nx, self.nu
        x, u = np.zeros((B, m, nx)), np.zeros((B, m - 1, nu))
        with_gains = bool(self.settings.use_feedback_policy) if with_gains is None else with_gains
        K = np.zeros((B, m - 1, nx, nu)) if with_gains else None
        log = (abi.IterLog * (B * self.settings.sqp_iteration))()
        n_iter, status, n_nodes = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        rc = _l.lib().b200sqp_fleet_download(self._f, C.c_int(m), _p(x), _p(u), None if K is None else _p(K), log, n_iter.ctypes.data_as(_l.ip),
                                             status.ctypes.data_as(_l.ip), n_nodes.ctypes.data_as(_l.ip))
        if rc != 0 and (raise_on_failure or rc != -4):
            _l.check(rc)
        logs = np.frombuffer(log, dtype=np.float64).reshape(B, self.settings.sqp_iteration, 16).copy()
        out = dict(x=x, u=u, n_nodes=n_nodes, n_iter=n_iter, status=status, log=logs)
        if K is not None:
            out["K"] = np.swapaxes(K, -1, -2).copy()
        return out

    def iterations_log(self):
        return self.primal_solution(with_gains=False)["log"]

    def rollout_policy(self, t: float, duration: float, x_start=None, settings: abi.RolloutSettings | None = None, stream=None) -> dict:
        """B200SqpSolver.rollout_policy (cen_rollout_policy on a centroidal model, with its default settings)"""
        if settings is None:
            settings = abi.cen_default_rollout_settings() if self.model.get("kind") == "centroidal" else abi.default_rollout_settings()
        B, nx, nu = self.batch, self.nx, self.nu
        xs = None if x_start is None else _f(x_start)
        out = dict(x=np.zeros((B, nx)), u=np.zeros((B, nu)), mode=np.zeros(B, dtype=np.int32), n_steps=np.zeros((B, 3), dtype=np.int32),
                   status=np.zeros(B, dtype=np.int32))
        _l.check(_l.lib().b200sqp_fleet_rollout_policy(self._f, C.c_double(t), C.c_double(duration), None if xs is None else _p(xs), C.byref(settings),
                                                       _p(out["x"]), _p(out["u"]), out["mode"].ctypes.data_as(_l.ip), out["n_steps"].ctypes.data_as(_l.ip),
                                                       out["status"].ctypes.data_as(_l.ip), C.c_void_p(stream or 0)))
        self.wait()
        return out

    def joint_actions(self, t: float, robot_state=None, use_policy: bool = True, stream=None) -> dict:
        """B200SqpSolver.joint_actions"""
        B, nx, nu, nj = self.batch, self.nx, self.nu, self.model["nj"]
        rs = None if robot_state is None else _f(robot_state)
        out = dict(q_des=np.zeros((B, nj)), qd_des=np.zeros((B, nj)), tau=np.zeros((B, nj)), x=np.zeros((B, nx)), u=np.zeros((B, nu)),
                   mode=np.zeros(B, dtype=np.int32))
        _l.check(_l.lib().b200sqp_fleet_joint_actions(self._f, C.c_double(t), None if rs is None else _p(rs), C.c_int(int(use_policy)), _p(out["q_des"]),
                                                      _p(out["qd_des"]), _p(out["tau"]), _p(out["x"]), _p(out["u"]), out["mode"].ctypes.data_as(_l.ip),
                                                      C.c_void_p(stream or 0)))
        self.wait()
        return out

    def joint_actions_device(self, t: float, robot_state=None, use_policy: bool = True, out: dict | None = None, stream=None) -> dict:
        """B200SqpSolver.joint_actions_device (b200sqp_fleet_joint_actions_dev), caller order"""
        import torch

        return _joint_actions_device(_l.lib().b200sqp_fleet_joint_actions_dev, self._f, torch.device("cuda", self.solver.device), self.batch, self.nx,
                                     self.nu, self.model["nj"], t, robot_state, use_policy, out, stream)

    def mrt_query(self, t: float, x=None, value: bool = True, gain: bool = True, stream=None) -> dict:
        """B200SqpSolver.mrt_query (b200sqp_fleet_mrt_query), caller order, each instance on its own plan"""
        return _mrt_query(_l.lib().b200sqp_fleet_mrt_query, self._f, self.wait, self.batch, self.nx, self.nu, t, x, value, gain, stream)

    def mrt_query_device(self, t: float, x=None, value: bool = True, gain: bool = True, stream=None) -> dict:
        """B200SqpSolver.mrt_query_device (b200sqp_fleet_mrt_query_dev), caller order"""
        import torch

        return _mrt_query_device(_l.lib().b200sqp_fleet_mrt_query_dev, self._f, torch.device("cuda", self.solver.device), self.batch, self.nx,
                                 self.nu, t, x, value, gain, stream)

    def value_function(self, max_nodes: int | None = None):
        """B200SqpSolver.value_function of the fleet (b200sqp_fleet_download_value_function): (P [B, m, nx, nx], p [B, m, nx], n_nodes [B]) with
        m = max_nodes or max(n_nodes), rows past an instance's n_nodes zero"""
        B, nx = self.batch, self.nx
        m = int(self.n_nodes.max()) if max_nodes is None else int(max_nodes)
        P, p, n = np.zeros((B, m, nx, nx)), np.zeros((B, m, nx)), np.zeros(B, dtype=np.int32)
        _l.check(_l.lib().b200sqp_fleet_download_value_function(self._f, C.c_int(m), _p(P), _p(p), n.ctypes.data_as(_l.ip)))
        return np.swapaxes(P, -1, -2).copy(), p, n

    def primal_solution_device(self, with_gains: bool | None = None, stream=None) -> dict:
        """B200SqpSolver.primal_solution_device (b200sqp_fleet_download_dev): x [B, m, nx], u [B, m - 1, nu] (m = max(n_nodes), rows past an
        instance's n_nodes zero), status, K with gains, as CUDA tensors, and n_nodes [B] (numpy)"""
        import torch

        dev = torch.device("cuda", self.solver.device)
        B, m, nx, nu = self.batch, int(self.n_nodes.max()), self.nx, self.nu
        with_gains = bool(self.settings.use_feedback_policy) if with_gains is None else with_gains
        o = _device_outputs(dev, dict(x=((B, m, nx), torch.float64), u=((B, m - 1, nu), torch.float64), status=((B,), torch.int32)), None)
        K = torch.empty((B, m - 1, nx, nu), dtype=torch.float64, device=dev) if with_gains else None
        n_nodes = np.zeros(B, dtype=np.int32)
        _l.check(_l.lib().b200sqp_fleet_download_dev(self._f, C.c_int(m), _vp(o["x"]), _vp(o["u"]), _vp(K), _vp(o["status"]), n_nodes.ctypes.data_as(_l.ip),
                                                     _stream(dev, stream)))
        if K is not None:
            o["K"] = K.transpose(-1, -2)
        o["n_nodes"] = n_nodes
        return o

    def benchmarks(self):
        """device milliseconds of {LQ approximation, solve QP, line search, projection} of the last solve, summed over its groups"""
        ms = (C.c_float * 4)()
        _l.check(_l.lib().b200sqp_fleet_get_stage_times(self._f, ms))
        return list(ms)
