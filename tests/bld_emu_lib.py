"""ctypes binding of the CPU development harness of the device builder (tests/emu/libbldemu.so, built from tests/emu/bld_emu.cu): the
__host__ __device__ functions of wb_builder.cuh and wb_fleet.cuh executed on the host, whole builds in the kernel order of
b200sqp_build_instances and the functions one at a time.  Test infrastructure only -- never linked into or called by the product library."""
from __future__ import annotations

import ctypes as C

import numpy as np

from emu_build import build
from oracle_lib import F, _p, _pi

NX, NU, CNX = 58, 35, 35
MAX_EVENTS = 192   # BLD_MAX_EVENTS
# the node pass's arrays in the layout of solver.stack_instances: per-node shape and dtype
NODE_ARRAYS = dict(x_init=((NX,), np.float64), u_init=((NU,), np.float64), t_nodes=((), np.float64), node_event=((), np.uint8),
                   contact_flags=((2,), np.uint8), swing_ref=((2, 3), np.float64), impact_factor=((2,), np.float64), arm_phase=((), np.float64),
                   x_ref=((NX,), np.float64))
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(str(build("bld_emu.cu", "libbldemu.so")))
        L.emu_bld_create.restype = C.c_void_p
        L.emu_gait_create.restype = C.c_void_p
        L.emu_batch_member.restype = C.c_char_p
        _lib = L
    return _lib


def _u8(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_uint8))


def _i64(a):
    return a.ctypes.data_as(C.POINTER(C.c_longlong))


def pad(a):
    """[..., CNX] -> [..., NX] with zero padding (the device row layout of a centroidal handle); rows of NX entries stay as they are"""
    a = F(a)
    if a.shape[-1] == NX:
        return a
    return np.ascontiguousarray(np.concatenate([a, np.zeros(a.shape[:-1] + (NX - a.shape[-1],))], axis=-1))


class EmuBuilder:
    """B instances of the device builder's state, kept across builds, as the handle's batch allocation holds them.  stateful: the stateful gait
    schedule; motion: the motion manager's b200sqp_motion_desc, or None; pose: pose commands; reset: None, or the automatic reset rule as a
    dict of reset_reason's keyword arguments on / on_solve / on_rollout / max_dev (dict(on=False): requested resets only).  A centroidal model
    selects the centroidal target rule and the base velocity of its device model."""

    def __init__(self, model, B, horizon, stateful=False, motion=None, pose=False, reset=None):
        from wb_humanoid_mpc_b200 import abi

        self.L = lib()
        self.desc, self.names = abi.builder_desc(model)
        self.cen = model.get("kind") == "centroidal"
        self.nx = model["nx"]
        self.B, self.horizon = B, horizon
        self.cap = int(horizon / self.desc.dt) + 2 + 96
        pd = abi.pose_desc(model) if pose else None
        on = dev = None
        if reset is not None:
            on = (C.c_int * 3)(*(int(reset.get(k, False)) for k in ("on", "on_solve", "on_rollout")))
            dev = _p(F(reset.get("max_dev", (0.0, 0.0, 0.0))))
        mdl, cd = (C.byref(abi.model_desc(model)), C.byref(abi.cen_desc(model))) if self.cen else (None, None)
        h = self.L.emu_bld_create(C.byref(self.desc), C.c_int(B), C.c_int(self.cap), C.c_int(int(stateful)), None if motion is None else C.byref(motion),
                                  None if pd is None else C.byref(pd), on, dev, mdl, cd)
        assert h, "the device conversion refused the model"
        self.h = C.c_void_p(h)

    def _gaits(self, gaits):
        return np.zeros(self.B, np.int32) if gaits is None else np.ascontiguousarray([self.names.index(g) for g in gaits], dtype=np.int32)

    def set_reset_states(self, rows, gaits, offsets):
        """the reset rows [B, nx], the gaits and gait offsets of the instances' next episodes (b200sqp_set_reset_states)"""
        self.L.emu_bld_set_reset_states(self.h, _p(pad(rows)), _pi(self._gaits(gaits)), _p(F(offsets)))

    def _set_previous(self, previous):
        if isinstance(previous, dict):   # one length: rows at the stride of its node count
            pT, pE = F(previous["t"]), np.ascontiguousarray(previous["event"], dtype=np.uint8)
            self.L.emu_bld_set_previous(self.h, None, C.c_int(pT.shape[1] - 1), _p(pT), _u8(pE), _p(pad(previous["x"])), _p(F(previous["u"])))
            return
        B, cap = self.B, self.cap   # one length per instance, rows at the capacity stride
        lens = np.array([len(p["t"]) for p in previous], dtype=np.int32)
        pT, pE, pX, pU = np.zeros((B, cap)), np.zeros((B, cap), np.uint8), np.zeros((B, cap, NX)), np.zeros((B, cap, NU))
        for b, p in enumerate(previous):
            pT[b, : lens[b]], pE[b, : lens[b]], pX[b, : lens[b]], pU[b, : lens[b] - 1] = p["t"], p["event"], pad(p["x"]), p["u"]
        self.L.emu_bld_set_previous(self.h, _pi(lens), C.c_int(0), _p(pT), _u8(pE), _p(pX), _p(pU))

    def build(self, t0, x0, cmd, gaits=None, gait_start=None, warm=True, nodes=None, previous=None, requests=None, commands=None, clears=()):
        """one build in the kernel order of b200sqp_build_instances.  x0 [B, nx] (None: the previous solution at t0); gaits: names (None: the
        first gait, for the manager's warm builds); gait_start [B] (None: 0).  nodes: None (grid only), "batch" (one view of the batch: node
        arrays [B, n, ...], -2 on mixed node counts) or "slots" (one view per instance through a slot map: node arrays [B, cap, ...], zero
        behind each instance's nodes).  previous: this warm build's previous solution instead of the one the last build carried, dict(t [B, n],
        event, x [B, n, nx], u [B, n-1, nu]) of one length, or a list of such dicts per instance.  requests [B]: reset requests.  commands
        {instance: pose delta [4]} latched and clears [instances] cleared at this build.
        -> dict of the builder state per instance (and the node arrays), or -1 (overflow) / -2"""
        B, cap, L = self.B, self.cap, self.L
        if previous is not None:
            self._set_previous(previous)
        pc = pdl = None
        if commands or clears:
            pc, pdl = np.zeros(B, np.uint8), np.zeros((B, 4))
            for i in clears:
                pc[i] = 2
            for i, dl in (commands or {}).items():
                pc[i], pdl[i] = 1, dl
        req = None if requests is None else np.ascontiguousarray(requests, np.uint8)
        gs = F(np.zeros(B) if gait_start is None else gait_start)
        rc = L.emu_bld_build(self.h, C.c_int(int(warm)), C.c_double(t0), C.c_double(self.horizon), None if x0 is None else _p(pad(x0)), _pi(self._gaits(gaits)),
                             _p(gs), _p(F(cmd)), _u8(req), _u8(pc), None if pdl is None else _p(pdl), C.c_int({None: 0, "batch": 1, "slots": 2}[nodes]))
        if rc < 0:
            return rc
        out = dict(n_nodes=np.zeros(B, np.int32), grid_t=np.zeros((B, cap)), bv=np.zeros((B, 6)), tt_time=np.zeros((B, 3)), tt_state=np.zeros((B, 3, NX)),
                   spr_len=np.zeros(B, np.int32), state=np.zeros(B, np.int32), last_change=np.zeros(B), origin=np.zeros(B), filtered=np.zeros((B, 4)),
                   active=np.zeros(B, np.int32), t_start=np.zeros(B), t_reach=np.zeros(B), target=np.zeros((B, 6)), error=np.zeros((B, 2)))
        nev, ev, modes = np.zeros(B, np.int32), np.zeros((B, MAX_EVENTS)), np.zeros((B, MAX_EVENTS + 1), np.int32)
        L.emu_bld_instances(self.h, _pi(out["n_nodes"]), _p(out["grid_t"]), _p(out["bv"]), _p(out["tt_time"]), _p(out["tt_state"]), _pi(out["spr_len"]),
                            _pi(nev), _p(ev), _pi(modes))
        L.emu_bld_motion(self.h, _pi(out["state"]), _p(out["last_change"]), _p(out["origin"]), _p(out["filtered"]))
        L.emu_bld_pose(self.h, _pi(out["active"]), _p(out["t_start"]), _p(out["t_reach"]), _p(out["target"]), _p(out["error"]))
        n = out["n_nodes"]
        out["active"] = out["active"].astype(bool)
        out["schedules"] = [(ev[b, : nev[b]].tolist(), modes[b, : nev[b] + 1].tolist()) for b in range(B)]
        out["grids"] = [out["grid_t"][b, : n[b]].tolist() for b in range(B)]
        out["pad_max"] = float(np.max(np.abs(out["tt_state"][..., self.nx:]), initial=0.0))   # (the target knots of a centroidal handle)
        out["tt_state"] = out["tt_state"][..., : self.nx].copy()
        if nodes is not None:
            raw = {k: np.zeros(B * cap * int(np.prod(shape)), dt) for k, (shape, dt) in NODE_ARRAYS.items()}
            L.emu_bld_nodes(self.h, *(_u8(v) if v.dtype == np.uint8 else _p(v) for v in raw.values()))
            for k, (shape, dt) in NODE_ARRAYS.items():
                per, u = int(np.prod(shape)), k == "u_init"
                if nodes == "batch":   # rows at the strides of the common node count
                    rows = n[0] - u
                    out[k] = raw[k][: B * rows * per].reshape((B, rows) + shape).copy()
                else:   # instance b's view starts at row b * cap (stage row b * (cap - 1))
                    stride, flat = cap - u, raw[k].reshape((-1,) + shape)
                    out[k] = np.zeros((B, stride) + shape, dt)
                    for b in range(B):
                        out[k][b, : n[b] - u] = flat[b * stride: b * stride + n[b] - u]
        return out

    def __del__(self):
        try:
            self.L.emu_bld_destroy(self.h)
        except Exception:
            pass


def build_instances(model, t0, horizon, x0, gaits, gait_start, cmd, previous=None):
    """one build on the path of a plain handle (closed-form schedule, one view of the batch; warm with previous = dict(t [B, n], event [B, n],
    x [B, n, nx], u [B, n-1, nu])) -> dict in the layout of solver.stack_instances, or a negative error code.  On a centroidal model:
    (that dict with the padding stripped, base velocities [B, 6], {key: max |padding entry|})."""
    x0 = F(x0)
    emu = EmuBuilder(model, x0.shape[0], horizon)
    r = emu.build(t0, x0, cmd, gaits, gait_start, warm=previous is not None, nodes="batch", previous=previous)
    if isinstance(r, int):
        return r
    res = {k: r[k] for k in NODE_ARRAYS}
    res["x0"] = x0
    if not emu.cen:
        return res
    padding = {}
    for k in ("x_init", "x_ref"):
        padding[k] = float(np.max(np.abs(res[k][..., CNX:])))
        res[k] = res[k][..., :CNX].copy()
    return res, r["bv"], padding


def warm_build(model, t0, horizon, x0, gaits, gait_start, cmd, previous, per_instance=True, stateful=False, t_prev=0.0):
    """warm build from previous = [dict(t [n_i], event [n_i], x [n_i, nx], u [n_i - 1, nu])] * B: with per_instance, the previous solutions keep
    their own lengths at the capacity stride and every instance is built through a slot map (the fleet's path); without, they share one length
    and one view of the batch is built.  stateful: the stateful gait schedule, seeded by a cold build at t_prev (the build of the previous
    solution).  -> (n_nodes [B], [dict of instance b's node arrays and x0])"""
    x0 = F(x0)
    B = x0.shape[0]
    emu = EmuBuilder(model, B, horizon, stateful=stateful)
    if stateful:
        r = emu.build(t_prev, x0, cmd, gaits, gait_start, warm=False)
        assert not isinstance(r, int), r
    if not per_instance:
        previous = {k: np.array([p[k] for p in previous]) for k in ("t", "event", "x", "u")}
    r = emu.build(t0, x0, cmd, gaits, gait_start, nodes="slots" if per_instance else "batch", previous=previous)
    assert not isinstance(r, int), r
    n = r["n_nodes"]
    return n, [{**{k: r[k][b, : n[b] - (k == "u_init")] for k in NODE_ARRAYS}, "x0": x0[b]} for b in range(B)]


# ---- the functions one at a time ---------------------------------------------------------------------------------------------------------------
class EmuGaitState:
    """one instance's BldGaitState driven by the device functions: seed (the cold build), get (getModeSchedule), update (updateGaitSchedule)"""

    def __init__(self, desc):
        self.L, self.desc = lib(), desc
        self.h = C.c_void_p(self.L.emu_gait_create())

    def seed(self, gait, start, t0, tf):
        assert self.L.emu_gait_seed(self.h, C.byref(self.desc), C.c_int(gait), C.c_double(start), C.c_double(t0), C.c_double(tf)) == 0

    def get_mode_schedule(self, lb, ub):
        assert self.L.emu_gait_get(self.h, C.byref(self.desc), C.c_double(lb), C.c_double(ub)) == 0
        return self.state()

    def update_gait(self, gait, t0, tf, ptst=0.0):
        return self.L.emu_gait_update(self.h, C.byref(self.desc), C.c_int(gait), C.c_double(t0), C.c_double(tf), C.c_double(ptst))

    def state(self, cap=MAX_EVENTS):
        ev, modes = np.zeros(cap), np.zeros(cap + 1, dtype=np.int32)
        n = self.L.emu_gait_state(self.h, _p(ev), _pi(modes), C.c_int(cap))
        assert n >= 0
        return ev[:n].tolist(), modes[: n + 1].tolist()

    def __del__(self):
        try:
            self.L.emu_gait_destroy(self.h)
        except Exception:
            pass


def spread(old_ev, old_modes, new_ev, new_modes, t, event, x, u):
    """bldSpreadStrategy + bldSpreadApply on one previous solution: t [n], event [n], x [n][NX], u [n-1][NU] -> dict(t, x, u (toPrimalSolution
    form), will_truncate, will_spread, post_event_indices, triples [(begin, end, value)])"""
    n = len(t)
    t, x, u = F(t), F(x), F(u)
    ev8 = np.ascontiguousarray(event, dtype=np.uint8)
    to, xo, uo = np.zeros(n), np.zeros((n, NX)), np.zeros((n, NU))
    ln, nps, nsp = C.c_int(0), C.c_int(0), C.c_int(0)
    fl, post, tri = np.zeros(2, dtype=np.int32), np.zeros(n + 200, dtype=np.int32), np.zeros(3 * 200, dtype=np.int32)
    rc = lib().emu_spread(C.c_int(len(old_ev)), _p(F(old_ev)), _pi(np.ascontiguousarray(old_modes, dtype=np.int32)), C.c_int(len(new_ev)), _p(F(new_ev)),
                          _pi(np.ascontiguousarray(new_modes, dtype=np.int32)), C.c_int(n), _p(t), _u8(ev8), _p(x), _p(u),
                          _p(to), _p(xo), _p(uo), C.byref(ln), _pi(fl), _pi(post), C.byref(nps), _pi(tri), C.byref(nsp))
    assert rc == 0
    m = ln.value
    return dict(t=to[:m], x=xo[:m], u=uo[:m], will_truncate=bool(fl[0]), will_spread=bool(fl[1]), post_event_indices=post[: nps.value].tolist(),
                triples=[tuple(tri[3 * k: 3 * k + 3]) for k in range(nsp.value)])


def motion_filter(md, raw, t0):
    f = np.zeros(4)
    lib().emu_motion_filter(C.byref(md), _p(F(raw)), C.c_double(t0), _p(f))
    return f


def motion_transition(state, last_change, f, bv, t0):
    s, lc = C.c_int(state), C.c_double(last_change)
    lib().emu_motion_transition(C.byref(s), C.byref(lc), _p(F(f)), _p(F(bv)), C.c_double(t0))
    return s.value, lc.value


def reset_reason(x, ref, *, requested=False, on=True, on_solve=False, on_rollout=False, max_dev=(0.0, 0.0, 0.0), cen=False, solve=0, rollout=0):
    x, ref = F(x), F(ref)
    return lib().emu_reset_reason(C.c_int(int(on)), C.c_int(int(on_solve)), C.c_int(int(on_rollout)), _p(F(max_dev)), C.c_int(int(requested)), _p(x), _p(ref),
                                  C.c_int(x.size), C.c_int(int(cen)), C.c_int(solve), C.c_int(rollout))


def reset_instances(x0, rows, books, *, warm=True, cen=False, t0=0.0, on=False, on_solve=False, on_rollout=False, max_dev=(0.0, 0.0, 0.0), req=None,
                    status=None, slot_inst=None, sim_info=None, sim_x=None):
    """bldResetDecide + bldResetApply over the batch; x0, sim_x and the books dict (episode, start, last_length, reason, rst) change in place"""
    B = x0.shape[0]
    req = np.zeros(B, np.uint8) if req is None else np.ascontiguousarray(req, np.uint8)
    flags = None
    if status is not None:
        flags = np.zeros((B, 8), np.int32)
        flags[:, 3] = status   # F_STATUS
    si = None if slot_inst is None else np.ascontiguousarray(slot_inst, np.int32)
    info = None if sim_info is None else np.ascontiguousarray(sim_info, np.int32)
    lib().emu_reset_instances(C.c_int(B), C.c_int(int(warm)), C.c_int(int(cen)), C.c_double(t0), C.c_int(int(on)), C.c_int(int(on_solve)),
                              C.c_int(int(on_rollout)), _p(F(max_dev)), _p(x0), _p(F(rows)), _u8(req), None if flags is None else _pi(flags),
                              None if si is None else _pi(si), None if info is None else _pi(info), None if sim_x is None else _p(sim_x),
                              _pi(books["episode"]), _p(books["start"]), _p(books["last_length"]), _pi(books["reason"]), _u8(books["rst"]))


def new_books(B):
    return dict(episode=np.zeros(B, np.int32), start=np.zeros(B), last_length=np.zeros(B), reason=np.zeros(B, np.int32), rst=np.zeros(B, np.uint8))


def partition(nodes, n_bins, threads=1024):
    """fleet_partition_kernel's phases -> (slot -> instance [B], group table [(nodes, first slot, count)])"""
    nodes = np.ascontiguousarray(nodes, dtype=np.int32)
    slot, gtab = np.zeros(len(nodes), dtype=np.int32), np.zeros(1 + 3 * n_bins, dtype=np.int32)
    lib().emu_fleet_partition(_pi(nodes), C.c_int(len(nodes)), C.c_int(n_bins), C.c_int(threads), _pi(slot), _pi(gtab))
    return slot, [tuple(gtab[1 + 3 * g: 4 + 3 * g]) for g in range(gtab[0])]


# ---- the batch layout (wb_batch.cuh) ---------------------------------------------------------------------------------------------------------------
ROW_KINDS = ("instance", "node", "stage", "handle")
MAX_ENTRIES = 64


def _layout_args(cen, value_function, feedback, raw, max_iter, raw_per):
    return (C.c_int(int(cen)), C.c_int(int(value_function)), C.c_int(int(feedback)), C.c_int(int(raw)), C.c_int(max_iter), C.c_longlong(raw_per))


def batch_layout(cen, value_function, feedback, raw, max_iter, raw_per):
    """forEachBatchArray of a handle with these settings (max_iter, raw_per: the widths of log and raw) -> [(member name, row kind, width,
    zero fill)] in allocation order"""
    L = lib()
    member, kind, zero = (np.zeros(MAX_ENTRIES, np.int32) for _ in range(3))
    width = np.zeros(MAX_ENTRIES, np.int64)
    n = L.emu_batch_layout(*_layout_args(cen, value_function, feedback, raw, max_iter, raw_per), _pi(member), _pi(kind), _i64(width), _pi(zero))
    assert (member[:n] >= 0).all(), "an entry of the table is no array member of WbDev"
    return [(L.emu_batch_member(int(m)).decode(), ROW_KINDS[k], int(w), bool(z)) for m, k, w, z in zip(member[:n], kind[:n], width[:n], zero[:n])]


def group_views(cen, value_function, feedback, raw, max_iter, raw_per, B, cap, groups):
    """the table's allocation of B instances at cap nodes, then groupView of every (n, first, count) of groups -> (bytes [E] allocated per
    entry, offsets [G, E] of each view's pointer into the entry's allocation in bytes, -1 for null), entries in allocation order"""
    gtab = np.array([len(groups), *(v for g in groups for v in g)], np.int32)
    bytes_, off = np.zeros(MAX_ENTRIES, np.int64), np.zeros(len(groups) * MAX_ENTRIES, np.int64)
    n = lib().emu_group_views(*_layout_args(cen, value_function, feedback, raw, max_iter, raw_per), C.c_int(B), C.c_int(cap), _pi(gtab), _i64(bytes_),
                              _i64(off))
    return bytes_[:n], off[: len(groups) * n].reshape(len(groups), n)


def fleet_slots(groups, B, cap):
    """fleetSlot of every slot (groups None: a plain handle) -> dict(n, first, count, node, stage) of [B] arrays"""
    gtab = None if groups is None else np.array([len(groups), *(v for g in groups for v in g)], np.int32)
    out = dict(n=np.zeros(B, np.int32), first=np.zeros(B, np.int32), count=np.zeros(B, np.int32), node=np.zeros(B, np.int64), stage=np.zeros(B, np.int64))
    lib().emu_fleet_slots(None if gtab is None else _pi(gtab), C.c_int(B), C.c_int(cap), _pi(out["n"]), _pi(out["first"]), _pi(out["count"]),
                          _i64(out["node"]), _i64(out["stage"]))
    return out


RIC_FIELDS = ("pq", "ab", "w", "y", "rs", "linv", "vec", "total", "kout")


def riccati_layout(nx, nm):
    """the shared-memory layouts of the generic Riccati kernels at (nx, nm) -> dict(one=..., cluster=...) of RIC_FIELDS (doubles), with
    one_doubles / cluster_doubles (the dynamic shared memory of each kernel), lx / lm (the one-CTA kernel's leading dimensions), supported
    (b200sqp_qp_create accepts the size) and limit (its byte limit)"""
    out = np.zeros(24, np.int64)
    lib().emu_riccati_layout(C.c_int(nx), C.c_int(nm), _i64(out))
    v = [int(x) for x in out]
    return dict(one=dict(zip(RIC_FIELDS, v[0:9])), cluster=dict(zip(RIC_FIELDS, v[9:18])), one_doubles=v[18], cluster_doubles=v[19], lx=v[20],
                lm=v[21], supported=bool(v[22]), limit=v[23])


def base_velocity(model, x):
    """bldCenBaseVelocity of centroidal states x [n, CNX] -> [n, 6]"""
    from wb_humanoid_mpc_b200 import abi

    desc, _ = abi.builder_desc(model)
    xp = pad(np.atleast_2d(x))
    out = np.zeros((xp.shape[0], 6))
    assert lib().emu_cen_base_velocity(C.byref(abi.model_desc(model)), C.byref(abi.cen_desc(model)), C.c_double(desc.total_mass), C.c_int(xp.shape[0]),
                                       _p(xp), _p(out)) == 0
    return out
