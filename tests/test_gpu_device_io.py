"""Device-pointer I/O of the closed loop (b200sqp_*_dev) on whole-body and centroidal handles, plain and fleets of at least two node-count
groups: builds from a CUDA-tensor x0 equal the host-pointer builds bit for bit; joint_actions_device equals joint_actions bit for bit, with
rejected robot-state rows flagged on the device; primal_solution_device equals primal_solution; the calls are ordered on the device without
a host synchronisation; the closed loop fed by joint_actions_device equals the warm = 2 loop; and foreign pointers are refused."""
import ctypes as C
import time

import numpy as np
import pytest

import mrt_ref
import test_gpu_builder
import test_gpu_cen_builder
import test_gpu_fleet
from test_gpu_mrt import LOOP, model_of
from wb_humanoid_mpc_b200 import abi
from wb_humanoid_mpc_b200 import lib as _l
from wb_humanoid_mpc_b200.lib import B200SqpError

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

B = 64
EINVAL = -1
FAMS = ["wb", "cen"]
KINDS = ["plain", "fleet"]
DT_MPC = 0.05
OUT_KEYS = ("q_des", "qd_des", "tau", "x", "u", "mode")


class Case:
    """one handle (plain: every instance walks from phase 0; fleet: stance / walk / slow_walk at random phases, several node counts)"""

    def __init__(self, fam, kind, batch=B, feedback=False, seed=21):
        from wb_humanoid_mpc_b200.solver import B200SqpFleet, B200SqpSolver

        self.fam, self.kind, self.B = fam, kind, batch
        self.model = model_of("wb" if fam == "wb" else "full")
        make = test_gpu_builder.make_inputs if fam == "wb" else test_gpu_cen_builder.make_inputs
        rng = np.random.default_rng(seed)
        self.x0s, self.cmds = make(self.model, rng, batch)
        self.solver = B200SqpSolver(self.model, abi.default_settings(self.model, sqp_iteration=1, use_feedback_policy=int(feedback)))
        if kind == "fleet":
            self.gaits, self.starts = test_gpu_fleet.mixed_batch(self.model, rng, batch)
            self.h = B200SqpFleet(self.solver)
        else:
            self.gaits, self.starts = ["walk"] * batch, np.zeros(batch)
            self.h = self.solver
        self.horizon, self.mrt_dt = LOOP["wb" if fam == "wb" else "full"]

    def build(self, t0, x0, warm=False):
        return self.h.build_instances(t0, self.horizon, x0, self.gaits, self.starts, self.cmds, warm=warm)

    def rollout(self, t, duration):
        if self.kind == "plain" and self.fam == "cen":
            return self.h.cen_rollout_policy(t, duration)
        return self.h.rollout_policy(t, duration)

    def robot_states(self, seed):
        return mrt_ref.random_robot_states(np.random.default_rng(seed), self.B, self.model["nj"])

    def check_groups(self):
        if self.kind == "fleet":
            assert self.h.n_groups >= 2


def cuda(a):
    return torch.tensor(np.asarray(a), dtype=torch.float64, device="cuda")


def same_dicts(a, b, keys=None):
    for k in keys or a:
        if k == "log":
            continue
        va = a[k]
        vb = b[k].cpu().numpy() if hasattr(b[k], "cpu") else b[k]
        assert va.shape == vb.shape, (k, va.shape, vb.shape)
        assert np.array_equal(va, vb, equal_nan=True), k


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fam", FAMS)
def test_builds_from_a_device_x0_equal_the_host_builds(fam, kind):
    a, b = Case(fam, kind), Case(fam, kind)
    assert np.array_equal(a.build(0.0, a.x0s), b.build(0.0, cuda(b.x0s)))
    b.check_groups()
    same_dicts(a.h.download_instances(), b.h.download_instances())
    a.h.solve()
    b.h.solve()
    same_dicts(a.h.primal_solution(), b.h.primal_solution())
    x1 = a.x0s + np.random.default_rng(9).normal(0.0, 1e-3, a.x0s.shape)   # a measured state off the plan
    assert np.array_equal(a.build(DT_MPC, x1, warm=True), b.build(DT_MPC, cuda(x1), warm=True))
    same_dicts(a.h.download_instances(), b.h.download_instances())
    a.h.solve()
    b.h.solve()
    same_dicts(a.h.primal_solution(), b.h.primal_solution())
    with pytest.raises(ValueError, match="warm"):
        b.build(2 * DT_MPC, cuda(x1), warm="rollout")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fam", FAMS)
def test_joint_actions_device_equal_the_host_path(fam, kind):
    c = Case(fam, kind, feedback=True)
    c.build(0.0, c.x0s)
    c.check_groups()
    c.h.solve()
    t = 0.05 + mrt_ref.POLICY_DT
    rs = c.robot_states(5)
    for use_policy in (True, False):
        host = c.h.joint_actions(t, rs, use_policy=use_policy)
        dev = c.h.joint_actions_device(t, cuda(rs), use_policy=use_policy)
        same_dicts(host, dev, OUT_KEYS)
        assert not dev["status"].any()
    c.rollout(0.0, c.mrt_dt)
    host = c.h.joint_actions(t)
    dev = c.h.joint_actions_device(t)
    same_dicts(host, dev, OUT_KEYS)
    assert not dev["status"].any()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fam", FAMS)
def test_rejected_rows(fam, kind):
    c = Case(fam, kind)
    c.build(0.0, c.x0s)
    c.h.solve()
    t = 0.031
    rs = c.robot_states(6)
    bad = rs.copy()
    bad[3, 20] = np.nan
    bad[7, 0] = np.inf
    bad[11, 3:7] *= (1.0 + 1e-5) / np.linalg.norm(bad[11, 3:7])
    rejected = [3, 7, 11]
    with pytest.raises(B200SqpError) as e:   # the host path refuses the whole call
        c.h.joint_actions(t, bad)
    assert e.value.code == EINVAL
    dev = c.h.joint_actions_device(t, cuda(bad))
    want = np.zeros(c.B, np.int32)
    want[rejected] = [1, 1, 2]
    assert dev["status"].cpu().numpy().tolist() == want.tolist()
    good = bad.copy()
    good[rejected] = rs[rejected]
    host = c.h.joint_actions(t, good)
    keep = np.setdiff1d(np.arange(c.B), rejected)
    for k in OUT_KEYS:
        d = dev[k].cpu().numpy()
        assert np.array_equal(d[keep], host[k][keep]), k
        if k == "mode":
            assert (d[rejected] == -1).all()
        else:
            assert np.isnan(d[rejected]).all(), k


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fam", FAMS)
def test_primal_solution_device_equals_primal_solution(fam, kind):
    c = Case(fam, kind, feedback=True)
    c.build(0.0, c.x0s)
    c.h.solve(wait=False)
    dev = c.h.primal_solution_device()   # enqueued behind the solve in flight
    host = c.h.primal_solution()
    assert dev["x"].shape[-1] == c.model["nx"] and dev["K"].shape[-1] == c.model["nx"]
    same_dicts(host, dev, ("x", "u", "K", "status"))
    if kind == "fleet":
        assert np.array_equal(dev["n_nodes"], c.h.n_nodes)
        n = c.h.n_nodes
        x, u = dev["x"].cpu().numpy(), dev["u"].cpu().numpy()
        for b in range(c.B):
            assert not x[b, n[b]:].any() and not u[b, n[b] - 1:].any(), b


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fam", FAMS)
def test_stream_order_without_a_host_wait(fam, kind):
    c = Case(fam, kind)
    c.build(0.0, c.x0s)
    c.h.solve()
    t = 0.02
    rs_old, rs_new = c.robot_states(7), c.robot_states(8)
    x, new = cuda(rs_old), cuda(rs_new)
    out = c.h.joint_actions_device(t, x)   # first call at this batch size: allocates, loads the kernels; `out` is reused below
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)   # ~50 ms
        x.copy_(new)
        t_call = time.perf_counter()
        c.h.joint_actions_device(t, x, out=out)
        t_call = time.perf_counter() - t_call
    assert t_call < 0.01, t_call
    torch.cuda.synchronize()
    same_dicts(c.h.joint_actions(t, rs_new), out, OUT_KEYS)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fam", FAMS)
def test_calls_run_in_call_order_across_streams(fam, kind):
    c = Case(fam, kind)
    c.build(0.0, c.x0s)
    c.h.solve()
    t = 0.02
    rs = c.robot_states(9)
    before = c.h.joint_actions(t, rs)   # the actions of the plan before the next build
    x = cuda(rs)
    out = c.h.joint_actions_device(t, x)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(100_000_000)
        c.h.joint_actions_device(t, x, out=out)
    c.build(DT_MPC, None, warm=True)   # rewrites the plan's buffers at once, from the host, on the handle's own stream
    torch.cuda.synchronize()
    same_dicts(before, out, OUT_KEYS)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fam", FAMS)
def test_closed_loop_fed_by_device_observations_equals_the_rollout_loop(fam, kind):
    """30 cycles with the dummy-simulation settings: joint_actions_device(t, None) -> build_instances(x0 = its x, warm) -> solve -> roll-out is
    bit-identical to build_instances(warm = "rollout") -> solve -> roll-out"""
    batch = 256 if fam == "wb" else 64
    feedback = fam == "wb"
    dev, ref = Case(fam, kind, batch, feedback), Case(fam, kind, batch, feedback)
    for c in (dev, ref):
        c.build(0.0, c.x0s)
        c.h.solve()
    dev.check_groups()
    for cyc in range(30):
        t0 = cyc * dev.mrt_dt
        if cyc > 0:
            obs = dev.h.joint_actions_device(t0 + mrt_ref.POLICY_DT)
            dev.build(t0, obs["x"], warm=True)
            ref.build(t0, None, warm="rollout")
            dev.h.solve()
            ref.h.solve()
            sd, sr = dev.h.primal_solution(), ref.h.primal_solution()
            assert np.array_equal(sd["x"], sr["x"]) and np.array_equal(sd["u"], sr["u"]), cyc
        rd, rr = dev.rollout(t0, dev.mrt_dt), ref.rollout(t0, ref.mrt_dt)
        assert np.array_equal(rd["x"], rr["x"]) and not rd["status"].any(), cyc


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fam", FAMS)
def test_foreign_pointers_are_refused(fam, kind):
    c = Case(fam, kind, batch=8, feedback=True)
    c.build(0.0, c.x0s)
    c.h.solve()
    L = _l.lib()
    fleet = kind == "fleet"
    h = c.h._f if fleet else c.h._h
    nj, nx = c.model["nj"], c.model["nx"]
    host_rs = np.ascontiguousarray(c.robot_states(1))
    pinned = torch.tensor(host_rs).pin_memory()
    rs_dev = cuda(host_rs)
    q = torch.full((c.B, nj), 7.0, dtype=torch.float64, device="cuda")
    st = torch.full((c.B,), 7, dtype=torch.int32, device="cuda")
    vp = C.c_void_p
    ja = L.b200sqp_fleet_joint_actions_dev if fleet else L.b200sqp_joint_actions_dev
    foreign = [vp(host_rs.ctypes.data), vp(pinned.data_ptr())]
    if torch.cuda.device_count() > 1:
        foreign.append(vp(torch.zeros_like(q, device="cuda:1").data_ptr()))
    for p in foreign:
        assert ja(h, C.c_double(0.01), p, C.c_int(1), vp(q.data_ptr()), None, None, None, None, None, vp(st.data_ptr()), None) == EINVAL
        assert ja(h, C.c_double(0.01), vp(rs_dev.data_ptr()), C.c_int(1), p, None, None, None, None, None, None, None) == EINVAL
        if fleet:
            rc = L.b200sqp_fleet_download_dev(h, C.c_int(int(c.h.n_nodes.max())), p, None, None, None, None, None)
        else:
            rc = L.b200sqp_download_dev(h, p, None, None, None, None)
        assert rc == EINVAL
    torch.cuda.synchronize()
    assert (q == 7.0).all() and (st == 7).all()   # nothing was enqueued
    n = np.zeros(c.B, np.int32)
    args = (C.c_int(c.B), C.c_double(DT_MPC), C.c_double(c.horizon), vp(np.ascontiguousarray(c.x0s).ctypes.data))
    gid = np.ascontiguousarray([c.solver._gait_names.index(g) for g in c.gaits], dtype=np.int32)
    rest = (gid.ctypes.data_as(_l.ip), np.ascontiguousarray(c.starts, dtype=np.float64).ctypes.data_as(_l.dp),
            np.ascontiguousarray(c.cmds).ctypes.data_as(_l.dp), C.c_int(1), n.ctypes.data_as(_l.ip))
    if fleet:
        G = C.c_int32()
        rc = L.b200sqp_fleet_build_instances_dev(h, *args, *rest, C.byref(G), None)
    else:
        rc = L.b200sqp_build_instances_dev(h, *args, *rest, None)
    assert rc == EINVAL
    with pytest.raises(ValueError, match="robot_state: the tensor is on cpu"):
        c.h.joint_actions_device(0.01, torch.tensor(host_rs))
