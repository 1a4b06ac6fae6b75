"""MRT-side queries on the device (b200sqp_mrt_query / _dev, b200sqp_fleet_mrt_query / _dev, b200sqp_fleet_download_value_function) after
real solves: the value function and the feedback gain at t against the restatement of getValueFunction / getLinearFeedbackGain
(mrt_query_ref.py) over the downloaded P, p, K and plan, on plain handles (whole-body and centroidal, a small batch and the benchmark's
B = 256 over a 3.5 s horizon, one and three SQP iterations) and on fleets of mixed schedules, also inside a stateful loop with the motion
manager and resets; the device-pointer twins bit-identical to the host path and ordered behind a producer kernel; queries that change
nothing in the device loop or in the next solve; and every error code."""
import ctypes as C

import numpy as np
import pytest

import mrt_query_ref as ref
import test_gpu_builder
import test_gpu_cen_builder
import test_gpu_fleet
from test_gpu_mrt import LOOP, model_of
from wb_humanoid_mpc_b200 import abi
from wb_humanoid_mpc_b200 import lib as _l

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

EINVAL, ESTATE = -1, -5
FAMS = ["wb", "cen"]
SIZES = {"small": (8, None), "bench": (256, 3.5)}   # (B, horizon; None: the family's loop horizon)


def fam_model(fam):
    return model_of("wb" if fam == "wb" else "full")


def inputs(fam, model, B, seed):
    make = test_gpu_builder.make_inputs if fam == "wb" else test_gpu_cen_builder.make_inputs
    return make(model, np.random.default_rng(seed), B)


def settings(model, iters=1, value=True, gain=True):
    return abi.default_settings(model, sqp_iteration=iters, use_feedback_policy=int(gain), create_value_function=int(value))


def plain(fam, B, horizon=None, iters=1, value=True, gain=True, seed=21):
    from wb_humanoid_mpc_b200.solver import B200SqpSolver

    model = fam_model(fam)
    x0s, cmds = inputs(fam, model, B, seed)
    s = B200SqpSolver(model, settings(model, iters, value, gain))
    s.build_instances(0.0, horizon or LOOP["wb" if fam == "wb" else "full"][0], x0s, ["walk"] * B, [0.0] * B, cmds)
    s.solve()
    return s, model, x0s


def query_times(T, ev):
    te = float(T[int(np.flatnonzero(ev == 1)[0])])
    return {"before": float(T[0]) - 0.3, "node": float(T[3]), "segment": 0.5 * (float(T[2]) + float(T[3])) + 1.3e-4, "event": te,
            "past": float(T[-1]) + 0.05}


def restate(t, t_nodes, events, n_nodes, P, p, K, x):
    """the restatement per instance over the downloads (P [B, m, nx, nx], p [B, m, nx], K [B, m-1, nu, nx], rows cut to n_nodes)"""
    out = {"dfdxx": [], "dfdx": [], "K": []}
    for b, n in enumerate(n_nodes):
        r = ref.query(t, t_nodes[b][:n], events[b][:n], P=P[b][:n], p=p[b][:n], K=K[b][: n - 1], x=x[b])
        for k in out:
            out[k].append(r[k])
    return {k: np.array(v) for k, v in out.items()}


def assert_close(dev, host, tol=1e-12):
    for k in ("dfdxx", "dfdx", "K"):
        d = dev[k].cpu().numpy() if hasattr(dev[k], "cpu") else dev[k]
        assert d.shape == host[k].shape, (k, d.shape, host[k].shape)
        for b in range(d.shape[0]):
            scale = max(1e-300, float(np.max(np.abs(host[k][b]))))
            assert float(np.max(np.abs(d[b] - host[k][b]))) <= tol * scale, (k, b)


def same(dev, host):
    for k in host:
        d = dev[k].cpu().numpy() if hasattr(dev[k], "cpu") else dev[k]
        assert np.array_equal(d, host[k]), k


@pytest.mark.parametrize("iters", [1, 3])
@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("fam", FAMS)
def test_plain_query_matches_the_restatement(fam, size, iters):
    B, horizon = SIZES[size]
    s, model, x0s = plain(fam, B, horizon, iters)
    inp, sol = s.download_instances(), s.primal_solution()
    P, p = s.value_function()
    n = np.full(B, s.n_nodes)
    x = x0s + np.random.default_rng(4).normal(0.0, 0.01, x0s.shape)
    for name, t in query_times(inp["t_nodes"][0], inp["node_event"][0]).items():
        dev = s.mrt_query(t, x)
        assert_close(dev, restate(t, inp["t_nodes"], inp["node_event"], n, P, p, sol["K"], x))


def mixed_fleet(fam, B=24, seed=31, iters=1):
    from wb_humanoid_mpc_b200.solver import B200SqpFleet, B200SqpSolver

    model = fam_model(fam)
    x0s, cmds = inputs(fam, model, B, seed)
    s = B200SqpSolver(model, settings(model, iters))
    f = B200SqpFleet(s)
    gaits, starts = test_gpu_fleet.mixed_batch(model, np.random.default_rng(seed), B)
    f.build_instances(0.0, LOOP["wb" if fam == "wb" else "full"][0], x0s, gaits, starts, cmds)
    assert f.n_groups >= 2
    f.solve()
    return s, f, model, x0s


@pytest.mark.parametrize("fam", FAMS)
def test_fleet_value_function_and_query(fam):
    s, f, model, x0s = mixed_fleet(fam)
    m = int(f.n_nodes.max())
    P, p, n = f.value_function(m + 2)
    assert np.array_equal(n, f.n_nodes) and P.shape == (f.batch, m + 2, model["nx"], model["nx"])
    for b in range(f.batch):   # zero padding past each instance's node count
        assert not P[b, n[b]:].any() and not p[b, n[b]:].any(), b
    # each instance's rows equal the value function of the same instances solved in plain handles, one per node count
    inp = f.download_instances()
    for nn, (idx, h) in test_gpu_fleet.per_group_plain(model, f, inp, create_value_function=1, use_feedback_policy=1).items():
        Ph, ph = h.value_function()
        assert np.array_equal(P[idx, :nn], Ph) and np.array_equal(p[idx, :nn], ph), nn
    sol = f.primal_solution()
    x = x0s + np.random.default_rng(5).normal(0.0, 0.01, x0s.shape)
    T0 = inp["t_nodes"][0][: n[0]]
    for t in (float(T0[0]) - 0.3, float(T0[4]), 0.2113, float(T0[-1]) + 0.05):
        assert_close(f.mrt_query(t, x), restate(t, inp["t_nodes"], inp["node_event"], n, P, p, sol["K"], x))
    te = min(float(inp["t_nodes"][b][k]) for b in range(f.batch) for k in range(n[b]) if inp["node_event"][b][k] == 1)
    assert_close(f.mrt_query(te, x), restate(te, inp["t_nodes"], inp["node_event"], n, P, p, sol["K"], x))


@pytest.mark.parametrize("fam", FAMS)
def test_fleet_stateful_loop_with_motion_manager_and_resets(fam):
    """the motion manager picks the gaits and one instance is reset on the way; every cycle's query equals the restatement over that
    cycle's downloads"""
    import test_gpu_resets as R
    from wb_humanoid_mpc_b200.solver import B200SqpFleet, B200SqpSolver

    model = R.model_loader.load_packaged_model("g1_wb" if fam == "wb" else "g1_centroidal")
    B = 9
    rng = np.random.default_rng(17)
    s = B200SqpSolver(model, settings(model))
    if fam == "wb":
        s.set_gait_schedule(True)
        s.set_motion_manager()
    else:
        s.cen_set_gait_schedule(True)
        s.cen_set_motion_manager()
    f = B200SqpFleet(s)
    raw = R.cmds(B, 0.5)
    raw[::3, 0] = 0.0   # some instances keep standing
    f.set_reset_states(*R.reset_rows(model, B))
    f.build_instances(0.0, R.HORIZON, R.standing_x0(model, rng, B), ["stance"] * B, [0.5] * B, raw)
    t = 0.0
    for c in range(8):
        f.solve()
        ro = f.rollout_policy(t, R.DT_MPC)
        inp, sol = f.download_instances(), f.primal_solution()
        P, p, n = f.value_function()
        tq = t + 0.005
        dev = f.mrt_query(tq)   # x = NULL: the roll-out's end state
        assert_close(dev, restate(tq, inp["t_nodes"], inp["node_event"], n, P, p, sol["K"], ro["x"]))
        t += R.DT_MPC
        if c == 4:
            f.request_resets([1])
        f.build_instances(t, R.HORIZON, None, None, [0.0] * B, raw, warm="rollout")
    assert f.episodes()["episode"][1] == 1 and f.n_groups >= 1


def cuda(a):
    return torch.tensor(np.asarray(a), dtype=torch.float64, device="cuda")


@pytest.mark.parametrize("kind", ["plain", "fleet"])
@pytest.mark.parametrize("fam", FAMS)
def test_device_twins_are_bit_identical(fam, kind):
    if kind == "plain":
        s, model, x0s = plain(fam, 16)
        h = s
    else:
        s, h, model, x0s = mixed_fleet(fam, B=16)
    x = x0s + np.random.default_rng(6).normal(0.0, 0.01, x0s.shape)
    t = 0.1371
    host = h.mrt_query(t, x)
    same(h.mrt_query_device(t, cuda(x)), host)
    # a producer kernel on the call's stream, just before the call: its x is the one read
    st = torch.cuda.Stream()
    xd = torch.zeros_like(cuda(x))
    src = cuda(x)
    with torch.cuda.stream(st):
        torch.cuda._sleep(20_000_000)
        xd.copy_(src)
        dev = h.mrt_query_device(t, xd, stream=st)
    st.synchronize()
    same(dev, host)
    # x = NULL after a roll-out is that roll-out's end state
    ro = h.cen_rollout_policy(0.0, 0.01) if (fam == "cen" and kind == "plain") else h.rollout_policy(0.0, 0.01)
    same(h.mrt_query(t), h.mrt_query(t, ro["x"]))
    same(h.mrt_query_device(t), h.mrt_query(t, ro["x"]))
    # the parts alone equal the parts of the whole
    same(h.mrt_query(t, x, gain=False), {k: host[k] for k in ("dfdxx", "dfdx")})
    same(h.mrt_query_device(t, cuda(x), value=False), {"K": host["K"]})


class Loop:
    """a closed loop build(warm = "rollout") -> solve -> roll-out on a plain handle (every instance walking) or a fleet (mixed schedules)"""

    def __init__(self, fam, kind, B=12, seed=41):
        from wb_humanoid_mpc_b200.solver import B200SqpFleet, B200SqpSolver

        self.fam, self.kind = fam, kind
        self.model = fam_model(fam)
        self.x0s, self.cmds = inputs(fam, self.model, B, seed)
        self.solver = B200SqpSolver(self.model, settings(self.model))
        if kind == "fleet":
            self.gaits, self.starts = test_gpu_fleet.mixed_batch(self.model, np.random.default_rng(seed), B)
            self.h = B200SqpFleet(self.solver)
        else:
            self.gaits, self.starts = ["walk"] * B, np.zeros(B)
            self.h = self.solver
        self.horizon, self.dt = LOOP["wb" if fam == "wb" else "full"]

    def build(self, t0, warm):
        self.h.build_instances(t0, self.horizon, None if warm else self.x0s, self.gaits, self.starts, self.cmds, warm="rollout" if warm else False)

    def rollout(self, t0):
        if self.kind == "plain" and self.fam == "cen":
            return self.h.cen_rollout_policy(t0, self.dt)
        return self.h.rollout_policy(t0, self.dt)


@pytest.mark.parametrize("kind", ["plain", "fleet"])
@pytest.mark.parametrize("fam", FAMS)
def test_queries_change_nothing_in_the_device_loop(fam, kind):
    """the same closed loop with and without queries between its calls: bit-identical plans, roll-outs, joint actions and launch counts"""
    a, b = Loop(fam, kind), Loop(fam, kind)
    nx = a.model["nx"]
    for c in range(5):
        t0 = c * a.dt
        for lp in (a, b):
            lp.build(t0, warm=c > 0)
        same(a.h.download_instances(), b.h.download_instances())
        B = a.h.batch
        for lp in (a, b):
            lp.h.solve()
        if kind == "plain":
            assert a.solver.launch_count() == b.solver.launch_count()
        a.h.mrt_query(t0, np.zeros((B, nx)))
        a.h.mrt_query_device(t0 + 0.003, cuda(np.ones((B, nx))), value=(c % 2 == 0))
        ra, rb = a.rollout(t0), b.rollout(t0)
        same(ra, rb)
        a.h.mrt_query(t0 + 0.005)
        a.h.mrt_query_device(t0 + 0.006)
        same(a.h.joint_actions(t0 + 0.005), b.h.joint_actions(t0 + 0.005))
        a.h.mrt_query(t0 + 0.007)
        pa, pb = a.h.primal_solution(), b.h.primal_solution()
        same({k: v for k, v in pa.items() if k != "log"}, {k: v for k, v in pb.items() if k != "log"})


def test_error_codes():
    from wb_humanoid_mpc_b200.solver import B200SqpFleet, B200SqpSolver

    L = _l.lib()
    model = fam_model("wb")
    nx, nu = model["nx"], model["nu"]
    x0s, cmds = inputs("wb", model, 2, 7)
    out = np.zeros((2, nx, nx))
    P = out.ctypes.data_as(_l.dp)

    def raw(h, t=0.0, x=None, dfdxx=P, dfdx=None, K=None, fn=L.b200sqp_mrt_query):
        return fn(h, C.c_double(t), x, dfdxx, dfdx, K, None)

    assert raw(None) == EINVAL
    s = B200SqpSolver(model, settings(model, value=False, gain=False))
    assert raw(s._h) == ESTATE   # nothing solved yet
    s.build_instances(0.0, 1.1, x0s, ["walk"] * 2, [0.0] * 2, cmds)
    assert raw(s._h, dfdxx=None) == 0   # nothing asked: nothing to check
    s.solve()
    assert raw(s._h, t=float("nan")) == EINVAL
    assert raw(s._h, t=float("inf")) == EINVAL
    assert raw(s._h) == ESTATE   # create_value_function = 0
    Kout = np.zeros((2, nu * nx))
    assert raw(s._h, dfdxx=None, K=Kout.ctypes.data_as(_l.dp)) == ESTATE   # feed-forward policy
    s.close()
    s = B200SqpSolver(model, settings(model))
    s.build_instances(0.0, 1.1, x0s, ["walk"] * 2, [0.0] * 2, cmds)
    s.solve()
    pv = np.zeros((2, nx))
    assert raw(s._h, dfdx=pv.ctypes.data_as(_l.dp)) == ESTATE   # x = NULL before a roll-out
    assert raw(s._h, dfdxx=P, fn=L.b200sqp_mrt_query_dev) == EINVAL   # host memory on the _dev path
    xd = cuda(x0s)
    assert raw(s._h, x=C.c_void_p(xd.data_ptr()), dfdx=pv.ctypes.data_as(_l.dp), dfdxx=None, fn=L.b200sqp_mrt_query_dev) == EINVAL
    f = B200SqpFleet(s)
    assert raw(s._h) == ESTATE   # a fleet is attached
    assert raw(f._f, fn=L.b200sqp_fleet_mrt_query) == ESTATE   # before the fleet's first build
    assert raw(None, fn=L.b200sqp_fleet_mrt_query) == EINVAL
    assert L.b200sqp_fleet_download_value_function(f._f, C.c_int(50), P, pv.ctypes.data_as(_l.dp), None) == ESTATE
    f.build_instances(0.0, 1.1, x0s, ["walk", "stance"], [0.0, 0.5], cmds)
    f.solve()
    assert L.b200sqp_fleet_download_value_function(f._f, C.c_int(int(f.n_nodes.max()) - 1), P, pv.ctypes.data_as(_l.dp), None) == EINVAL
    assert L.b200sqp_fleet_download_value_function(f._f, C.c_int(int(f.n_nodes.max())), None, pv.ctypes.data_as(_l.dp), None) == EINVAL
    assert raw(f._f, t=float("nan"), fn=L.b200sqp_fleet_mrt_query_dev) == EINVAL
