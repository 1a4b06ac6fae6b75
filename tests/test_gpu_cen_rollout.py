"""Policy roll-out on centroidal handles (b200sqp_cen_rollout_policy, cen_policy_rollout_kernel) after real centroidal solves (B = 8, horizon
1.2 s, both centroidal model types): against the restatement of MRT_BASE::rolloutPolicy around the oracle's centroidal flow map (rollout_ref.py)
for both controllers, the closed loop build(warm = 2) -> solve -> roll-out equal bit for bit to the same loop driven through host copies, and the
error paths."""
import numpy as np
import pytest

import oracle_lib as orc
import rollout_ref
from test_gpu_cen_builder import make_inputs
from wb_humanoid_mpc_b200 import abi, model_loader
from wb_humanoid_mpc_b200.lib import B200SqpError

pytestmark = pytest.mark.gpu
MRT_DT = 1.0 / 100.0   # the centroidal dummy simulation: one 1/100 s MRT step per MPC cycle
B, HORIZON = 8, 1.2
EINVAL, ESTATE = -1, -5


@pytest.fixture(scope="module", params=[0, 1], ids=["full", "srbd"])
def model(request):
    m = dict(model_loader.load_packaged_model("g1_centroidal"))
    m["centroidalModelType"] = request.param
    return m


def solved(model, feedback, seed=21):
    from wb_humanoid_mpc_b200.solver import B200SqpSolver

    x0s, cmds = make_inputs(model, np.random.default_rng(seed), B)
    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=1, use_feedback_policy=int(feedback)))
    s.build_instances(0.0, HORIZON, x0s, ["walk"] * B, [0.0] * B, cmds)
    s.solve()
    return s, x0s, cmds


def plans(solver):
    inp = solver.download_instances()
    sol = solver.primal_solution()
    return [(dict(t_nodes=inp["t_nodes"][b], node_event=inp["node_event"][b], contact_flags=inp["contact_flags"][b], x=sol["x"][b], u=sol["u"][b]),
             sol.get("K", [None] * solver.batch)[b]) for b in range(solver.batch)]


def plan_state(plan, t):
    i, a = rollout_ref.time_segment(t, list(plan["t_nodes"]))
    return a * plan["x"][i] + (1 - a) * plan["x"][i + 1]


def rel(a, b):
    return float(np.max(np.abs(a - b)) / max(1e-300, np.max(np.abs(b))))


@pytest.mark.parametrize("feedback", [False, True], ids=["feedforward", "feedback"])
def test_kernel_matches_the_reference_restatement(model, feedback):
    solver, _, _ = solved(model, feedback)
    ps = plans(solver)
    te = min(float(p["t_nodes"][k]) for p, _ in ps for k in range(len(p["t_nodes"])) if p["node_event"][k] == 1)
    flow = orc.CenOracle(model).flow_map
    rs = abi.cen_default_rollout_settings()
    rng = np.random.default_rng(4)
    for t in (0.05, te - 0.4 * MRT_DT):   # a step without and one with a contact switch inside it
        xs = np.array([plan_state(p, t) for p, _ in ps])
        xs[:, 0:6] += rng.normal(0.0, 0.2, (B, 6))   # a push on the normalized momentum
        dev = solver.cen_rollout_policy(t, MRT_DT, x_start=xs)
        assert dev["x"].shape == (B, 35)
        for b, (p, K) in enumerate(ps):
            ref = rollout_ref.rollout_policy(flow, p, t, MRT_DT, xs[b], K=K, abs_tol=rs.abs_tol, rel_tol=rs.rel_tol, time_step=rs.time_step,
                                             max_steps_per_second=rs.max_steps_per_second)
            assert dev["status"][b] == ref["status"] == 0
            assert tuple(dev["n_steps"][b]) == (ref["accepted"], ref["rejected"], ref["calls"]), (b, t)
            assert dev["mode"][b] == ref["mode"]
            assert rel(dev["x"][b], ref["x"]) < 1e-12 and rel(dev["u"][b], ref["u"]) < 1e-12, (b, t)


def closed_loops_agree(model, feedback, cycles=40):
    """cycles of build(warm = 2) -> solve -> roll-out without host copies equal, bit for bit, the loop that downloads x_end and uploads it as the
    next measured state (build_instances(x0 = x_end, warm = 1))"""
    dev, x0s, cmds = solved(model, feedback)
    host, _, _ = solved(model, feedback)
    gaits, start = ["walk"] * B, [0.0] * B
    for c in range(cycles):
        t = c * MRT_DT
        rd = dev.cen_rollout_policy(t, MRT_DT)
        rh = host.cen_rollout_policy(t, MRT_DT)
        assert np.array_equal(rd["x"], rh["x"]) and np.array_equal(rd["u"], rh["u"]) and not rd["status"].any() and not rh["status"].any(), c
        dev.build_instances(t + MRT_DT, HORIZON, None, gaits, start, cmds, warm="rollout")
        host.build_instances(t + MRT_DT, HORIZON, rh["x"], gaits, start, cmds, warm=True)
        assert np.array_equal(dev.download_instances()["x0"], rh["x"])
        dev.solve()
        host.solve()
        sd, sh = dev.primal_solution(), host.primal_solution()
        assert np.array_equal(sd["x"], sh["x"]) and np.array_equal(sd["u"], sh["u"]), c
        if feedback:
            assert np.array_equal(sd["K"], sh["K"]), c


def test_closed_loop_on_the_device_equals_the_host_driven_loop(model):
    """the feed-forward policy of the centroidal task.info (useFeedbackPolicy false), both model types, 40 cycles"""
    closed_loops_agree(model, False)


def test_closed_loop_with_feedback_equals_the_host_driven_loop():
    """the linear feedback policy (x, u and K bit for bit), 40 cycles, full centroidal dynamics.  (The SRBD model is left out here: under the
    feedback policy of these one-iteration solves two of its eight instances exceed the flow-map call budget from cycle 4 on and diverge.)"""
    m = dict(model_loader.load_packaged_model("g1_centroidal"))
    m["centroidalModelType"] = 0
    closed_loops_agree(m, True)


def test_call_order_and_handle_kind_are_checked(model):
    from wb_humanoid_mpc_b200.solver import B200SqpSolver

    x0s, cmds = make_inputs(model, np.random.default_rng(2), 2)
    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=1))
    s.build_instances(0.0, HORIZON, x0s, ["walk"] * 2, [0.0] * 2, cmds)
    with pytest.raises(B200SqpError) as e:   # no solve yet
        s.cen_rollout_policy(0.0, MRT_DT)
    assert e.value.code == ESTATE
    s.solve()
    with pytest.raises(B200SqpError) as e:   # warm = 2 without a roll-out
        s.build_instances(MRT_DT, HORIZON, None, ["walk"] * 2, [0.0] * 2, cmds, warm="rollout")
    assert e.value.code == ESTATE
    with pytest.raises(B200SqpError) as e:   # a negative duration
        s.cen_rollout_policy(0.0, -MRT_DT)
    assert e.value.code == EINVAL
    for bad in (dict(abs_tol=0.0), dict(rel_tol=-1.0), dict(time_step=0.0), dict(max_steps_per_second=0.5)):
        with pytest.raises(B200SqpError) as e:
            s.cen_rollout_policy(0.0, MRT_DT, settings=abi.cen_default_rollout_settings(**bad))
        assert e.value.code == EINVAL, bad
    with pytest.raises(B200SqpError) as e:   # the whole-body entry point keeps refusing centroidal handles
        s.rollout_policy(0.0, MRT_DT)
    assert e.value.code == EINVAL
    # the simulated state is the next measured state
    r = s.cen_rollout_policy(0.0, MRT_DT)
    s.build_instances(MRT_DT, HORIZON, None, ["walk"] * 2, [0.0] * 2, cmds, warm="rollout")
    assert np.array_equal(s.download_instances()["x0"], r["x"])
    s.solve()
    # a roll-out past the plan's last node holds the policy at its end (the reference only warns)
    r = s.cen_rollout_policy(MRT_DT + HORIZON - 0.005, 0.05)
    assert not r["status"].any() and np.all(np.isfinite(r["x"]))
    wmodel = model_loader.load_packaged_model()
    ws = B200SqpSolver(wmodel, abi.default_settings(wmodel, sqp_iteration=1))
    with pytest.raises(B200SqpError) as e:
        ws.cen_rollout_policy(0.0, MRT_DT)
    assert e.value.code == EINVAL
