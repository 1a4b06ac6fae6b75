"""The CPU restatement of the reference's policy roll-out (rollout_ref.py) against the reference's own test recipes and independent checks:
    IntegrationTest.cpp::SecondOrderSystem_ODE45_OCS2 and testRungeKuttaDormandPrince5.cpp::integrateLinearSystem (x(10) = (0, 1) to 1e-3, first
    and last time stamps to 1e-6); the Dormand-Prince stepper against scipy's DOP853 at rtol 1e-12 on that system and on the G1 flow map under a
    fixed feedback policy; findActiveModesTimeInterval's edge cases, cross-checked with the time grid of test_oracle_spreading.py; the
    controller against the host layer's policy message (host/MpcPolicyMsg.hpp evaluatePolicySample) at node times and across a PreEvent /
    PostEvent pair."""
import ctypes as C

import numpy as np
import pytest
from scipy.integrate import solve_ivp

import oracle_lib as orc
import rollout_ref as rr

A = np.array([[-2.0, -1.0], [1.0, 0.0]])
Bv = np.array([1.0, 0.0])


def linear_system(x, t):
    return A @ x + Bv * 1.0


def test_integrate_linear_system():
    """testRungeKuttaDormandPrince5.cpp::integrateLinearSystem: integrateAdaptive(x0 = 0, [0, 10], dt = 0.01) with the default tolerances"""
    ts, xs, _ = rr.integrate_adaptive(linear_system, np.zeros(2), 0.0, 10.0, 0.01, 1e-6, 1e-3)
    assert abs(ts[0] - 0.0) < 1e-6 and abs(ts[-1] - 10.0) < 1e-6
    assert np.allclose(xs[0], 0.0)
    assert abs(xs[-1][0] - 0.0) < 1e-3 and abs(xs[-1][1] - 1.0) < 1e-3


def test_second_order_system_under_a_linear_controller():
    """IntegrationTest.cpp::SecondOrderSystem_ODE45_OCS2: the same system as a controlled system, LinearController(time stamps {0, 10}, uff = 1,
    K = 0), rolled out over [0, 10] (one interval, no events)"""
    ctrl = rr.PlanController([0.0, 10.0], [0, 0], np.zeros((2, 2)), np.ones((1, 1)), np.zeros((1, 1, 2)))
    r = rr.time_triggered_rollout(lambda x, u: A @ x + Bv * u[0], ctrl, 0.0, np.zeros(2), 10.0, [], abs_tol=1e-6, rel_tol=1e-3, time_step=0.01)
    assert r["status"] == rr.OK
    assert abs(r["t"][0] - rr.WEAK_EPS) < 1e-6 and abs(r["t"][-1] - 10.0) < 1e-6
    assert abs(r["x"][-1][0]) < 1e-3 and abs(r["x"][-1][1] - 1.0) < 1e-3
    assert np.allclose(r["u"], 1.0)


def test_dp5_against_dop853_on_the_linear_system():
    """every accepted step stays within the requested tolerance of the exact step from the same state, in the stepper's own error scale
    absTol + relTol (|x| + dt |dxdt|) (the step control bounds the local error; the global error of a 10 s run may add up beyond it)"""
    ts, xs, dp = rr.integrate_adaptive(linear_system, np.array([0.3, -0.2]), 0.0, 10.0, 0.01, 1e-6, 1e-3)
    for k in range(len(ts) - 1):
        ref = solve_ivp(lambda t, x: linear_system(x, t), (ts[k], ts[k + 1]), xs[k], method="DOP853", rtol=1e-12, atol=1e-12).y[:, -1]
        h = ts[k + 1] - ts[k]
        scale = 1e-6 + 1e-3 * (np.abs(xs[k]) + h * np.abs(linear_system(xs[k], ts[k])))
        assert np.all(np.abs(xs[k + 1] - ref) <= scale), k
    end = solve_ivp(lambda t, x: linear_system(x, t), (0.0, 10.0), [0.3, -0.2], method="DOP853", rtol=1e-12, atol=1e-12).y[:, -1]
    assert np.max(np.abs(xs[-1] - end)) < 1e-3
    assert dp.accepted > 10 and dp.calls == 1 + 6 * (dp.accepted + dp.rejected)


def test_dp5_against_dop853_on_the_g1_flow_map():
    """one MRT step (1/80 s) of a walking plan's feedback policy from a pushed state, no event inside: the roll-out's end state agrees with a
    rtol 1e-12 DOP853 solution within the requested tolerance"""
    from test_emu_rollout import MRT_DT, walking_plan

    model, plan, K = walking_plan()
    wb = orc.WbOracle(model)
    t0 = 0.05
    i, a = rr.time_segment(t0, list(plan["t_nodes"]))
    x0 = a * plan["x"][i] + (1 - a) * plan["x"][i + 1]
    x0[29:35] += np.random.default_rng(1).normal(0.0, 0.2, 6)
    ctrl = rr.PlanController(plan["t_nodes"], plan["node_event"], plan["x"], plan["u"], K)
    r = rr.time_triggered_rollout(wb.flow_map, ctrl, t0, x0, t0 + MRT_DT, [])
    assert r["status"] == rr.OK
    a0 = r["t"][0]   # (the interval starts weakEpsilon after t0)
    ref = solve_ivp(lambda t, x: wb.flow_map(x, ctrl.compute_input(t, x)), (a0, t0 + MRT_DT), r["x"][0], method="DOP853", rtol=1e-12, atol=1e-12)
    want = ref.y[:, -1]
    assert np.all(np.abs(r["x"][-1] - want) <= 1e-5 + 1e-3 * np.abs(want)), np.max(np.abs(r["x"][-1] - want))


def test_active_mode_intervals_edge_cases():
    iv = rr.find_active_modes_time_interval(1.0, 2.0, [1.0, 1.5, 2.0, 2.5])
    # an event at the initial time is excluded, an event at the final time is included and leaves a degenerate last interval
    assert [b for _, b in iv] == [1.5, 2.0, 2.0]
    assert iv[0][0] == 1.0 + rr.WEAK_EPS and iv[1][0] == 1.5 + rr.WEAK_EPS
    assert iv[2][0] == iv[2][1] == 2.0
    # a degenerate interval contributes one sample (its end time, the state it starts from)
    ctrl = rr.PlanController([0.0, 3.0], [0, 0], np.zeros((2, 1)), np.zeros((1, 1)))
    r = rr.time_triggered_rollout(lambda x, u: -x, ctrl, 1.0, np.ones(1), 2.0, [1.0, 1.5, 2.0, 2.5])
    assert r["t"][-1] == 2.0 and np.array_equal(r["x"][-1], r["x"][-2]) and len(r["post_event_indices"]) == 2
    assert r["t"][r["post_event_indices"][-1]] == 2.0 and r["t"][r["post_event_indices"][-1] - 1] == r["t"][-2]


@pytest.mark.parametrize("case", ["final_time_is_the_same_as_event_time_1", "partially_matching_modes", "fully_matched_modes"])
def test_interval_boundaries_agree_with_the_spreading_time_grid(case):
    """the same intervals as test_oracle_spreading.py's restatement: first / last sample and the samples around every event"""
    from test_oracle_spreading import CASES, rollout

    ev, modes, _, _, period, _ = CASES[case]
    t_s, _, post_s, _ = rollout(ev, modes, period)
    ctrl = rr.PlanController([0.0, 5.0], [0, 0], np.zeros((2, 1)), np.zeros((1, 1)))
    r = rr.time_triggered_rollout(lambda x, u: -x, ctrl, period[0], np.ones(1), period[1], ev, time_step=0.01)
    t_r, post_r = r["t"], r["post_event_indices"]
    assert len(post_r) == len(post_s)
    assert t_r[0] == t_s[0] and t_r[-1] == t_s[-1]
    for pr, ps in zip(post_r, post_s):
        assert t_r[pr - 1] == t_s[ps - 1] and t_r[pr] == t_s[ps]


def test_controller_matches_the_policy_message():
    """PlanController (built as the shim's toPrimalSolution builds it) equals MpcPolicyMsg.hpp's evaluatePolicySample at every node time for the
    node's own state, and at the PreEvent / PostEvent pair of a switch (at the event time the PreEvent sample applies, weakEpsilon later the
    PostEvent one); float32 wire precision."""
    from test_emu_rollout import walking_plan

    from wb_humanoid_mpc_b200 import host_lib

    model, plan, K = walking_plan()
    n, nx, nu = len(plan["t_nodes"]), 58, 35
    ctrl = rr.PlanController(plan["t_nodes"], plan["node_event"], plan["x"], plan["u"], K)
    L = host_lib.lib()
    L.b200host_policy_msg.restype = C.c_int
    dp, u8p = C.POINTER(C.c_double), C.POINTER(C.c_uint8)
    tt = np.ascontiguousarray(plan["t_nodes"], dtype=np.float64)
    ev = np.ascontiguousarray(plan["node_event"], dtype=np.uint8)
    xx, uu = np.ascontiguousarray(plan["x"]), np.ascontiguousarray(plan["u"])
    Kc = np.ascontiguousarray(np.swapaxes(K, 1, 2))
    data = np.zeros((n, nu * (1 + nx)), dtype=np.float32)
    post = np.zeros(n, dtype=np.uint16)
    n_post = C.c_int(0)

    def sample(k):
        up = np.zeros(nu)
        rc = L.b200host_policy_msg(n, nx, nu, tt.ctypes.data_as(dp), ev.ctypes.data_as(u8p), xx.ctypes.data_as(dp), uu.ctypes.data_as(dp), Kc.ctypes.data_as(dp),
                                   data.ctypes.data_as(C.POINTER(C.c_float)), data.size, post.ctypes.data_as(C.POINTER(C.c_uint16)), C.byref(n_post), k,
                                   xx[k].ctypes.data_as(dp), up.ctypes.data_as(dp))
        assert rc == nu * (1 + nx), L.b200host_last_error()
        return up

    scale = np.max(np.abs(plan["u"]))
    for k in range(n):
        if plan["node_event"][k] == 2:
            continue   # a PostEvent node shares its time with the PreEvent node before it: at that time the PreEvent sample applies
        assert np.allclose(ctrl.compute_input(float(tt[k]), xx[k]), sample(k), atol=2e-6 * scale, rtol=0), k
    pre = int(np.nonzero(ev == 1)[0][0])
    te = float(tt[pre])
    assert np.allclose(ctrl.compute_input(te, xx[pre]), sample(pre), atol=2e-6 * scale, rtol=0)
    i, a = rr.time_segment(te + rr.WEAK_EPS, list(tt))
    assert i == pre + 1 and a > 1.0 - 1e-6   # just after the switch the PostEvent node's policy applies
    assert np.allclose(ctrl.compute_input(float(tt[pre + 1]) + rr.WEAK_EPS, xx[pre + 1]), sample(pre + 1), atol=2e-6 * scale + 1e-6, rtol=0)
