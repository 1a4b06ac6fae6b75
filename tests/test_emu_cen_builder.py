"""The device-side instance builder on centroidal handles (wb_humanoid_mpc_b200/csrc/wb_builder.cuh: bldCenBaseVelocity, bldCenTargetKnots and
the shared schedule / grid / initializer functions) executed on the CPU harness against the host restatement of SolverBase::preRun for the
centroidal MPC (references.build_instance with the centroidal target rule), for both centroidal model types: integer arrays exactly,
floating-point arrays to 1e-12 relative, the padding of the device state rows exactly zero.  The base velocity Ab^-1 hbar is checked against
the oracle's flow map (full centroidal dynamics) and the closed form of the single-rigid-body model."""
import numpy as np
import pytest

import bld_emu_lib as cbe
import oracle_lib as orc
from wb_humanoid_mpc_b200 import centroidal, model_loader, references
from wb_humanoid_mpc_b200.solver import stack_instances

FLOAT_KEYS = ["x0", "x_init", "u_init", "t_nodes", "swing_ref", "impact_factor", "arm_phase", "x_ref"]
INT_KEYS = ["node_event", "contact_flags"]


@pytest.fixture(scope="module", params=[0, 1], ids=["full", "srbd"])
def model(request):
    m = dict(model_loader.load_packaged_model("g1_centroidal"))
    m["centroidalModelType"] = request.param
    return m


@pytest.fixture(scope="module")
def host_base_velocity(model):
    """Ab^-1 hbar on the host: the oracle's flow map at u = 0 over the mass (full model), the closed form of centroidal.py (SRBD)"""
    if model["centroidalModelType"] == 1:
        return lambda x: centroidal.srbd_base_velocity(model, np.asarray(x, float))
    o = orc.CenOracle(model)
    m = sum(model["mass"])
    return lambda x: o.flow_map(x, np.zeros(model["nu"]))[6:12] / m


def make_inputs(model, rng, B):
    """perturbed measured states, all but the first with a non-zero normalized momentum, and velocity commands"""
    x0s, cmds = [], []
    for b in range(B):
        x0 = np.array(model["x_init"], float)
        x0[6:8] += rng.uniform(-0.02, 0.02, 2)
        x0[9:12] += rng.uniform(-0.05, 0.05, 3)
        x0[12:] += rng.uniform(-0.1, 0.1, model["nj"])
        if b > 0:
            x0[:6] += rng.uniform(-0.2, 0.2, 6)
        x0s.append(x0)
        cmds.append([rng.uniform(-0.5, 1.0), rng.uniform(-0.3, 0.3), model["reference"]["defaultBaseHeight"], rng.uniform(-0.5, 0.5)])
    return np.array(x0s), np.array(cmds)


def compare(dev, host_insts):
    ref = stack_instances(host_insts)
    for k in INT_KEYS:
        assert np.array_equal(dev[k], ref[k]), k
    for k in FLOAT_KEYS:
        err = np.max(np.abs(dev[k] - ref[k]))
        assert err <= 1e-12 * max(1.0, np.max(np.abs(ref[k]))), (k, err)


@pytest.mark.parametrize("gait,start,horizon,t0", [("walk", 0.0, 1.2, 0.0), ("stance", 0.5, 1.2, 0.0), ("run", -0.23, 1.2, 0.0), ("jump", 0.0, 0.8, 0.0),
                                                   ("slow_walk", -1.1, 3.5, 0.0), ("trot", 0.3, 1.2, 0.0), ("walk", 0.0, 1.2, 7.3)])
def test_cold_start_arrays_match_the_host_builder(model, host_base_velocity, gait, start, horizon, t0):
    rng = np.random.default_rng(abs(int(start * 100)) + len(gait))
    B = 3
    x0s, cmds = make_inputs(model, rng, B)
    r = cbe.build_instances(model, t0, horizon, x0s, [gait] * B, [start] * B, cmds)
    assert not isinstance(r, int), r
    dev, bv, padding = r
    assert padding == {"x_init": 0.0, "x_ref": 0.0}
    host_bv = [host_base_velocity(x) for x in x0s]
    assert np.max(np.abs(bv - np.array(host_bv))) <= 1e-12
    assert np.all(bv[0] == 0.0) and np.all(np.abs(bv[1:]).max(axis=1) > 1e-3)   # zero momentum, then non-zero momentum
    host = [references.build_instance(model, x0s[b], t0=t0, horizon=horizon, gait=gait, gait_start=(None if gait == "stance" else start), cmd=list(cmds[b]),
                                      base_vel=host_bv[b]) for b in range(B)]
    assert dev["t_nodes"].shape[1] == len(host[0]["t_nodes"])
    compare(dev, host)
    # the layout of a target knot: normalized momentum (v_gx, v_gy, 0, 0, 0, yaw rate / m), base pose, default joints
    assert np.all(dev["x_ref"][:, :, 2:5] == 0.0) and np.all(dev["x_ref"][:, :, 10:12] == 0.0)
    assert np.allclose(dev["x_ref"][:, :, 12:], model["reference"]["defaultJointState"], rtol=0, atol=1e-15)


def test_warm_start_matches_the_host_shift(model, host_base_velocity):
    rng = np.random.default_rng(3)
    B, horizon = 2, 1.2
    x0s, cmds = make_inputs(model, rng, B)
    first, _, _ = cbe.build_instances(model, 0.0, horizon, x0s, ["walk"] * B, [0.0] * B, cmds)
    n = first["t_nodes"].shape[1]
    # a made-up previous solution on the first grid, near the measured states (momentum included)
    xs = first["x_init"] + 0.05 * rng.normal(size=(B, n, 35))
    us = rng.normal(size=(B, n - 1, 35))
    for t1 in (0.1, 0.35, 0.62):
        prevs = [references.to_primal_solution(first["t_nodes"][b], first["node_event"][b], xs[b], us[b]) for b in range(B)]
        x1 = np.array([references.linear_interpolate(t1, p["t"], p["x"]) for p in prevs])
        dev, bv, padding = cbe.build_instances(model, t1, horizon, x1, ["walk"] * B, [0.0] * B, cmds,
                                               previous=dict(t=first["t_nodes"], event=first["node_event"], x=xs, u=us))
        assert padding == {"x_init": 0.0, "x_ref": 0.0}
        host_bv = [host_base_velocity(x) for x in x1]
        assert np.max(np.abs(bv - np.array(host_bv))) <= 1e-12
        host = [references.build_instance(model, x1[b], t0=t1, horizon=horizon, gait="walk", gait_start=0.0, cmd=list(cmds[b]), previous=prevs[b],
                                          base_vel=host_bv[b]) for b in range(B)]
        assert dev["t_nodes"].shape[1] == len(host[0]["t_nodes"])
        compare(dev, host)


def test_base_velocity_matches_the_host_over_random_states(model, host_base_velocity):
    rng = np.random.default_rng(5)
    xs = []
    for _ in range(64):
        x = np.array(model["x_init"], float)
        x[:6] = rng.uniform(-0.5, 0.5, 6)
        x[6:9] += rng.uniform(-0.5, 0.5, 3)
        x[9:12] += rng.uniform(-0.6, 0.6, 3)
        x[12:] += rng.uniform(-0.4, 0.4, model["nj"])
        xs.append(x)
    bv = cbe.base_velocity(model, np.array(xs))
    ref = np.array([host_base_velocity(x) for x in xs])
    assert np.max(np.abs(bv - ref)) <= 1e-12


def test_mixed_node_counts_are_detected(model):
    rng = np.random.default_rng(1)
    x0s, cmds = make_inputs(model, rng, 2)
    assert cbe.build_instances(model, 0.0, 3.5, x0s, ["walk", "trot"], [0.0, 0.0], cmds) == -2
