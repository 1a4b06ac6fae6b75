"""The device-side instance builder's work-item functions (wb_humanoid_mpc_b200/csrc/wb_builder.cuh) executed on the CPU harness against the host
restatement of SolverBase::preRun (references.py): the same checks as tests/test_gpu_builder.py, where no GPU is available."""
import numpy as np
import pytest

import bld_emu_lib
from wb_humanoid_mpc_b200 import model_loader, references
from wb_humanoid_mpc_b200.solver import stack_instances

FLOAT_KEYS = ["x0", "x_init", "u_init", "t_nodes", "swing_ref", "impact_factor", "arm_phase", "x_ref"]
INT_KEYS = ["node_event", "contact_flags"]


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


def make_inputs(model, rng, B):
    x0s, cmds = [], []
    for _ in range(B):
        x0 = np.array(model["x_init"], float)
        x0[2] = model["reference"]["defaultBaseHeight"]
        x0[0:2] += rng.uniform(-0.02, 0.02, 2)
        x0[3:6] += rng.uniform(-0.05, 0.05, 3)
        x0[6:29] += rng.uniform(-0.1, 0.1, 23)
        x0[29:] += rng.uniform(-0.2, 0.2, 29)
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


@pytest.mark.parametrize("gait,start,horizon,t0", [("walk", 0.0, 3.5, 0.0), ("stance", 0.5, 1.1, 0.0), ("run", -0.23, 1.1, 0.0), ("jump", 0.0, 0.8, 0.0),
                                                   ("slow_walk", -1.1, 3.5, 0.0), ("trot", 0.3, 1.1, 0.0), ("walk", 0.0, 1.1, 7.3),
                                                   ("stance", 0.5, 1.1, 4.2)])
def test_cold_start_arrays_match_the_host_builder(model, gait, start, horizon, t0):
    rng = np.random.default_rng(abs(int(start * 100)) + len(gait))
    B = 3
    x0s, cmds = make_inputs(model, rng, B)
    dev = bld_emu_lib.build_instances(model, t0, horizon, x0s, [gait] * B, [start] * B, cmds)
    assert not isinstance(dev, int), dev
    host = [references.build_instance(model, x0s[b], t0=t0, horizon=horizon, gait=gait, gait_start=(None if gait == "stance" else start), cmd=list(cmds[b]))
            for b in range(B)]
    assert dev["t_nodes"].shape[1] == len(host[0]["t_nodes"])
    compare(dev, host)


def test_warm_start_matches_the_host_shift(model):
    rng = np.random.default_rng(3)
    B, horizon = 2, 1.1
    x0s, cmds = make_inputs(model, rng, B)
    first = bld_emu_lib.build_instances(model, 0.0, horizon, x0s, ["walk"] * B, [0.0] * B, cmds)
    n = first["t_nodes"].shape[1]
    xs, us = rng.normal(size=(B, n, 58)), rng.normal(size=(B, n - 1, 35))   # a made-up previous solution on the first grid
    for t1 in (0.1, 0.35, 0.62):
        prevs = [references.to_primal_solution(first["t_nodes"][b], first["node_event"][b], xs[b], us[b]) for b in range(B)]
        x1 = np.array([references.linear_interpolate(t1, p["t"], p["x"]) for p in prevs])
        dev = bld_emu_lib.build_instances(model, t1, horizon, x1, ["walk"] * B, [0.0] * B, cmds,
                                      previous=dict(t=first["t_nodes"], event=first["node_event"], x=xs, u=us))
        host = [references.build_instance(model, x1[b], t0=t1, horizon=horizon, gait="walk", gait_start=0.0, cmd=list(cmds[b]), previous=prevs[b]) for b in range(B)]
        assert dev["t_nodes"].shape[1] == len(host[0]["t_nodes"])
        compare(dev, host)


def test_mixed_node_counts_are_detected(model):
    rng = np.random.default_rng(1)
    x0s, cmds = make_inputs(model, rng, 2)
    assert bld_emu_lib.build_instances(model, 0.0, 3.5, x0s, ["walk", "trot"], [0.0, 0.0], cmds) == -2
