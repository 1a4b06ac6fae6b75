"""The centroidal policy roll-out's arithmetic (wb_sim.cuh: simRollout through SimCenSystem, run on the CPU harness with 40 thread slices
visited in reverse) against the restatement of MRT_BASE::rolloutPolicy around the oracle's own centroidal flow map (rollout_ref.py with
CenOracle.flow_map), for both centroidal model types: end state and input to 1e-12 relative, the same accepted and rejected step counts,
flow-map calls, mode and status, for the feed-forward and the feedback policy of a walking plan, a 1/100 s MRT step with and without a contact
switch inside it, and a pushed start.  The output state's padding is exactly zero, and NaN in the padded columns of K and in the padded state
slots changes nothing (only the 35 state entries are read)."""
import functools

import numpy as np
import pytest

import cen_sim_emu_lib
import oracle_lib as orc
import rollout_ref
from wb_humanoid_mpc_b200 import abi, model_loader, references

MRT_DT = 1.0 / 100.0   # the centroidal task.info: mrtDesiredFrequency 100 (one MRT step per 80 Hz MPC cycle, MRT_ROS_Dummy_Loop.cpp:83)
MODEL_TYPES = {"full": 0, "srbd": 1}


def centroidal_model(kind):
    m = dict(model_loader.load_packaged_model("g1_centroidal"))
    m["centroidalModelType"] = MODEL_TYPES[kind]
    return m


@functools.lru_cache(maxsize=None)
def centroidal_plan(kind):
    """one SQP iteration of a walking centroidal instance (horizon 1.2 s, non-zero momentum) on the oracle: its primal solution and remapped
    gains -> (model, plan, K [n-1, 35, 35])"""
    model = centroidal_model(kind)
    rng = np.random.default_rng(3)
    x0 = np.array(model["x_init"], float)
    x0[:6] += rng.uniform(-0.1, 0.1, 6)
    x0[12:] += rng.uniform(-0.1, 0.1, model["nj"])
    o = orc.CenOracle(model)
    base_vel = o.flow_map(x0, np.zeros(model["nu"]))[6:12] / sum(model["mass"])
    inst = references.build_instance(model, x0, t0=0.0, horizon=1.2, gait="walk", cmd=[0.4, 0.0, 0.7925, 0.1], base_vel=base_vel)
    o.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
    res = o.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1))
    plan = dict(t_nodes=np.asarray(inst["t_nodes"], float), node_event=np.asarray(inst["node_event"]), contact_flags=np.asarray(inst["contact_flags"]),
                x=res["x"], u=res["u"])
    return model, plan, np.array(res["K"])


def rel(a, b):
    return float(np.max(np.abs(a - b)) / max(1e-300, np.max(np.abs(b))))


def first_event(plan):
    return min(float(plan["t_nodes"][k]) for k in range(len(plan["t_nodes"])) if plan["node_event"][k] == 1)


def start(plan, case):
    """start time and state: no event in the step, the first contact switch inside it, or a push on the normalized momentum and the joints"""
    t = first_event(plan) - 0.4 * MRT_DT if case == "event" else 0.05
    i, a = rollout_ref.time_segment(t, list(plan["t_nodes"]))
    x0 = a * plan["x"][i] + (1 - a) * plan["x"][i + 1]
    if case == "perturbed":
        rng = np.random.default_rng(5)
        x0 = x0.copy()
        x0[0:6] += rng.normal(0.0, 0.2, 6)
        x0[12:] += rng.normal(0.0, 0.05, len(x0) - 12)
    return t, x0


@pytest.mark.parametrize("kind", list(MODEL_TYPES))
@pytest.mark.parametrize("feedback", [False, True], ids=["feedforward", "feedback"])
@pytest.mark.parametrize("case", ["smooth", "event", "perturbed"])
def test_emu_cen_rollout_matches_the_reference_restatement(kind, feedback, case):
    model, plan, K = centroidal_plan(kind)
    t, x0 = start(plan, case)
    Kf = K if feedback else None
    rs = abi.cen_default_rollout_settings()
    ref = rollout_ref.rollout_policy(orc.CenOracle(model).flow_map, plan, t, MRT_DT, x0, K=Kf, abs_tol=rs.abs_tol, rel_tol=rs.rel_tol,
                                     time_step=rs.time_step, max_steps_per_second=rs.max_steps_per_second)
    emu = cen_sim_emu_lib.rollout_policy(model, plan, t, MRT_DT, x0, K=Kf)
    assert ref["status"] == 0 and emu["status"] == 0
    assert (emu["accepted"], emu["rejected"], emu["calls"], emu["mode"]) == (ref["accepted"], ref["rejected"], ref["calls"], ref["mode"])
    assert rel(emu["x"], ref["x"]) < 1e-12
    assert rel(emu["u"], ref["u"]) < 1e-12
    assert np.array_equal(emu["padding"], np.zeros(23))
    if case == "event":
        assert t < first_event(plan) <= t + MRT_DT
    assert ref["calls"] == (2 if case == "event" else 1) + 6 * (ref["accepted"] + ref["rejected"])
    # NaN in every padded entry the kernel could read (plan states, gains, start state) leaves the result unchanged to the bit
    nan = cen_sim_emu_lib.rollout_policy(model, plan, t, MRT_DT, x0, K=Kf, fill=np.nan)
    assert np.array_equal(nan["x"], emu["x"]) and np.array_equal(nan["u"], emu["u"]) and np.array_equal(nan["padding"], np.zeros(23))
    assert [nan[k] for k in ("status", "accepted", "rejected", "calls", "mode")] == [emu[k] for k in ("status", "accepted", "rejected", "calls", "mode")]


@pytest.mark.parametrize("kind", list(MODEL_TYPES))
def test_emu_cen_rollout_reports_the_call_budget(kind):
    """maxNumStepsPerSecond caps the flow-map calls of one roll-out (IntegratorBase::systemFunction throws; here a status)"""
    model, plan, K = centroidal_plan(kind)
    rs = abi.cen_default_rollout_settings(max_steps_per_second=5.0)
    x0 = plan["x"][3]
    t = float(plan["t_nodes"][3])
    emu = cen_sim_emu_lib.rollout_policy(model, plan, t, MRT_DT, x0, K=K, settings=rs)
    ref = rollout_ref.rollout_policy(orc.CenOracle(model).flow_map, plan, t, MRT_DT, x0, K=K, abs_tol=rs.abs_tol, rel_tol=rs.rel_tol, max_steps_per_second=5.0)
    assert emu["status"] == ref["status"] == rollout_ref.BUDGET
    assert emu["calls"] == ref["calls"] == 6
