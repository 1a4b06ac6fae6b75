"""The policy roll-out kernel's arithmetic (wb_sim.cuh: simRollout and its phase functions, run on the CPU harness with 48 thread slices visited in
reverse) against the restatement of MRT_BASE::rolloutPolicy around the oracle's own whole-body flow map (rollout_ref.py): end state and input
to 1e-12 relative, the same accepted and rejected step counts, the same number of flow-map calls and the same mode, for the feed-forward and
the feedback policy of a walking plan, a 1/80 s MRT step with and without a contact switch inside it, and a perturbed start."""
import functools

import numpy as np
import pytest

import sim_emu_lib
import oracle_lib as orc
import rollout_ref
from wb_humanoid_mpc_b200 import abi, model_loader

MRT_DT = 1.0 / 80.0   # WBMpcDummySimNode.cpp: the MRT runs at 80 Hz


@functools.lru_cache(maxsize=None)
def walking_plan():
    """one SQP iteration of a walking instance on the oracle: its primal solution and remapped gains (the PreEvent stages have no input and a zero
    gain, as on the device)"""
    from test_gpu_wb import make_instances, oracle_solve

    model = model_loader.load_packaged_model()
    inst = make_instances(model, np.random.default_rng(3), [("walk", 1.1, [0.4, 0.0, 0.7925, 0.1])])[0]
    st = abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1)
    res = oracle_solve(model, inst, st)
    K = np.array(res["K"])
    K[np.asarray(inst["node_event"][:-1]) == 1] = 0.0
    plan = dict(t_nodes=np.asarray(inst["t_nodes"], float), node_event=np.asarray(inst["node_event"]), contact_flags=np.asarray(inst["contact_flags"]),
                x=res["x"], u=res["u"])
    return model, plan, K


def rel(a, b):
    return float(np.max(np.abs(a - b)) / max(1e-300, np.max(np.abs(b))))


def pre_event_times(plan):
    return [float(plan["t_nodes"][k]) for k in range(len(plan["t_nodes"])) if plan["node_event"][k] == 1]


def start_times(plan):
    """a start time whose MRT step contains no event and one whose step contains the first contact switch"""
    te = pre_event_times(plan)[0]
    return {"smooth": 0.05, "event": te - 0.4 * MRT_DT}


@pytest.mark.parametrize("feedback", [False, True], ids=["feedforward", "feedback"])
@pytest.mark.parametrize("case", ["smooth", "event", "perturbed"])
def test_emu_rollout_matches_the_reference_restatement(feedback, case):
    model, plan, K = walking_plan()
    t = start_times(plan)["event" if case == "event" else "smooth"]
    i, a = rollout_ref.time_segment(t, list(plan["t_nodes"]))
    x0 = a * plan["x"][i] + (1 - a) * plan["x"][i + 1]
    if case == "perturbed":
        rng = np.random.default_rng(5)
        x0 = x0.copy()
        x0[29:35] += rng.normal(0.0, 0.3, 6)    # a push: base velocity
        x0[35:] += rng.normal(0.0, 0.2, 23)     # and joint velocities
    Kf = K if feedback else None
    wb = orc.WbOracle(model)
    ref = rollout_ref.rollout_policy(wb.flow_map, plan, t, MRT_DT, x0, K=Kf)
    emu = sim_emu_lib.rollout_policy(abi.model_desc(model), plan, t, MRT_DT, x0, K=Kf)
    assert ref["status"] == 0 and emu["status"] == 0
    assert (emu["accepted"], emu["rejected"], emu["calls"], emu["mode"]) == (ref["accepted"], ref["rejected"], ref["calls"], ref["mode"])
    assert rel(emu["x"], ref["x"]) < 1e-12
    assert rel(emu["u"], ref["u"]) < 1e-12
    # every integration interval costs one call at its start and six per tried step; a step that crosses the switch integrates two intervals
    n_intervals = 2 if case == "event" else 1
    if case == "event":
        te = pre_event_times(plan)[0]
        assert t < te <= t + MRT_DT
    assert ref["calls"] == n_intervals + 6 * (ref["accepted"] + ref["rejected"])


def test_emu_rollout_reports_the_call_budget():
    """maxNumStepsPerSecond caps the flow-map calls of one roll-out (IntegratorBase::systemFunction throws; here a status)"""
    model, plan, K = walking_plan()
    rs = abi.default_rollout_settings(max_steps_per_second=5.0)
    x0 = plan["x"][3]
    emu = sim_emu_lib.rollout_policy(abi.model_desc(model), plan, float(plan["t_nodes"][3]), MRT_DT, x0, K=K, settings=rs)
    ref = rollout_ref.rollout_policy(orc.WbOracle(model).flow_map, plan, float(plan["t_nodes"][3]), MRT_DT, x0, K=K, max_steps_per_second=5.0)
    assert emu["status"] == ref["status"] == rollout_ref.BUDGET
    assert emu["calls"] == ref["calls"] == 6
