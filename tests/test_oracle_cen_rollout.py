"""The centroidal roll-out's settings and the CPU restatement of the reference's roll-out (rollout_ref.py) on the centroidal flow map:
abi.cen_default_rollout_settings() is the rollout block of the centroidal task.info, and rollout_ref around CenOracle.flow_map agrees with scipy's
DOP853 (rtol 1e-12) within the requested tolerance on one MRT step of a walking plan's feedback policy from a pushed state, for both centroidal
model types."""
from pathlib import Path

import numpy as np
import pytest
from scipy.integrate import solve_ivp

import oracle_lib as orc
import rollout_ref as rr
from test_emu_cen_rollout import MODEL_TYPES, MRT_DT, centroidal_plan, start
from wb_humanoid_mpc_b200 import abi, model_loader

TASK_INFO = Path(__file__).resolve().parent / "golden" / "g1_config" / "robot_models" / "unitree_g1" / "g1_centroidal_mpc" / "config" / "mpc" / "task.info"


def test_cen_default_rollout_settings_are_the_task_info_rollout_block():
    blk = model_loader.parse_info(TASK_INFO)["rollout"]
    rs = abi.cen_default_rollout_settings()
    assert blk["integratorType"] == "ODE45"
    assert [rs.abs_tol, rs.rel_tol, rs.time_step, rs.max_steps_per_second] == [float(blk[k]) for k in ("AbsTolODE", "RelTolODE", "timeStep", "maxNumStepsPerSecond")]
    assert [rs.abs_tol, rs.rel_tol, rs.time_step, rs.max_steps_per_second] == [5e-5, 5e-3, 0.015, 10000.0]
    # the whole-body defaults are unchanged, and overrides apply on top of the centroidal values
    assert abi.default_rollout_settings().abs_tol == 1e-5
    over = abi.cen_default_rollout_settings(abs_tol=1e-6, time_step=0.01)
    assert [over.abs_tol, over.rel_tol, over.time_step] == [1e-6, 5e-3, 0.01]


@pytest.mark.parametrize("kind", list(MODEL_TYPES))
def test_dp5_against_dop853_on_the_centroidal_flow_map(kind):
    model, plan, K = centroidal_plan(kind)
    t0, x0 = start(plan, "perturbed")
    o = orc.CenOracle(model)
    ctrl = rr.PlanController(plan["t_nodes"], plan["node_event"], plan["x"], plan["u"], K)
    rs = abi.cen_default_rollout_settings()
    r = rr.time_triggered_rollout(o.flow_map, ctrl, t0, x0, t0 + MRT_DT, [], abs_tol=rs.abs_tol, rel_tol=rs.rel_tol, time_step=rs.time_step)
    assert r["status"] == rr.OK and r["accepted"] >= 1
    a0 = r["t"][0]   # (the interval starts weakEpsilon after t0)
    ref = solve_ivp(lambda t, x: o.flow_map(x, ctrl.compute_input(t, x)), (a0, t0 + MRT_DT), r["x"][0], method="DOP853", rtol=1e-12, atol=1e-12)
    want = ref.y[:, -1]
    assert np.all(np.abs(r["x"][-1] - want) <= rs.abs_tol + rs.rel_tol * np.abs(want)), np.max(np.abs(r["x"][-1] - want))
    # and the end state moved: the push and the policy act over the step
    assert np.max(np.abs(r["x"][-1] - x0)) > 1e-4
