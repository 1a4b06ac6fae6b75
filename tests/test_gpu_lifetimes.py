"""Re-sizing a handle or a fleet after every lazily allocated array exists (the batch, the builder's arrays, the stateful schedules, the
motion-manager states or the pose targets, the roll-out and joint-action arrays, the pinned staging): every output at the new size equals,
bit for bit, that of a fresh handle that has only ever seen that size and horizon."""
import numpy as np
import pytest

import mrt_ref
from test_gpu_device_io import DT_MPC, FAMS, KINDS, Case, cuda
from wb_humanoid_mpc_b200 import abi

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

B1, B2 = 32, 48
LONGER = 0.3   # seconds added to the horizon at B2: more nodes, so the node capacity grows too
FEATURES = ["motion", "pose"]   # the motion manager and pose commands exclude each other


def new_handle(c, feature):
    """a handle (and fleet) of c's family and kind with the stateful schedule and the loop feature"""
    from wb_humanoid_mpc_b200.solver import B200SqpFleet, B200SqpSolver

    s = B200SqpSolver(c.model, abi.default_settings(c.model, sqp_iteration=1, use_feedback_policy=1))
    cen = c.fam == "cen"
    (s.cen_set_gait_schedule if cen else s.set_gait_schedule)(True)
    if feature == "motion":
        (s.cen_set_motion_manager if cen else s.set_motion_manager)()
    else:
        s.set_pose_commands()
    return B200SqpFleet(s) if c.kind == "fleet" else s


def sequence(c, h, feature, horizon):
    """cold build, solve, roll-out, warm build from the roll-out, solve, joint actions (host and device), device plan download: every output"""
    out = {"n_cold": h.build_instances(0.0, horizon, c.x0s, c.gaits, c.starts, c.cmds)}
    if c.kind == "fleet":
        assert h.n_groups >= 2
    h.solve()
    out["plan0"] = h.primal_solution()
    roll = h.cen_rollout_policy if (c.fam == "cen" and c.kind == "plain") else h.rollout_policy
    out["rollout"] = roll(0.0, DT_MPC)
    if feature == "pose":
        h.command_poses([0, 5, 9], [[0.5, 0.1, 0.0, 30.0], [0.0, 0.0, 0.1, -45.0], [1.0, -0.2, 0.0, 0.0]])
    out["n_warm"] = h.build_instances(DT_MPC, horizon, None, c.gaits, c.starts, c.cmds, warm="rollout")
    out["instances"] = h.download_instances()
    out[feature] = h.motion_state() if feature == "motion" else h.pose_targets()
    h.solve()
    out["plan1"] = h.primal_solution()
    t = DT_MPC + mrt_ref.POLICY_DT
    rs = c.robot_states(3)
    out["actions"] = h.joint_actions(t, rs)
    out["actions_dev"] = h.joint_actions_device(t, cuda(rs))
    out["plan_dev"] = h.primal_solution_device()
    torch.cuda.synchronize()
    return out


def same(a, b, path="out"):
    """equal bit for bit, NaN equal to NaN; the iteration logs are skipped, as in test_gpu_device_io.same_dicts"""
    if isinstance(a, dict):
        assert a.keys() == b.keys(), path
        for k in a:
            if k != "log":
                same(a[k], b[k], f"{path}.{k}")
        return
    va = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    vb = b.cpu().numpy() if hasattr(b, "cpu") else np.asarray(b)
    assert va.shape == vb.shape and va.dtype == vb.dtype, (path, va.shape, vb.shape, va.dtype, vb.dtype)
    assert np.array_equal(va, vb, equal_nan=va.dtype.kind in "fc"), path


@pytest.mark.parametrize("feature", FEATURES)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fam", FAMS)
def test_resized_handle_equals_a_fresh_one(fam, kind, feature):
    h = None
    for batch, longer in ((B1, 0.0), (B2, LONGER), (B1, 0.0)):
        c = Case(fam, kind, batch)   # the inputs of this size (its own handle stays unused)
        horizon = c.horizon + longer
        if h is None:
            h = new_handle(c, feature)
        same(sequence(c, h, feature, horizon), sequence(c, new_handle(c, feature), feature, horizon), f"B={batch}")
