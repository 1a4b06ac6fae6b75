"""Device-pointer I/O (b200sqp_*_dev), the parts that run without a GPU: the per-row robot-state check that b200sqp_joint_actions_dev runs on
the device (wb_devio.cuh: mrtRobotStateStatus, on the CPU harness) against the host entry point's rule, and the tensor checks of the Python
wrappers (solver.check_device_tensor)."""
import numpy as np
import pytest

import devio_emu_lib
import mrt_ref

NJ = 23
RS = 13 + 2 * NJ


def host_rule(r):
    """the loop b200sqp_joint_actions runs on the host (wb_capi.inc, jointActions), restated: 1 a non-finite entry, 2 the quaternion norm off"""
    with np.errstate(invalid="ignore"):
        if any(not (v - v == 0.0) for v in r):
            return 1
    n = np.sqrt(r[3] * r[3] + r[4] * r[4] + r[5] * r[5] + r[6] * r[6])
    return 0 if abs(n - 1.0) <= 1e-6 else 2


def scaled_quaternion(row, norm):
    r = row.copy()
    r[3:7] *= norm / np.linalg.norm(r[3:7])
    return r


def test_rows_with_non_finite_entries_are_rejected_in_every_field_group():
    base = mrt_ref.random_robot_states(np.random.default_rng(3), 1, NJ)[0]
    groups = {"position": 0, "quaternion": 3, "linear velocity": 7, "angular velocity": 10, "joint position": 13, "joint velocity": 13 + NJ,
              "last entry": RS - 1}
    rows, want = [base], [0]
    for _, i in groups.items():
        for bad in (np.nan, np.inf, -np.inf):
            r = base.copy()
            r[i] = bad
            rows.append(r)
            want.append(1)
    got = devio_emu_lib.robot_state_status(np.array(rows))
    assert got.tolist() == want
    assert [host_rule(r) for r in rows] == want


def test_quaternion_norm_bound():
    base = mrt_ref.random_robot_states(np.random.default_rng(4), 1, NJ)[0]
    norms = [1.0, 1.0 + 0.9e-6, 1.0 - 0.9e-6, 1.0 + 1.1e-6, 1.0 - 1.1e-6, 1.0 + 1e-5, 0.0, 2.0]
    rows = np.array([scaled_quaternion(base, n) for n in norms])
    got = devio_emu_lib.robot_state_status(rows)
    assert got.tolist() == [0, 0, 0, 2, 2, 2, 2, 2]
    assert got.tolist() == [host_rule(r) for r in rows]


def test_seeded_rows_agree_with_the_host_rule():
    rng = np.random.default_rng(11)
    rows = mrt_ref.random_robot_states(rng, 64, NJ)
    for b in range(0, 64, 3):   # norms spread around the bound, and a few non-finite entries
        rows[b] = scaled_quaternion(rows[b], 1.0 + rng.uniform(-2e-6, 2e-6))
    rows[5, 20] = np.nan
    rows[9, 2] = np.inf
    got = devio_emu_lib.robot_state_status(rows)
    assert got.tolist() == [host_rule(r) for r in rows]
    assert {0, 1, 2} <= set(got.tolist())


def test_tensor_checks():
    torch = pytest.importorskip("torch")
    from wb_humanoid_mpc_b200.solver import check_device_tensor

    cpu = torch.device("cpu")
    good = torch.zeros((4, RS), dtype=torch.float64)
    assert check_device_tensor(good, "robot_state", cpu, torch.float64, (4, RS)) is good
    with pytest.raises(ValueError, match="robot_state: the tensor is on cpu"):   # a CPU tensor where the handle's CUDA device is expected
        check_device_tensor(good, "robot_state", torch.device("cuda", 0), torch.float64, (4, RS))
    with pytest.raises(ValueError, match="robot_state: dtype torch.float32"):
        check_device_tensor(good.float(), "robot_state", cpu, torch.float64, (4, RS))
    with pytest.raises(ValueError, match=r"x0: shape \(4, 59\), expected \(4, 58\)"):
        check_device_tensor(good, "x0", cpu, torch.float64, (4, 58))
    with pytest.raises(ValueError, match="out\\['mode'\\]: the tensor is not C-contiguous"):
        check_device_tensor(torch.zeros((8,), dtype=torch.int32)[::2], "out['mode']", cpu, torch.int32, (4,))
    with pytest.raises(ValueError, match="expected a torch tensor"):
        check_device_tensor(np.zeros((4, RS)), "robot_state", cpu, torch.float64, (4, RS))
