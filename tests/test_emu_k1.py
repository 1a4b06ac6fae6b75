"""Device-math check without a GPU: the __host__ __device__ phase functions of K1/K3 executed on the host by the development
harness (tests/emu) against the oracle.  This validates the kernels' arithmetic and the barrier placement (work items of every
phase are visited in reverse order); the GPU tests (-m gpu) validate the real launches through the C ABI."""
import numpy as np
import pytest

import emu_lib as emu
import oracle_lib as orc
from test_oracle_wb import rand_input, rand_state
from wb_humanoid_mpc_b200 import abi, model_loader


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


@pytest.fixture(scope="module")
def wb(model):
    return orc.WbOracle(model)


def rel(a, b):
    return np.max(np.abs(a - b)) / max(1e-12, np.max(np.abs(b))) if b.size else 0.0


def test_flow_map_and_base_acceleration_jacobian(model, wb):
    rng = np.random.default_rng(0)
    for _ in range(3):
        x, u = rand_state(model, rng), rand_input(model, rng)
        f, A, B = wb.flow_map_lin(x, u)
        xd, G = emu.dyn(wb.desc, x, u, True)
        assert np.max(np.abs(xd - f)) < 1e-12
        assert rel(G, np.hstack([A[29:35], B[29:35]])) < 1e-11
        xd2, _ = emu.dyn(wb.desc, x, u, False)
        assert np.max(np.abs(xd2 - f)) < 1e-12


@pytest.mark.parametrize("contact", [(1, 1), (1, 0), (0, 1), (0, 0)])
def test_lq_node_blocks_and_projection(model, wb, contact):
    rng = np.random.default_rng(sum(contact) + 3)
    x, u = rand_state(model, rng, 0.5), rand_input(model, rng)
    u[2] += 100
    u[8] += 100
    xn = x + rng.uniform(-0.01, 0.01, 58)
    xref = np.array(model["x_init"])
    xref[29:31] = [0.4, 0.1]
    swing = np.array([[0.03, 0.2, -1.0], [0.05, -0.1, 0.5]])
    impact, arm, dt = [0.7, 0.4], 0.3, 0.035
    wb.set_nodes(np.array([contact, contact], dtype=np.uint8), np.stack([swing, swing]), np.array([impact, impact]), np.array([arm, arm]),
                 np.stack([xref, xref]))
    st = abi.default_settings(model, sqp_iteration=1)
    wb.sqp(np.array([0.0, dt]), np.array([0, 0], dtype=np.uint8), x, np.stack([x, xn]), u[None], st, keep_raw=True)
    raw = wb.last_raw_blocks(2)[0]
    e = emu.lq_node(wb.desc, x, u, xn, xref, dt, contact, swing, impact, arm)
    assert e["raw"]["nc"] == raw["nc"] and e["nut"] == 35 - raw["nc"]
    for k in ["A", "B", "b", "Q", "S", "R", "q", "r", "C", "D", "e"]:
        assert rel(e["raw"][k], raw[k]) < 1e-10, k
    assert abs(e["raw"]["c"] - raw["c"]) < 1e-10 * max(1.0, abs(raw["c"]))
    r = e["raw"]
    assert np.abs(r["D"] @ e["Pu"]).max() < 1e-10 and np.abs(r["D"] @ e["Px"] + r["C"]).max() < 1e-9 and np.abs(r["D"] @ e["u0"] + r["e"]).max() < 1e-9
    pr = orc.change_of_input_variables(r["A"], r["B"], r["b"], r["Q"], r["S"], r["R"], r["q"], r["r"], r["c"], e["Pu"], e["Px"], e["u0"])
    for k in ["A", "B", "b", "Q", "S", "R", "q", "r"]:
        assert rel(e[k], pr[k]) < 1e-10, k


@pytest.mark.parametrize("contact", [(1, 1), (1, 0), (0, 1), (0, 0)])
@pytest.mark.parametrize("mode", [1, 2])
def test_cuda_k1b_schedules_equal_the_one_pass_schedule(model, wb, contact, mode):
    """The GPU runs K1b as lu_kernel + wb_node_b1.inc (projection, dynamics) + wb_node_b2.inc (cost; mode 2: Q accumulated in place in its
    output block, pre-scaled by dt).  The same includes on the CPU harness must reproduce the one-pass schedule that is checked against the oracle
    above: identical arithmetic for every block but Q (exactly equal), Q up to the rounding of dt (a + b) vs dt a + dt b in mode 2."""
    rng = np.random.default_rng(11 + sum(contact))
    x, u = rand_state(model, rng, 0.5), rand_input(model, rng)
    u[2] += 100
    u[8] += 100
    xn = x + rng.uniform(-0.01, 0.01, 58)
    xref = np.array(model["x_init"])
    swing = np.array([[0.03, 0.2, -1.0], [0.05, -0.1, 0.5]])
    args = (wb.desc, x, u, xn, xref, 0.035, contact, swing, [0.7, 0.4], 0.3)
    one = emu.lq_node(*args)
    two = emu.lq_node(*args, mode=mode)
    assert one["nut"] == two["nut"]
    for k in ["A", "B", "b", "S", "R", "q", "r", "Pu", "Px", "u0"]:
        assert np.array_equal(one[k], two[k]), k
    assert rel(two["Q"], one["Q"]) < (1e-14 if mode == 2 else 1e-300) or np.array_equal(one["Q"], two["Q"])
    for k in ["A", "B", "b", "Q", "S", "R", "q", "r", "C", "D", "e"]:
        assert rel(two["raw"][k], one["raw"][k]) < 1e-14, k


def test_joint_torque_map(model, wb):
    """computeJointTorques: the thread-per-node world-frame recursion (csrc/wb_torque.cuh) against the oracle (RNEA - J'W) and, for the
    oracle itself, the identity that the base rows of the same inverse dynamics vanish up to the dropped lin/ang coupling of M_bb"""
    rng = np.random.default_rng(5)
    for _ in range(4):
        x, u = rand_state(model, rng), rand_input(model, rng)
        tau, qddb = emu.joint_torques(wb.desc, x, u)
        to, qo = wb.joint_torques(x, u)
        assert np.max(np.abs(qddb - qo)) < 1e-10 * max(1.0, np.abs(qo).max())
        assert np.max(np.abs(tau - to)) < 1e-10 * max(1.0, np.abs(to).max())
        assert np.allclose(qo, wb.flow_map(x, u)[29:35], atol=1e-12)
    # at rest under weight-compensating wrenches the knees carry load and the base does not accelerate
    from wb_humanoid_mpc_b200 import references

    x = np.array(model["x_init"], float)
    x[29:] = 0.0
    u = references.weight_compensating_input(model, [1, 1])
    tau, qddb = emu.joint_torques(wb.desc, x, u)
    assert np.abs(qddb[:3]).max() < 1e-9 and abs(tau[3]) > 1.0 and abs(tau[9]) > 1.0
