"""Joint-torque cost of the whole-body OCP (JointTorqueCostCppAd) on the CPU: the oracle's term against the oracle's torque map, finite
differences and its own Gauss-Newton algebra; the device phases (wb_torque_cost.cuh) on the CPU harness against the oracle; the task.info
loaders."""
import subprocess

import numpy as np
import pytest

import jt_oracle_lib as jt
import mrt_ref
import oracle_lib as orc
from test_oracle_wb import fd_jac, rand_input, rand_state
from wb_humanoid_mpc_b200 import abi, model_loader, references

ROOT = jt.ROOT
TASK = ROOT / "tests/golden/g1_config/robot_models/unitree_g1/g1_wb_mpc/config/mpc/task.info"


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


def weights(rng, nj=23):
    return rng.uniform(1e-4, 2e-3, nj)


def swing_input(model, rng, c):
    u = rand_input(model, rng)
    u[6 * c:6 * c + 6] = 0.0
    return u


def rel(a, b):
    return np.max(np.abs(a - b)) / max(1e-12, np.max(np.abs(b)))


def test_residual_is_weighted_torque_map(model):
    rng = np.random.default_rng(0)
    w = weights(rng)
    o = jt.JtOracle(model, w)
    wb = orc.WbOracle(model)
    for u_of in (lambda: rand_input(model, rng), lambda: swing_input(model, rng, 0), lambda: swing_input(model, rng, 1)):
        x, u = rand_state(model, rng), u_of()
        r, _ = o.residual(x, u)
        tau = wb.joint_torques(x, u)[0]
        plan = dict(t_nodes=np.array([0.0, 0.1]), node_event=np.zeros(2, np.uint8), contact_flags=np.ones((2, 2), np.uint8), x=np.stack([x, x]),
                    u=np.stack([u]))
        tau_mrt = mrt_ref.joint_action(model, wb, 0.05, x_obs=x, plan=plan)["tau"]
        assert rel(r / np.sqrt(w), tau) < 1e-12
        assert rel(o.torques(x, u), tau) < 1e-12
        assert rel(tau_mrt, tau) < 1e-12


def test_jacobian_matches_finite_differences(model):
    rng = np.random.default_rng(1)
    o = jt.JtOracle(model, weights(rng))
    nx = model["nx"]
    for c in (None, 0):
        x = rand_state(model, rng)
        u = rand_input(model, rng) if c is None else swing_input(model, rng, c)
        r, J = o.residual(x, u)
        Jfd = fd_jac(lambda z: o.residual(z[:nx], z[nx:])[0], np.concatenate([x, u]))
        assert np.max(np.abs(J - Jfd)) < 1e-6 * max(1.0, np.max(np.abs(J)))


@pytest.mark.parametrize("contact", [(1, 1), (1, 0), (0, 0)])
def test_gauss_newton_blocks(model, contact):
    """cost_quad with the term minus cost_quad without it = (1/2 |r|^2, J'r, J'J)"""
    rng = np.random.default_rng(2)
    w = weights(rng)
    on, off = jt.JtOracle(model, w), jt.JtOracle(model, None)
    n = 2
    xref = np.tile(model["x_init"], (n, 1))
    for o in (on, off):
        o.set_nodes(np.tile(contact, (n, 1)), np.zeros((n, 2, 3)), np.ones((n, 2)), np.full(n, 0.3), xref)
    x, u = rand_state(model, rng), rand_input(model, rng)
    r, J = on.residual(x, u)
    a, b = on.cost_quad(0, x, u), off.cost_quad(0, x, u)
    nx = model["nx"]
    H = J.T @ J
    g = J.T @ r
    assert abs((a["f"] - b["f"]) - 0.5 * r @ r) < 1e-9 * max(1.0, a["f"])
    assert abs(on.cost(0, x, u) - off.cost(0, x, u) - 0.5 * r @ r) < 1e-9 * max(1.0, a["f"])
    assert rel(a["q"] - b["q"], g[:nx]) < 1e-9 and rel(a["r"] - b["r"], g[nx:]) < 1e-9
    assert rel(a["Q"] - b["Q"], H[:nx, :nx]) < 1e-9
    assert rel(a["S"] - b["S"], H[nx:, :nx]) < 1e-9
    assert rel(a["R"] - b["R"], H[nx:, nx:]) < 1e-9


def _instance(model, gait="walk", horizon=1.1):
    rng = np.random.default_rng(3)
    x0 = np.array(model["x_init"], float)
    x0[2] = model["reference"]["defaultBaseHeight"]
    x0[6:29] += rng.uniform(-0.1, 0.1, 23)
    return references.build_instance(model, x0, t0=0.0, horizon=horizon, gait=gait, cmd=[0.4, 0.0, 0.7925, 0.0])


def test_event_and_terminal_nodes_untouched_zero_weights_identical(model):
    inst = _instance(model)
    ev = inst["node_event"]
    assert (ev == 1).any()
    st = abi.default_settings(model, sqp_iteration=1)
    off = jt.solve(model, inst, st, None, keep_raw=True)
    zero = jt.solve(model, inst, st, np.zeros(23), keep_raw=True)
    on = jt.solve(model, inst, st, np.full(23, 1e-3), keep_raw=True)
    for k in range(len(ev) - 1):
        for key in ("Q", "S", "R", "q", "r", "c", "A", "B", "b"):
            assert np.array_equal(zero["raw"][k][key], off["raw"][k][key]), (k, key)
        if ev[k] == 1:   # PreEvent: identity jump map, no cost
            for key in ("Q", "q", "c"):
                assert np.array_equal(on["raw"][k][key], off["raw"][k][key]), (k, key)
        else:
            assert not np.array_equal(on["raw"][k]["R"], off["raw"][k]["R"]), k
    # the terminal node keeps the final cost only: the value function's last Hessian is Q_final in both problems
    P_on = jt.JtOracle(model, np.full(23, 1e-3))
    P_on.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
    P_on.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], st)
    P_off = jt.JtOracle(model, None)
    P_off.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
    P_off.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], st)
    Pa, _ = P_on.last_value_function(inst["x_init"])
    Pb, _ = P_off.last_value_function(inst["x_init"])
    assert np.array_equal(Pa[-1], Pb[-1])


def test_sqp_step_with_term_is_stationary(model):
    """KKT of the projected QP of the oracle's last iteration with the term: the Riccati solution satisfies the stage-wise stationarity
    (OcpToKkt-style, from the raw blocks, the constraint projection and the value function): with the raw cost approximation of node k,
    the input step minimises 1/2 [dx; du]' H [dx; du] + g'[dx; du] + V_{k+1}(A dx + B du + b) on C dx + D du + e = 0."""
    inst = _instance(model, gait="stance", horizon=0.3)
    st = abi.default_settings(model, sqp_iteration=1)
    o = jt.JtOracle(model, np.full(23, 1e-3))
    o.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
    res = o.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], st, keep_raw=True)
    raw = o.last_raw_blocks(len(inst["t_nodes"]))
    P, p = o.last_value_function(inst["x_init"])
    p = p + np.einsum("kij,kj->ki", P, inst["x_init"])   # back to the value function of the step dx (before re-centring)
    dx, du = res["dx"], res["du"]
    nx = model["nx"]
    for k in range(len(inst["t_nodes"]) - 1):
        if inst["node_event"][k] == 1:
            continue
        blk = raw[k]
        lam = P[k + 1] @ dx[k + 1] + p[k + 1]
        grad_u = blk["S"] @ dx[k] + blk["R"] @ du[k] + blk["r"] + blk["B"].T @ lam
        # stationarity up to the constraint multipliers: grad_u lies in the row space of D
        D = blk["D"]
        nu_ = np.linalg.lstsq(D.T, grad_u, rcond=None)[0]
        resid = grad_u - D.T @ nu_
        assert np.max(np.abs(resid)) < 1e-6 * max(1.0, np.max(np.abs(grad_u))), (k, np.max(np.abs(resid)))
        assert np.max(np.abs(blk["C"] @ dx[k] + D @ du[k] + blk["e"])) < 1e-8


@pytest.mark.parametrize("c", [None, 0, 1])
def test_device_phases_match_oracle(model, c):
    """jtPhaseJacobian / jtPhaseRaw on the CPU harness (work items in reverse order): tau, J and the raw Gauss-Newton blocks at 1e-9; the
    projected blocks of jtPhaseProject / jtPhaseAccumulate equal the change of input variables of the term's own raw blocks"""
    rng = np.random.default_rng(4 if c is None else 5 + c)
    w = weights(rng)
    x = rand_state(model, rng)
    u = rand_input(model, rng) if c is None else swing_input(model, rng, c)
    dt = 0.0137
    r, J = jt.JtOracle(model, w).residual(x, u)
    nu, nut = model["nu"], 23 if c is None else 22
    Pu, Px, u0 = rng.normal(size=(nu, nut)), rng.normal(size=(nu, model["nx"])), rng.normal(size=nu)
    e = jt.emu_node(model, w, x, u, dt, Pu, Px, u0)
    assert rel(e["r"], r) < 1e-9 and rel(e["J"], J) < 1e-9
    nx = model["nx"]
    H, g = dt * J.T @ J, dt * J.T @ r
    raw = e["raw"]
    assert rel(raw["Q"], H[:nx, :nx]) < 1e-9 and rel(raw["S"], H[nx:, :nx]) < 1e-9 and rel(raw["R"], H[nx:, nx:]) < 1e-9
    assert rel(raw["q"], g[:nx]) < 1e-9 and rel(raw["r"], g[nx:]) < 1e-9 and abs(raw["c"] - dt * 0.5 * r @ r) < 1e-9 * raw["c"]
    # changeOfInputVariables of the term's raw blocks
    cv = orc.change_of_input_variables(np.eye(nx), np.zeros((nx, nu)), np.zeros(nx), raw["Q"], raw["S"], raw["R"], raw["q"], raw["r"], raw["c"],
                                       Pu, Px, u0)
    assert rel(e["Q"], cv["Q"]) < 1e-9 and rel(e["S"], cv["S"]) < 1e-9 and rel(e["R"], cv["R"]) < 1e-9
    assert rel(e["q"], cv["q"]) < 1e-9 and rel(e["r_t"], cv["r"]) < 1e-9
    assert abs(e["perf"][0] + e["perf"][3] - cv["c"]) < 1e-9 * abs(cv["c"])


def test_loaders(tmp_path):
    assert model_loader.joint_torque_weights(TASK) is None
    w = np.linspace(0.001, 0.023, 23)
    task = tmp_path / "task.info"
    text = TASK.read_text() + "\njoint_torque_weights\n{\n  scaling 1e-1\n" + "".join(f"  ({i},0) {10 * float(v)!r}\n" for i, v in enumerate(w)) + "}\n"
    task.write_text(text)
    got = model_loader.joint_torque_weights(task)
    assert np.allclose(got, w, rtol=1e-15, atol=0)
    prog = tmp_path / "jt.cpp"
    prog.write_text('#include <cstdio>\n#include "wb_humanoid_mpc_b200/host/model_from_config.hpp"\n'
                    "int main(int argc, char** argv) {\n  for (double v : b200sqp::host::loadJointTorqueWeights(argv[1])) std::printf(\"%.17g\\n\", v);\n"
                    "  std::printf(\"end\\n\");\n}\n")
    exe = tmp_path / "jt"
    subprocess.run(["g++", "-std=c++17", "-O1", f"-I{ROOT}", str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe), str(task)], capture_output=True, text=True, check=True).stdout.split()
    assert out[-1] == "end" and np.array_equal(np.array(out[:-1], float), got)
    out = subprocess.run([str(exe), str(TASK)], capture_output=True, text=True, check=True).stdout.split()
    assert out == ["end"]
