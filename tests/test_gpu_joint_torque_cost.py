"""Joint-torque cost of the whole-body OCP on the GPU (b200sqp_set_joint_torque_cost) against the CPU oracle with the term
(tests/oracle_jt): raw stage blocks, SQP iterates, gains and logs, the off path, per-instance payload models, the global-step ladder,
behaviour and error codes.  Tolerances as tests/test_gpu_wb.py: 1e-9 for blocks, 1e-7 for SQP outputs."""
import numpy as np
import pytest

import jt_oracle_lib as jt
from test_gpu_builder import make_inputs
from test_gpu_fleet import KEYS, mixed_batch
from test_gpu_wb import make_instances, rel
from wb_humanoid_mpc_b200 import abi, lib as _l, model_loader
from wb_humanoid_mpc_b200.lib import B200SqpError
from wb_humanoid_mpc_b200.solver import B200SqpFleet, B200SqpSolver, joint_torques, stack_instances

pytestmark = pytest.mark.gpu

W = np.linspace(2e-4, 2e-3, 23)


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


def specs(n):
    base = [("stance", 1.1, None), ("walk", 1.1, [0.4, 0.0, 0.7925, 0.1]), ("stance", 1.1, [0.3, 0.1, 0.7925, 0.0]), ("walk", 1.1, [0.2, 0.1, 0.7925, 0.0])]
    return [base[i % len(base)] for i in range(n)]


def test_raw_blocks_match_oracle_at_batch_256(model):
    insts = make_instances(model, np.random.default_rng(1), specs(256))
    st = abi.default_settings(model, sqp_iteration=1)
    solver = B200SqpSolver(model, st, capture_raw_blocks=True)
    solver.set_joint_torque_cost(W)
    solver.run(insts)
    raw = solver.raw_stage_blocks()
    for b in (0, 1, 130, 255):
        ref = jt.solve(model, insts[b], st, W, keep_raw=True)
        for k in range(len(insts[b]["t_nodes"]) - 1):
            g, o = jt.orc.unpack_raw_blocks(raw[b, k], 58, 35), ref["raw"][k]
            for key in ("Q", "S", "R", "q", "r", "C", "D", "e"):
                assert rel(g[key], o[key]) < 1e-9, (b, k, key, rel(g[key], o[key]))
            assert abs(g["c"] - o["c"]) <= 1e-9 * max(1.0, abs(o["c"])), (b, k)


def test_sqp_iterations_match_oracle(model):
    insts = make_instances(model, np.random.default_rng(2), specs(3))
    st = abi.default_settings(model, sqp_iteration=4, use_feedback_policy=1)
    solver = B200SqpSolver(model, st)
    solver.set_joint_torque_cost(W)
    sol = solver.run(insts)
    assert not sol["status"].any()
    for b, inst in enumerate(insts):
        ref = jt.solve(model, inst, st, W)
        nit = len(ref["log"])
        assert sol["n_iter"][b] == nit
        for it in range(nit):
            g, o = sol["log"][b, it], ref["log"][it]
            assert g[8] == o[8] and int(g[9]) == int(o[9]) and int(g[13]) == int(o[13]), (b, it)
            for j in (0, 1, 2, 3, 4, 5, 6, 7, 10, 11):   # merits and costs include the term
                assert abs(g[j] - o[j]) <= 1e-7 * max(1.0, abs(o[j])), (b, it, j, g[j], o[j])
        assert rel(sol["x"][b], ref["x"]) < 1e-7
        assert rel(sol["u"][b], ref["u"]) < 1e-7
        assert rel(sol["K"][b], ref["K"]) < 1e-6


def test_off_path_is_bit_identical(model):
    insts = make_instances(model, np.random.default_rng(3), specs(8))
    st = abi.default_settings(model, sqp_iteration=2)
    runs = []
    for setup in (lambda s: None, lambda s: (s.set_joint_torque_cost(W), s.set_joint_torque_cost(None)), lambda s: s.set_joint_torque_cost(np.zeros(23))):
        s = B200SqpSolver(model, st)
        setup(s)
        sol = s.run(insts)
        runs.append((sol, s.launch_count()))
    for sol, n in runs[1:]:
        assert n == runs[0][1]
        for key in ("x", "u", "log"):
            assert np.array_equal(sol[key], runs[0][0][key]), key
    on = B200SqpSolver(model, st)
    on.set_joint_torque_cost(W)
    on.run(insts)
    assert on.launch_count() > runs[0][1]


def test_payload_model_record_matches_oracle(model):
    insts = make_instances(model, np.random.default_rng(4), specs(2))
    st = abi.default_settings(model, sqp_iteration=2)
    solver = B200SqpSolver(model, st)
    solver.set_joint_torque_cost(W)
    solver.upload(stack_instances(insts))
    base = solver.default_robot_params()
    p = model_loader.add_payload(base, 0, 10.0, [0.05, 0.0, 0.1], np.diag([0.1, 0.1, 0.05]), model=model)
    recs = {k: np.stack([np.asarray(base[k]), np.asarray(p[k])]) for k in base}
    solver.set_robot_params(np.arange(2), recs, "model")
    solver.solve()
    sol = solver.primal_solution()
    for b, m in enumerate((model, model_loader.with_robot_params(model, p))):
        ref = jt.solve(m, insts[b], st, W)
        assert rel(sol["x"][b], ref["x"]) < 1e-7 and rel(sol["u"][b], ref["u"]) < 1e-7, b


def host_merit(model, inst, x, u, w):
    """the merit of (x, u) on the oracle with the term (weights w, None: without): sum of dt * cost over the intermediate nodes, dt as
    getIntervalDuration with the weak epsilon at events, plus the final cost (the equality constraints are projected: merit = cost)"""
    o = jt.JtOracle(model, w)
    o.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
    t, ev = inst["t_nodes"], inst["node_event"]
    n = len(t) - 1
    m = 0.0
    for i in range(n):
        if ev[i] == 1:
            continue
        dt = (t[i + 1] - (1e-9 if ev[i + 1] == 1 else 0.0)) - (t[i] + (1e-9 if ev[i] == 2 else 0.0))
        m += dt * o.cost(i, x[i], u[i])
    d = x[n] - inst["x_ref"][n]
    return m + 0.5 * float(np.sum(np.asarray(model["Qf_diag"]) * d * d))


def test_global_step_ladder_includes_the_term(model):
    """single-process global_step = 1: the candidate the ladder applies is accepted by every instance, and its summed trial merit
    (ladder_eval_kernel) is the oracle's merit with the term at the iterates the step produced -- not the merit without it"""
    insts = make_instances(model, np.random.default_rng(5), specs(4))
    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=1, global_step=1))
    s.enable_global_step()
    s.set_joint_torque_cost(W)
    sol = s.run(insts)
    g, idx = s.global_stats()
    assert idx >= 0 and sol["log"][0, 0, 8] > 0, (idx, sol["log"][:, 0, 8])
    assert g[idx, 0] == g[idx, 3] == len(insts)
    on = [host_merit(model, inst, sol["x"][b], sol["u"][b], W) for b, inst in enumerate(insts)]
    off = [host_merit(model, inst, sol["x"][b], sol["u"][b], None) for b, inst in enumerate(insts)]
    assert np.allclose(sol["log"][:, 0, 4], on, rtol=1e-9, atol=0), (sol["log"][:, 0, 4], on)
    assert abs(g[idx, 1] - sum(on)) <= 1e-9 * abs(sum(on))
    assert abs(g[idx, 1] - sum(off)) > 1e-6 * abs(sum(on))


def test_heavier_weights_lower_planned_torques(model):
    insts = make_instances(model, np.random.default_rng(6), specs(8))
    st = abi.default_settings(model, sqp_iteration=3)
    mean_tau = []
    for w in (None, 50 * W):
        s = B200SqpSolver(model, st)
        s.set_joint_torque_cost(w)
        sol = s.run(insts)
        tau, _ = joint_torques(model, sol["x"][:, :-1], sol["u"])
        ev = np.stack([i["node_event"][:-1] for i in insts]) != 1
        mean_tau.append(np.abs(tau[ev]).mean())
    assert mean_tau[1] < mean_tau[0], mean_tau


def test_error_codes(model):
    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=1))
    f = _l.lib().b200sqp_set_joint_torque_cost
    for bad in (-1.0, np.nan, np.inf):
        w = W.copy()
        w[3] = bad
        assert f(s._h, w.ctypes.data_as(_l.dp)) == _l.EINVAL
    assert f(None, None) == _l.EINVAL
    cm = model_loader.load_packaged_model("g1_centroidal")
    c = B200SqpSolver(cm, abi.default_settings(cm, sqp_iteration=1))
    assert f(c._h, W.ctypes.data_as(_l.dp)) == _l.EINVAL
    assert f(c._h, None) == _l.EINVAL


def test_refused_while_a_fleet_is_attached(model):
    rng = np.random.default_rng(8)
    x0s, cmds = make_inputs(model, rng, 3)
    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=1))
    fl = B200SqpFleet(s)
    for w in (W, None):
        with pytest.raises(B200SqpError) as e:
            s.set_joint_torque_cost(w)
        assert e.value.code == _l.ESTATE
    fl.close()
    s.set_joint_torque_cost(W)   # detached: accepted again
    s.build_instances(0.0, 1.1, x0s, ["walk"] * 3, [0.0] * 3, cmds)
    s.solve()
    assert not s.primal_solution()["status"].any()


def test_mixed_gait_fleet_matches_the_plain_handle_per_group(model):
    """a fleet (builder path, one group view per node count) with the term on: each group's solve is bitwise the solve of the same
    instances uploaded to a plain handle with the term on, and differs from the fleet without the term"""
    rng = np.random.default_rng(9)
    B = 12
    x0s, cmds = make_inputs(model, rng, B)
    gaits, starts = mixed_batch(model, rng, B)
    st = abi.default_settings(model, sqp_iteration=2, use_feedback_policy=1)
    sols = []
    for w in (W, None):
        s = B200SqpSolver(model, st)
        s.set_joint_torque_cost(w)
        fl = B200SqpFleet(s)
        fl.build_instances(0.0, 1.1, x0s, gaits, starts, cmds)
        dev = fl.download_instances()
        fl.solve()
        sols.append((fl, dev, fl.primal_solution()))
    fl, dev, sol = sols[0]
    assert not sol["status"].any() and fl.n_groups >= 2
    for n in sorted(set(fl.n_nodes.tolist())):
        idx = np.flatnonzero(fl.n_nodes == n)
        p = B200SqpSolver(model, st)
        p.set_joint_torque_cost(W)
        p.upload({k: np.stack([dev[k][b] if k == "x0" else dev[k][b][: n - 1] if k == "u_init" else dev[k][b][:n] for b in idx]) for k in KEYS})
        p.solve()
        ref = p.primal_solution()
        assert np.array_equal(sol["x"][idx][:, :n], ref["x"]) and np.array_equal(sol["u"][idx][:, : n - 1], ref["u"]), n
        assert np.array_equal(sol["K"][idx][:, : n - 1], ref["K"]) and np.array_equal(sol["log"][idx], ref["log"]), n
        assert not np.array_equal(sols[1][2]["x"][idx], sol["x"][idx]), n


def test_device_closed_loop_with_the_term(model):
    """the builder path with the term on: the cold build's solve matches the oracle with the term; then build(warm = 2) -> solve ->
    roll-out cycles run without status errors"""
    rng = np.random.default_rng(10)
    B, dt = 8, 1.0 / 80.0
    x0s, cmds = make_inputs(model, rng, B)
    st = abi.default_settings(model, sqp_iteration=1)
    s = B200SqpSolver(model, st)
    s.set_joint_torque_cost(W)
    s.build_instances(0.0, 1.1, x0s, ["walk"] * B, [0.0] * B, cmds)
    dev = s.download_instances()
    s.solve()
    sol = s.primal_solution()
    assert not sol["status"].any()
    for b in (0, B - 1):
        ref = jt.solve(model, {k: dev[k][b] for k in KEYS}, st, W)
        assert rel(sol["x"][b], ref["x"]) < 1e-7 and rel(sol["u"][b], ref["u"]) < 1e-7, b
    for c in range(10):
        t = c * dt
        r = s.rollout_policy(t, dt)
        assert not r["status"].any(), c
        s.build_instances(t + dt, 1.1, None, ["walk"] * B, [0.0] * B, cmds, warm="rollout")
        s.solve()
        assert not s.primal_solution()["status"].any(), c
