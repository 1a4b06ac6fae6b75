"""Policy roll-out on the device (b200sqp_rollout_policy, policy_rollout_kernel) after real solves: against the restatement of
MRT_BASE::rolloutPolicy around the oracle's flow map (rollout_ref.py) for both controllers, the closed loop build(warm = 2) -> solve -> roll-out
equal bit for bit to the same loop driven through host copies, and the error paths."""
import ctypes as C
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest

import oracle_lib as orc
import rollout_ref
from test_gpu_builder import make_inputs
from wb_humanoid_mpc_b200 import abi, model_loader
from wb_humanoid_mpc_b200.lib import B200SqpError

ROOT = Path(__file__).resolve().parents[1]
MRT_DT = 1.0 / 80.0
B, HORIZON = 8, 1.1


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


def solved(model, feedback, sqp_iteration=1, seed=21):
    from wb_humanoid_mpc_b200.solver import B200SqpSolver

    x0s, cmds = make_inputs(model, np.random.default_rng(seed), B)
    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=sqp_iteration, use_feedback_policy=int(feedback)))
    s.build_instances(0.0, HORIZON, x0s, ["walk"] * B, [0.0] * B, cmds)
    s.solve()
    return s, x0s, cmds


def plans(solver):
    inp = solver.download_instances()
    sol = solver.primal_solution()
    out = []
    for b in range(solver.batch):
        out.append((dict(t_nodes=inp["t_nodes"][b], node_event=inp["node_event"][b], contact_flags=inp["contact_flags"][b], x=sol["x"][b], u=sol["u"][b]),
                    sol.get("K", [None] * solver.batch)[b]))
    return out


def plan_state(plan, t):
    i, a = rollout_ref.time_segment(t, list(plan["t_nodes"]))
    return a * plan["x"][i] + (1 - a) * plan["x"][i + 1]


def rel(a, b):
    return float(np.max(np.abs(a - b)) / max(1e-300, np.max(np.abs(b))))


@pytest.mark.gpu
@pytest.mark.parametrize("feedback", [False, True], ids=["feedforward", "feedback"])
def test_kernel_matches_the_reference_restatement(model, feedback):
    solver, _, _ = solved(model, feedback)
    ps = plans(solver)
    te = min(float(p["t_nodes"][k]) for p, _ in ps for k in range(len(p["t_nodes"])) if p["node_event"][k] == 1)
    wb = orc.WbOracle(model)
    rng = np.random.default_rng(4)
    for t in (0.0, te - 0.4 * MRT_DT):   # a step without and one with a contact switch inside it
        xs = np.array([plan_state(p, t) for p, _ in ps])
        xs[:, 29:35] += rng.normal(0.0, 0.2, (B, 6))
        dev = solver.rollout_policy(t, MRT_DT, x_start=xs)
        for b, (p, K) in enumerate(ps):
            ref = rollout_ref.rollout_policy(wb.flow_map, p, t, MRT_DT, xs[b], K=K)
            assert dev["status"][b] == ref["status"] == 0
            assert tuple(dev["n_steps"][b]) == (ref["accepted"], ref["rejected"], ref["calls"]), (b, t)
            assert dev["mode"][b] == ref["mode"]
            assert rel(dev["x"][b], ref["x"]) < 1e-12 and rel(dev["u"][b], ref["u"]) < 1e-12, (b, t)


@pytest.mark.gpu
def test_closed_loop_on_the_device_equals_the_host_driven_loop(model):
    """40 cycles of build(warm = 2) -> solve -> roll-out without host copies equal, bit for bit, the loop that downloads x_end and uploads it as
    the next measured state (build_instances(x0 = x_end, warm = 1))"""
    dev, x0s, cmds = solved(model, True)
    host, _, _ = solved(model, True)
    gaits, start = ["walk"] * B, [0.0] * B
    for c in range(40):
        t = c * MRT_DT
        rd = dev.rollout_policy(t, MRT_DT)
        rh = host.rollout_policy(t, MRT_DT)
        assert np.array_equal(rd["x"], rh["x"]) and not rd["status"].any(), c
        dev.build_instances(t + MRT_DT, HORIZON, None, gaits, start, cmds, warm="rollout")
        host.build_instances(t + MRT_DT, HORIZON, rh["x"], gaits, start, cmds, warm=True)
        assert np.array_equal(dev.download_instances()["x0"], rh["x"])
        dev.solve()
        host.solve()
        sd, sh = dev.primal_solution(), host.primal_solution()
        assert np.array_equal(sd["x"], sh["x"]) and np.array_equal(sd["u"], sh["u"]) and np.array_equal(sd["K"], sh["K"]), c


@pytest.mark.gpu
def test_call_order_and_handle_kind_are_checked(model):
    from wb_humanoid_mpc_b200.solver import B200SqpSolver

    x0s, cmds = make_inputs(model, np.random.default_rng(2), 2)
    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=1))
    s.build_instances(0.0, HORIZON, x0s, ["walk"] * 2, [0.0] * 2, cmds)
    with pytest.raises(B200SqpError) as e:   # no solve yet
        s.rollout_policy(0.0, MRT_DT)
    assert e.value.code == -5
    s.solve()
    with pytest.raises(B200SqpError) as e:   # warm = 2 without a roll-out
        s.build_instances(MRT_DT, HORIZON, None, ["walk"] * 2, [0.0] * 2, cmds, warm="rollout")
    assert e.value.code == -5
    with pytest.raises(B200SqpError) as e:   # a negative duration
        s.rollout_policy(0.0, -MRT_DT)
    assert e.value.code == -1
    # a roll-out past the plan's last node holds the policy at its end (the reference only warns)
    r = s.rollout_policy(HORIZON - 0.005, 0.05)
    assert not r["status"].any() and np.all(np.isfinite(r["x"]))
    cmodel = model_loader.load_packaged_model("g1_centroidal")
    cs = B200SqpSolver(cmodel, abi.default_settings(cmodel, sqp_iteration=1))
    with pytest.raises(B200SqpError) as e:
        cs.rollout_policy(0.0, MRT_DT)
    assert e.value.code == -1


def test_rollout_settings_struct_matches_the_header():
    src = '#include "b200sqp.h"\n#include <stdio.h>\nint main(){printf("%zu\\n", sizeof(b200sqp_rollout_settings));}\n'
    with tempfile.TemporaryDirectory() as td:
        p = Path(td) / "probe.c"
        p.write_text(src)
        exe = Path(td) / "probe"
        subprocess.run(["gcc", "-I", str(ROOT / "include"), str(p), "-o", str(exe)], check=True)
        size = int(subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout)
    assert size == C.sizeof(abi.RolloutSettings)


def test_default_rollout_settings_agree():
    from wb_humanoid_mpc_b200 import lib

    rs = abi.RolloutSettings()
    lib.lib().b200sqp_default_rollout_settings(C.byref(rs))
    py = abi.default_rollout_settings()
    assert [getattr(rs, f) for f, _ in rs._fields_] == [getattr(py, f) for f, _ in py._fields_] == [1e-5, 1e-3, 0.015, 10000.0]
