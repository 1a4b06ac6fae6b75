"""The device builder's pose commands (wb_builder.cuh bldPoseUpdate / bldPoseLatch / bldPoseKnots, then bldNode's getDesiredState) on the CPU
harness tests/emu/bld_emu.cu, whole-body and centroidal: x_ref at every node against the restatement references.pose_command_targets, the latch
across warm builds, clear / reset / re-latch, and bit-identity with the mode off for every instance without a command."""
import numpy as np
import pytest

from bld_emu_lib import NX, EmuBuilder
from wb_humanoid_mpc_b200 import model_loader, references

WEAK_EPS = 1e-9
B, HORIZON = 4, 1.0


@pytest.fixture(scope="module", params=["g1_wb", "g1_centroidal"])
def model(request):
    return model_loader.load_packaged_model(request.param)


def _states(model, seed, t=0.0):
    """B measured states at the device stride (the base pose moving with t); centroidal: zero momentum and padding"""
    rng = np.random.default_rng(seed)
    cen = model.get("kind") == "centroidal"
    o = 6 if cen else 0
    x = np.zeros((B, NX))
    x[:, o + 6:o + 6 + model["nj"]] = np.asarray(model["reference"]["defaultJointState"]) + 0.05 * rng.normal(size=(B, model["nj"]))
    x[:, o:o + 6] = [0.0, 0.0, 0.76, 0.0, 0.02, -0.01] + 0.1 * rng.normal(size=(B, 6))
    x[:, o] += 0.3 * t
    x[:, o + 3] += 0.2 * t
    if not cen:
        x[:, 6 + model["nj"]:] = 0.1 * rng.normal(size=(B, NX - 6 - model["nj"]))
    return x


def _args(model):
    h = model["reference"]["defaultBaseHeight"]
    cmd = np.array([[0.3, 0.0, h, 0.1], [0.0, 0.1, h, -0.2], [0.2, -0.1, h, 0.0], [0.0, 0.0, h, 0.3]])
    return cmd, ["walk", "stance", "walk", "stance"], np.zeros(B)


def _expect_xref(model, t0, x0row, delta, out, i):
    """the restatement's 2-knot targets latched at t0 from x0row, interpolated at the node times (getIntervalStart) of instance i"""
    nx = model["nx"]
    tt, ss = references.pose_command_targets(model, t0, x0row[:nx], delta)
    n = out["n_nodes"][i]
    want = np.zeros((n, NX))
    for k in range(n):
        t = out["t_nodes"][i, k] + (WEAK_EPS if out["node_event"][i, k] == 2 else 0.0)
        want[k, :nx] = references.interp_targets(tt, ss, t)
    return tt, ss, want


def test_latch_matches_the_restatement_and_leaves_other_instances_alone(model):
    on, off = EmuBuilder(model, B, HORIZON, stateful=True, pose=True), EmuBuilder(model, B, HORIZON, stateful=True)
    cmd, gaits, gs = _args(model)
    cmds = {1: [1.0, 0.0, 0.0, 0.0], 3: [0.2, -0.3, 0.5, 90.0]}
    x0 = _states(model, 1)
    a = on.build(0.0, x0, cmd, gaits, gs, warm=False, commands=cmds, nodes="slots")
    b = off.build(0.0, x0, cmd, gaits, gs, warm=False, nodes="slots")
    assert np.array_equal(a["t_nodes"], b["t_nodes"]) and np.array_equal(a["n_nodes"], b["n_nodes"])
    for i in range(B):
        n = a["n_nodes"][i]
        if i in cmds:
            tt, ss, want = _expect_xref(model, 0.0, x0[i], cmds[i], a, i)
            assert np.allclose(a["x_ref"][i, :n], want, rtol=0, atol=1e-12), i
            assert a["active"][i] and a["t_start"][i] == 0.0 and abs(a["t_reach"][i] - tt[1]) < 1e-12
            o = 6 if model.get("kind") == "centroidal" else 0
            assert np.allclose(a["target"][i], ss[1][o:o + 6], rtol=0, atol=1e-12)
            assert np.allclose(a["error"][i], [np.hypot(*(x0[i, o:o + 2] - ss[1][o:o + 2])), abs(x0[i, o + 3] - ss[1][o + 3])], rtol=0, atol=1e-12)
        else:
            assert np.array_equal(a["x_ref"][i], b["x_ref"][i]), i   # the velocity rule, bit for bit
            assert not a["active"][i] and not a["error"][i].any()


def test_zero_displacement_switches_to_the_target_after_t0(model):
    on = EmuBuilder(model, B, HORIZON, stateful=True, pose=True)
    cmd, gaits, gs = _args(model)
    x0 = _states(model, 2)
    a = on.build(0.5, x0, cmd, gaits, gs, warm=False, commands={0: [0.0, 0.0, 0.0, 0.0]}, nodes="slots")
    assert a["t_reach"][0] == a["t_start"][0] == 0.5
    tt, ss, want = _expect_xref(model, 0.5, x0[0], [0.0, 0.0, 0.0, 0.0], a, 0)
    n = a["n_nodes"][0]
    assert np.isfinite(a["x_ref"][0, :n]).all() and np.array_equal(a["x_ref"][0, :n], want)
    assert np.array_equal(a["x_ref"][0, 1, :model["nx"]], ss[1])


def test_latched_target_survives_warm_builds_and_relatches(model):
    on = EmuBuilder(model, B, HORIZON, stateful=True, pose=True)
    cmd, gaits, gs = _args(model)
    d2 = [1.5, 0.5, -0.1, -30.0]
    x0 = _states(model, 3)
    first = on.build(0.0, x0, cmd, gaits, gs, warm=False, commands={2: d2}, nodes="slots")
    o = 6 if model.get("kind") == "centroidal" else 0
    for step in range(1, 6):
        t0 = 0.1 * step
        xs = _states(model, 3, t=t0)   # the measured state moves
        w = on.build(t0, xs, cmd, gaits, gs, nodes="slots")
        assert w["active"][2] and w["t_start"][2] == 0.0 and w["t_reach"][2] == first["t_reach"][2]
        assert np.array_equal(w["target"][2], first["target"][2])
        _, ss, want = _expect_xref(model, 0.0, x0[2], d2, w, 2)   # the targets of the first latch, at this build's nodes
        n = w["n_nodes"][2]
        assert np.allclose(w["x_ref"][2, :n], want, rtol=0, atol=1e-12)
        assert np.allclose(w["error"][2], [np.hypot(*(xs[2, o:o + 2] - ss[1][o:o + 2])), abs(xs[2, o + 3] - ss[1][o + 3])], rtol=0, atol=1e-12)
    # a new command on the active instance re-latches it from the new build's state
    xs = _states(model, 3, t=0.6)
    d3 = [0.0, 1.0, 0.0, 45.0]
    w = on.build(0.6, xs, cmd, gaits, gs, commands={2: d3}, nodes="slots")
    _, _, want = _expect_xref(model, 0.6, xs[2], d3, w, 2)
    assert w["t_start"][2] == 0.6 and np.allclose(w["x_ref"][2, :w["n_nodes"][2]], want, rtol=0, atol=1e-12)


def test_clear_reset_and_cold_build_restore_the_velocity_rule(model):
    on = EmuBuilder(model, B, HORIZON, stateful=True, pose=True, reset=dict(on=False))   # (requested resets only)
    off = EmuBuilder(model, B, HORIZON, stateful=True, reset=dict(on=False))
    cmd, gaits, gs = _args(model)
    x0 = _states(model, 4)
    cmds = {0: [1.0, 0.0, 0.0, 0.0], 1: [0.0, 0.5, 0.0, 30.0], 3: [-0.5, 0.0, 0.2, -60.0]}
    on.build(0.0, x0, cmd, gaits, gs, warm=False, commands=cmds, nodes="slots")
    off.build(0.0, x0, cmd, gaits, gs, warm=False, nodes="slots")
    xs = _states(model, 4, t=0.1)
    a = on.build(0.1, xs, cmd, gaits, gs, nodes="slots")
    off.build(0.1, xs, cmd, gaits, gs, nodes="slots")
    assert a["active"][[0, 1, 3]].all()
    # instance 0 cleared, instance 1 reset (to the reset row xs[1]), instance 3 keeps its target
    rst = np.array([0, 1, 0, 0], np.uint8)
    xr = _states(model, 4, t=0.2)
    for emu in (on, off):
        emu.set_reset_states(xr, ["stance"] * B, np.zeros(B))
    a = on.build(0.2, xr, cmd, gaits, gs, requests=rst, clears=[0], nodes="slots")
    b = off.build(0.2, xr, cmd, gaits, gs, requests=rst, nodes="slots")
    assert a["active"].tolist() == [False, False, False, True]
    for i in (0, 1, 2):
        assert np.array_equal(a["x_ref"][i], b["x_ref"][i]), i
    assert not np.array_equal(a["x_ref"][3], b["x_ref"][3])
    # the next warm build: still the velocity rule for 0 and 1
    xs = _states(model, 4, t=0.3)
    a, b = on.build(0.3, xs, cmd, gaits, gs, nodes="slots"), off.build(0.3, xs, cmd, gaits, gs, nodes="slots")
    assert a["active"].tolist() == [False, False, False, True]
    assert all(np.array_equal(a["x_ref"][i], b["x_ref"][i]) for i in (0, 1, 2))
    # a cold build drops every target, then latches the commands pending for it
    a = on.build(0.0, x0, cmd, gaits, gs, warm=False, commands={2: [0.3, 0.0, 0.0, 0.0]}, nodes="slots")
    b = off.build(0.0, x0, cmd, gaits, gs, warm=False, nodes="slots")
    assert a["active"].tolist() == [False, False, True, False]
    assert all(np.array_equal(a["x_ref"][i], b["x_ref"][i]) for i in (0, 1, 3))


def test_mode_off_is_bit_identical_to_a_run_without_commands(model):
    """pose commands enabled but never issued: every build equals the builder without them, bit for bit"""
    on, off = EmuBuilder(model, B, HORIZON, stateful=True, pose=True), EmuBuilder(model, B, HORIZON, stateful=True)
    cmd, gaits, gs = _args(model)
    for step in range(4):
        xs = _states(model, 5, t=0.1 * step)
        a, b = on.build(0.1 * step, xs, cmd, gaits, gs, warm=step > 0, nodes="slots"), off.build(0.1 * step, xs, cmd, gaits, gs, warm=step > 0, nodes="slots")
        for k in ("n_nodes", "t_nodes", "node_event", "x_ref"):
            assert np.array_equal(a[k], b[k]), k
        assert not a["active"].any()
