"""Automatic gait selection on the centroidal MPC (the ProceduralMpcMotionManager of the reference's centroidal node): the numpy restatement
(references.ProceduralMpcMotionManager with a centroidal model) pinned with hand-derived cases, the device builder's stateful grid pass on a
centroidal handle (wb_builder.cuh: bldCenBaseVelocity + bldGridInstance, with and without the manager) run on the CPU against it, and the C++
host layer's manager (host/references.hpp) against it.  CPU only."""
import math

import numpy as np
import pytest

import bld_emu_lib as E
import oracle_lib as orc
from wb_humanoid_mpc_b200 import abi, centroidal, host_lib, model_loader
from wb_humanoid_mpc_b200 import references as R

PM = R.ProceduralMpcMotionManager
HORIZON, DT_MPC = 1.2, 1.0 / 80.0   # the centroidal task.info: timeHorizon 1.2, mpcDesiredFrequency 80


def cen_model(model_type):
    m = dict(model_loader.load_packaged_model("g1_centroidal"))
    m["centroidalModelType"] = model_type
    return m


@pytest.fixture(scope="module", params=[0, 1], ids=["full", "srbd"])
def model(request):
    return cen_model(request.param)


def x0_with(model, hbar=(0, 0, 0, 0, 0, 0)):
    x0 = np.array(model["x_init"], float)
    x0[:6] = hbar
    return x0


def template(model, gait):
    g = model["gaits"][gait]
    return [R.MODE_NAMES[m] for m in g["modeSequence"]], g["switchingTimes"]


def edge_values():
    """every band threshold of the table (and its negative), exactly"""
    v = set()
    for _, mn, mx, amn, amx, lt, at in PM.STATES:
        v |= {mn, mx, mn + lt, mx - lt, amn, amx, amn + at, amx - at}
    return sorted(v | {-x for x in v})


# ---- the restatement, hand-derived -------------------------------------------------------------------------------------------------------------
def test_the_centroidal_scales_are_those_of_its_reference_info():
    model = cen_model(0)
    r = model["reference"]
    assert (r["maxDisplacementVelocityX"], r["maxDisplacementVelocityY"], r["maxRotationVelocity"]) == (2.4, 1.2, 1.0)
    _, names = abi.builder_desc(model)
    md = abi.motion_desc(model, names, 0.25)
    assert (md.max_velocity_x, md.max_velocity_y, md.max_rotation_velocity, md.filter_origin) == (2.4, 1.2, 1.0, 0.25)
    m = PM(model)
    assert m.scaled_command([1.0, 0.5, 0.8, -0.5]) == [2.4, 0.6, 0.8, -0.5]
    assert m.scaled_command([0.25, -2.0, 1.7, 3.0]) == [0.6, -1.2, 1.0, 1.0]   # clamped, then scaled (0.25 * 2.4 = 0.6 exactly)


def test_the_targets_follow_the_centroidal_rule_with_one_cycle_of_delay():
    model = cen_model(1)
    m = PM(model, filter_origin=-0.5)
    hbar = [0.3, -0.1, 0.02, 0.01, -0.02, 0.05]
    x0 = x0_with(model, hbar)
    bv = centroidal.srbd_base_velocity(model, x0)
    tt0, ts0 = m.start([0.5, 0.2, 0.8, 0.3], 0.0, HORIZON, x0, base_vel=bv)
    f0 = m.filtered_command([0.5, 0.2, 0.8, 0.3], 0.0)
    ett, ets = R.velocity_command_targets_centroidal(model, 0.0, x0, f0, HORIZON, bv)
    assert np.array_equal(tt0, ett) and np.array_equal(ts0, ets)
    # the knot layout: normalized momentum (v_gx, v_gy, 0, 0, 0, yaw rate / m) of the filtered command, then the base pose
    a = 0.5 / (0.5 + 1 / (2 * math.pi * 5.0))
    yaw = x0[9]
    assert ts0[0][0] == pytest.approx(math.cos(yaw) * a * 1.2 - math.sin(yaw) * a * 0.24, abs=1e-15)
    assert ts0[0][5] == pytest.approx(a * 0.3 / sum(model["mass"]), abs=1e-15)
    assert ts0.shape == (3, model["nx"])
    (tt1, ts1), _ = m.pre_solver_run([0.0, 0.0, 0.8, 0.0], DT_MPC, DT_MPC + HORIZON, x0, base_vel=bv)
    assert np.array_equal(tt1, tt0) and np.array_equal(ts1, ts0)   # this cycle solves with the previous cycle's targets
    with pytest.raises(ValueError, match="base_vel"):   # a non-zero momentum needs Ab^-1 hbar
        m.pre_solver_run([0.0, 0.0, 0.8, 0.0], 2 * DT_MPC, 2 * DT_MPC + HORIZON, x0)


def test_a_transition_fires_on_hbar_that_the_base_velocity_would_not_fire():
    """walk -> slower_trot needs |v| > 0.45 of the measured base velocity: hbar[0] = 0.5 passes, Ab^-1 hbar (about hbar / m) would not"""
    model = cen_model(1)
    m = PM(model, filter_origin=-1e6, state="walk")   # alpha = 1 to round-off
    x0 = x0_with(model, [0.5, 0.0, 0.0, 0.0, 0.0, 0.0])
    bv = centroidal.srbd_base_velocity(model, x0)
    assert abs(bv[0]) < 0.05 and np.max(np.abs(bv[[1, 3]])) < 0.05
    raw = [0.3, 0.0, 0.8, 0.0]   # 0.3 * 2.4 = 0.72 > walk's maxLinVelCmd 0.5
    m.start(raw, 0.0, HORIZON, x0, base_vel=bv)
    f = m.filtered_command(raw, 0.3)
    assert not PM.faster(f, bv, PM.STATES[2]) and PM.faster(f, x0[:6], PM.STATES[2])
    _, cmd = m.pre_solver_run(raw, 0.3, 0.3 + HORIZON, x0, base_vel=bv)
    assert (m.state, m.last_change, cmd) == (3, 0.3, "slower_trot")
    # and back: a zero command with hbar slow enough, once the hold has passed
    x0 = x0_with(model, [0.4999, 0.0, 0.0, 0.0, 0.0, 0.0])   # |hbar0| < slower_trot's 0.45 + 0.1
    _, cmd = m.pre_solver_run([0.0, 0.0, 0.8, 0.0], 0.6, 0.6 + HORIZON, x0, base_vel=centroidal.srbd_base_velocity(model, x0))
    assert (m.state, cmd) == (2, "walk")


# ---- the device functions on the CPU ------------------------------------------------------------------------------------------------------------
def random_state(model, rng, edges):
    """a measured state with a random normalized momentum, its linear x / y and yaw rows on band edges a third of the time"""
    x0 = x0_with(model, rng.uniform(-1, 1, 6) * [1.5, 0.3, 0.1, 0.3, 0.1, 0.3])
    for k in (0, 1, 3):
        if rng.uniform() < 0.3:
            x0[k] = edges[rng.integers(len(edges))]
    x0[6:8] += rng.uniform(-0.1, 0.1, 2)
    x0[9:12] += rng.uniform(-0.1, 0.1, 3)
    x0[12:] += rng.uniform(-0.05, 0.05, model["nj"])
    return x0


@pytest.mark.parametrize("manager", [True, False], ids=["manager", "plain"])
def test_stateful_grid_pass_equals_the_restatement(model, manager):
    """300 cycles of random raw commands and measured states (momentum on band edges included), instances starting in different gaits: the
    schedules exactly, the targets to 1e-12 with their padding exactly zero, the manager state exactly, against the restatement driving
    GaitSchedule.update_gait.  Without a manager the gait commands come from the caller and the targets from the raw command."""
    B, cycles, origin = 4, 300, -0.05
    rng = np.random.default_rng(23 + int(manager) + 2 * model["centroidalModelType"])
    _, names = abi.builder_desc(model)
    md = abi.motion_desc(model, names, origin) if manager else None
    emu = E.EmuBuilder(model, B, HORIZON, stateful=True, motion=md)
    start = ["stance", "walk", "slow_trot", "run"]
    mgr = [PM(model, filter_origin=origin, state=g) for g in start]
    gs = []
    for g in start:
        s = R.GaitSchedule()
        if g != "stance":
            s.insert_template(*template(model, g), 0.0, 2 * HORIZON)
        gs.append(s)
    last = list(start)
    edges = edge_values()
    level = rng.uniform(-1.2, 1.2, (B, 4))
    gaits = list(start)
    seen, switches = set(), 0
    for c in range(cycles):
        t0 = c * 4 * DT_MPC
        if c % 20 == 0:   # piecewise-constant commands, so that the state machine gets somewhere
            level = rng.uniform(-1.2, 1.2, (B, 4))
            level[:, 1] *= 0.3
            level[:, 3] *= 0.3
            level[:, 2] = rng.uniform(0.0, 1.2, B)
            if c > 0 and not manager:
                gaits = [str(rng.choice(abi.MOTION_GAITS)) for _ in range(B)]
        raw = level + rng.normal(0, 0.02, (B, 4))
        x0 = np.array([random_state(model, rng, edges) for _ in range(B)])
        tf = t0 + HORIZON
        dev = emu.build(t0, x0, raw, gaits if (c == 0 or not manager) else start, gait_start=[0.5 if g == "stance" else 0.0 for g in start], warm=c > 0)
        assert dev["pad_max"] == 0.0, c
        for b in range(B):
            bv = dev["bv"][b]   # bldCenBaseVelocity of x0 (tests/test_emu_cen_builder.py checks it against the oracle)
            T = tf - t0   # the window of the device, in its arithmetic
            ms = gs[b].get_mode_schedule(t0 - T, tf + T)
            if manager:
                if c == 0:
                    tt, ts = mgr[b].start(raw[b], t0, tf, x0[b], base_vel=bv)
                else:
                    (tt, ts), cmd = mgr[b].pre_solver_run(raw[b], t0, tf, x0[b], base_vel=bv)
                    if cmd is not None:
                        gs[b].update_gait(*template(model, cmd), t0, tf)
                        switches += 1
                assert dev["state"][b] == mgr[b].state and dev["last_change"][b] == mgr[b].last_change, (c, b)
                assert np.allclose(dev["filtered"][b], mgr[b].filtered, rtol=0, atol=1e-12)
                seen.add(mgr[b].state)
            else:
                tt, ts = R.velocity_command_targets_centroidal(model, t0, x0[b], raw[b], T, bv)
                if c > 0 and gaits[b] != last[b]:
                    gs[b].update_gait(*template(model, gaits[b]), t0, tf)
                    last[b] = gaits[b]
                    switches += 1
                seen.add(gaits[b])
            assert np.allclose(dev["tt_time"][b], tt, rtol=0, atol=1e-12)
            assert np.allclose(dev["tt_state"][b], ts, rtol=0, atol=1e-12)
            ev, modes = dev["schedules"][b]
            assert modes == ms.mode_sequence and ev == ms.event_times, (c, b)
    assert switches >= 10 and len(seen) >= 5, (switches, seen)


# ---- the C++ host layer --------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hmodel():
    m = host_lib.HostModel(host_lib.CEN_MODEL_TXT)
    yield m
    m.close()


@pytest.mark.parametrize("start,origin,seed", [("stance", 0.0, 4), ("trot", -0.2, 5)])
def test_cpp_centroidal_manager_equals_the_python_restatement(hmodel, start, origin, seed):
    """500 cycles each, the base velocity Ab^-1 hbar from the oracle's flow map (full centroidal dynamics) given to both"""
    model = cen_model(0)
    assert hmodel.dump()[12:15].tolist() == [2.4, 1.2, 1.0]
    oracle = orc.CenOracle(model)
    mass = sum(model["mass"])
    rng = np.random.default_rng(seed)
    cycles, dt = 500, 0.03
    cc = host_lib.HostMotionManager(hmodel, origin, start)
    py = PM(model, filter_origin=origin, state=start)
    edges = edge_values()
    changes, seen = 0, set()
    for c in range(cycles):
        t0 = origin + 0.01 + c * dt
        tf = t0 + HORIZON
        if c % 25 == 0:
            level = rng.uniform(-1.3, 1.3, 4)
            level[2] = rng.uniform(0.0, 1.3)
            slow = rng.uniform() < 0.5   # a stop: every velocity small, the momentum small too
            if slow:
                level[[0, 1, 3]] *= 0.03
        raw = level + rng.normal(0, 0.01, 4)
        x0 = random_state(model, rng, edges)
        if slow:
            x0[:6] *= 0.05
        bv = oracle.flow_map(x0, np.zeros(model["nu"]))[6:12] / mass
        out = cc.step_bv(c == 0, t0, tf, x0, raw, bv)
        if c == 0:
            tt, ts = py.start(raw, t0, tf, x0, base_vel=bv)
            cmd = None
        else:
            (tt, ts), cmd = py.pre_solver_run(raw, t0, tf, x0, base_vel=bv)
        assert out["state"] == py.state and out["last_change"] == py.last_change, c
        assert out["changed"] == (cmd is not None), c
        assert np.allclose(out["filtered"], py.filtered, rtol=0, atol=1e-12)
        assert np.allclose(out["targets"][0], tt, rtol=0, atol=1e-12)
        assert np.allclose(out["targets"][1], ts, rtol=0, atol=1e-12)
        changes += cmd is not None
        seen.add(py.state)
    assert changes >= 10 and len(seen) >= 5, (changes, seen)
