"""Automatic gait selection (ProceduralMpcMotionManager, ProceduralMpcMotionManager.cpp:44-160): the numpy restatement
(references.ProceduralMpcMotionManager) pinned with hand-derived cases, then the device functions (wb_builder.cuh: bldMotionFilter,
bldMotionTransition, and the stateful grid pass bldGridInstance with the manager) run on the CPU against it.  CPU only."""
import math

import numpy as np
import pytest

from wb_humanoid_mpc_b200 import abi, model_loader
from wb_humanoid_mpc_b200 import references as R

PM = R.ProceduralMpcMotionManager
HORIZON, DT_MPC = 1.1, 0.05


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


def x0_with(model, bv=(0, 0, 0, 0, 0, 0)):
    x0 = np.array(model["x_init"], float)
    nv = 6 + model["nj"]
    x0[nv:nv + 6] = bv
    return x0


def test_seven_gaits_and_scales_are_packaged(model):
    _, names = abi.builder_desc(model)
    assert all(g in names for g in abi.MOTION_GAITS)
    assert [s[0] for s in PM.STATES] == abi.MOTION_GAITS
    r = model["reference"]
    assert (r["maxDisplacementVelocityX"], r["maxDisplacementVelocityY"], r["maxRotationVelocity"]) == (2.0, 1.2, 1.0)
    md = abi.motion_desc(model, names, 0.5)
    assert [names[g] for g in md.gait] == abi.MOTION_GAITS and md.filter_origin == 0.5
    with pytest.raises(ValueError, match="run"):
        abi.motion_desc(model, [n for n in names if n != "run"])


def test_alpha_of_the_time_since_construction(model):
    m = PM(model, filter_origin=1.0)
    tau = 1 / (2 * math.pi * 5.0)
    assert tau == pytest.approx(0.0318309886183791, abs=1e-15)
    assert m.alpha(1.0) == 0.0
    assert m.alpha(1.0 + tau) == pytest.approx(0.5, abs=1e-15)
    assert m.alpha(1.1) == pytest.approx(0.1 / (0.1 + 0.0318309886183791), abs=1e-15)
    assert m.alpha(11.0) == pytest.approx(10 / 10.0318309886183791, abs=1e-15)
    # the filter never keeps its output: the same input gives the same output at the same time, whatever came before
    a = m.filtered_command([0.5, 0, 0.8, 0], 2.0)
    m.filtered_command([1, 1, 1, 1], 1.5)
    assert np.array_equal(a, m.filtered_command([0.5, 0, 0.8, 0], 2.0))


def test_command_is_clamped_then_scaled(model):
    m = PM(model)
    assert PM.message_command([2.0, -3.0, 0.1, 0.5]) == [1.0, -1.0, 0.2, 0.5]
    assert PM.message_command([-0.3, 0.4, 1.7, -4.0]) == [-0.3, 0.4, 1.0, -1.0]
    assert m.scaled_command([2.0, -3.0, 0.1, 0.5]) == [2.0, -1.2, 0.2, 0.5]
    assert m.scaled_command([0.25, 0.5, 0.8, -0.5]) == [0.5, 0.6, 0.8, -0.5]   # the height is not scaled
    f = m.filtered_command([0.25, 0.5, 0.8, -0.5], 1.0)
    a = 1.0 / (1.0 + 1 / (2 * math.pi * 5.0))
    assert np.array_equal(f, [a * 0.5, a * 0.6, a * 0.8, a * -0.5])   # the height ramps too


@pytest.mark.parametrize("state,f,bv,fires", [
    (0, [0.1, 0, 0, 0], [0] * 6, False),               # stance: |f0| > 0.1 is strict
    (0, [0.1000001, 0, 0, 0], [0] * 6, True),          # ... and the base-speed term passes with the 10.0 threshold
    (0, [0, -0.2, 0, 0], [0] * 6, True),
    (0, [0, 0, 0, 0.1000001], [0] * 6, True),
    (2, [0.6, 0, 0, 0], [0.45, 0, 0, 0, 0, 0], False),   # walk: |bv0| > 0.5 - 0.05 is strict
    (2, [0.6, 0, 0, 0], [0.4500001, 0, 0, 0, 0, 0], True),
    (2, [0.6, 0, 0, 0], [0, 0, 0, 0.3000001, 0, 0], True),   # the yaw term reads bv3
    (2, [0.6, 0, 0, 0], [0, 0, 0, 0, 0, 5.0], False),
])
def test_faster_at_band_edges(state, f, bv, fires):
    assert PM.faster(f, bv, PM.STATES[state]) is fires


@pytest.mark.parametrize("state,f,bv,fires", [
    (1, [0.0499999, 0, 0, 0], [0] * 6, True),          # slow_walk: all of |f0|, |f1| < 0.05, |f3| < 0.05
    (1, [0.05, 0, 0, 0], [0] * 6, False),
    (1, [0, 0, 0, 0.05], [0] * 6, False),
    (1, [0, 0, 0, 0], [0.1, 0, 0, 0, 0, 0], False),    # |bv0| < 0.05 + 0.05 is strict
    (1, [0, 0, 0, 0], [0.0999999, 0.0999999, 0, 0, 0, 0], True),
    (1, [0, 0, 0, 0], [0, 0, 0, 5.0, 0, 5.0], True),   # the quirk: the last term tests |f3|, so a fast yaw of the base does not block it
    (0, [0, 0, 0, 0], [0] * 6, False),                 # stance never goes slower (|f| < -0.1 is impossible)
])
def test_slower_at_band_edges(state, f, bv, fires):
    assert PM.slower(f, bv, PM.STATES[state]) is fires


def run_cycles(model, m, raws, bvs, t_start=0.0):
    out = []
    for c, (raw, bv) in enumerate(zip(raws, bvs)):
        t0 = t_start + c * DT_MPC
        x0 = x0_with(model, bv)
        if c == 0:
            tt = m.start(raw, t0, t0 + HORIZON, x0)
            cmd = None
        else:
            tt, cmd = m.pre_solver_run(raw, t0, t0 + HORIZON, x0)
        out.append((t0, tt, cmd, m.state, m.last_change))
    return out


def test_hold_is_strict_and_starts_at_zero(model):
    m = PM(model, filter_origin=-1e6)   # alpha = 1 to round-off
    x0 = x0_with(model)
    m.start([0.5, 0, 0.8, 0], 0.0, HORIZON, x0)
    _, cmd = m.pre_solver_run([0.5, 0, 0.8, 0], 0.2, 0.2 + HORIZON, x0)
    assert (m.state, cmd) == (0, None)   # 0.2 > 0.0 + 0.2 is false
    _, cmd = m.pre_solver_run([0.5, 0, 0.8, 0], 0.2000001, 0.2000001 + HORIZON, x0)
    assert (m.state, m.last_change, cmd) == (1, 0.2000001, "slow_walk")
    _, cmd = m.pre_solver_run([0.5, 0, 0.8, 0], 0.4000001, 0.4000001 + HORIZON, x0)
    assert (m.state, cmd) == (1, None)   # held: 0.4000001 > 0.2000001 + 0.2 is false in double arithmetic


def test_one_step_per_cycle_and_the_delay_of_the_targets(model):
    m = PM(model, filter_origin=0.0)
    n = 80
    raws = [[1.0, 0.0, 0.8, 0.0]] * 40 + [[0.0, 0.0, 0.8, 0.0]] * 40
    bvs = [[2.0, 0, 0, 0, 0, 0]] * 40 + [[0.0] * 6] * 40
    res = run_cycles(model, m, raws, bvs)
    states = [r[3] for r in res]
    assert max(states) == 6 and states[-1] == 0
    assert all(abs(a - b) <= 1 for a, b in zip(states, states[1:]))
    changes = [r[0] for r, p in zip(res[1:], res[:-1]) if r[3] != p[3]]
    assert all(b - a > 0.2 for a, b in zip(changes, changes[1:]))
    for r, p in zip(res[1:], res[:-1]):
        assert (r[2] is not None) == (r[3] != p[3])
    # cycle c solves with the knots of cycle c - 1: the times and the filtered command of that cycle
    for c in range(1, n):
        t_prev = res[c - 1][0]
        tt_prev, ts_prev = R.velocity_command_targets(model, t_prev, x0_with(model, bvs[c - 1]), PM(model).filtered_command(raws[c - 1], t_prev),
                                                    (t_prev + HORIZON) - t_prev)
        tt, ts = res[c][1]
        assert np.array_equal(tt, tt_prev) and np.allclose(ts, ts_prev, rtol=0, atol=1e-15)
    # the cold build uses its own knots
    assert res[0][1][0][0] == 0.0


# ---- the device functions on the CPU ------------------------------------------------------------------------------------------------------------
def test_device_filter_and_transitions_equal_the_restatement(model):
    import bld_emu_lib as E

    _, names = abi.builder_desc(model)
    md = abi.motion_desc(model, names, 0.3)
    m = PM(model, filter_origin=0.3)
    rng = np.random.default_rng(5)
    for _ in range(200):
        raw = rng.uniform(-1.5, 1.5, 4)
        raw[2] = rng.uniform(0.0, 1.2)
        t0 = 0.3 + rng.uniform(0, 5)
        assert np.array_equal(E.motion_filter(md, raw, t0), m.filtered_command(raw, t0))
    # every band edge of every state, for both transitions, exactly on and next to the edge
    for s, cfg in enumerate(PM.STATES):
        _, mn, mx, amn, amx, lt, at = cfg
        for v in (mn, mx, mn + lt, mx - lt, amn, amx, amn + at, amx - at):
            for e in (np.nextafter(v, -np.inf), v, np.nextafter(v, np.inf)):
                for k in range(8):
                    f, bv = np.zeros(4), np.zeros(6)
                    if k & 1:
                        f[0] = e
                    else:
                        f[3] = e
                    if k & 2:
                        bv[0] = e
                    if k & 4:
                        bv[3] = e
                    exp = s
                    if PM.faster(f, bv, cfg) and s < 6:
                        exp = s + 1
                    elif PM.slower(f, bv, cfg) and s > 0:
                        exp = s - 1
                    got, lc = E.motion_transition(s, 0.0, f, bv, 1.0)
                    assert got == exp and lc == (1.0 if exp != s else 0.0), (s, v, k)
                    assert E.motion_transition(s, 0.8, f, bv, 1.0) == (s, 0.8)   # the hold


def template(model, gait):
    g = model["gaits"][gait]
    return [R.MODE_NAMES[m] for m in g["modeSequence"]], g["switchingTimes"]


def test_stateful_grid_pass_with_the_manager_equals_the_restatement(model):
    """300 cycles of random raw commands (the clamp included) and measured base velocities, instances starting in different states: the
    manager state, the gait schedules and the targets of every pass against the restatement driving GaitSchedule.update_gait"""
    import bld_emu_lib as E

    B, cycles, origin = 4, 300, -0.05
    rng = np.random.default_rng(17)
    _, names = abi.builder_desc(model)
    md = abi.motion_desc(model, names, origin)
    emu = E.EmuBuilder(model, B, HORIZON, stateful=True, motion=md)
    start = ["stance", "walk", "slow_trot", "run"]
    mgr = [PM(model, filter_origin=origin, state=g) for g in start]
    gs = []
    for g in start:
        s = R.GaitSchedule()
        if g != "stance":
            s.insert_template(*template(model, g), 0.0, 2 * HORIZON)
        gs.append(s)
    level = rng.uniform(-1.2, 1.2, (B, 4))
    seen, switches = set(), 0
    for c in range(cycles):
        t0 = c * DT_MPC
        if c % 20 == 0:   # piecewise-constant commands, so that the state machine gets somewhere
            level = rng.uniform(-1.2, 1.2, (B, 4))
            level[:, 1] *= 0.3
            level[:, 3] *= 0.3
            level[:, 2] = rng.uniform(0.0, 1.2, B)
        raw = level + rng.normal(0, 0.02, (B, 4))
        x0 = np.array([x0_with(model, rng.uniform(-1, 1, 6) * [1.5, 0.3, 0.1, 0.3, 0.1, 0.3]) for _ in range(B)])
        for b in range(B):
            x0[b, :4] += rng.uniform(-0.1, 0.1, 4)
        tf = t0 + HORIZON
        # (the stance template started at 0.5 is GaitSchedule's default schedule)
        dev = emu.build(t0, x0, raw, gaits=start, gait_start=[0.5 if g == "stance" else 0.0 for g in start], warm=c > 0)
        for b in range(B):
            T = tf - t0   # the window of the device, in its arithmetic
            ms = gs[b].get_mode_schedule(t0 - T, tf + T)
            if c == 0:
                tt, ts = mgr[b].start(raw[b], t0, tf, x0[b])
            else:
                (tt, ts), cmd = mgr[b].pre_solver_run(raw[b], t0, tf, x0[b])
                if cmd is not None:
                    gs[b].update_gait(*template(model, cmd), t0, tf)
                    switches += 1
            assert dev["state"][b] == mgr[b].state and dev["last_change"][b] == mgr[b].last_change, (c, b)
            assert np.allclose(dev["filtered"][b], mgr[b].filtered, rtol=0, atol=1e-12)
            assert np.allclose(dev["tt_time"][b], tt, rtol=0, atol=1e-12)
            assert np.allclose(dev["tt_state"][b], ts, rtol=0, atol=1e-12)
            ev, modes = dev["schedules"][b]
            assert modes == ms.mode_sequence and ev == ms.event_times, (c, b)
            seen.add(mgr[b].state)
    assert switches >= 10 and len(seen) >= 5
