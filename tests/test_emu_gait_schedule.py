"""The device builder's stateful gait schedule and trajectorySpread functions (wb_builder.cuh) on the CPU harness (tests/emu/bld_emu.cu):
the spreading strategy and its application against the oracle (oracle/trajectory_spreading.hpp) on the reference's 17 recipes and on random
schedule changes, the inputs against the Python restatement in toPrimalSolution form, and the schedule / updater functions against both host
restatements over 300 cycles of random gait commands."""
import bisect

import numpy as np
import pytest

import bld_emu_lib as emu
import oracle_lib as orc
from test_oracle_spreading import CASES, rollout
from wb_humanoid_mpc_b200 import abi, host_lib, model_loader, references as R


def device_spread(ev, modes, nev, nmodes, t, tags, rng=None):
    """the harness on a previous solution whose state column 0 and input column 0 carry the sample tags; PreEvent nodes drawn by rng"""
    n = len(t)
    event = np.zeros(n, dtype=np.uint8)
    if rng is not None:
        event[1:-1] = rng.random(n - 2) < 0.2
    x = np.zeros((n, emu.NX))
    x[:, 0] = tags
    u = np.zeros((n - 1, emu.NU))
    u[:, 0] = np.arange(n - 1) + 0.5
    return emu.spread(ev, modes, nev, nmodes, t, event, x, u), event, u


def check_against_oracle(ev, modes, nev, nmodes, t, tags, event_data, rng=None):
    out = orc.trajectory_spread(ev, modes, nev, nmodes, t, tags[:, None].astype(float), tags, event_data)
    dev, event, u = device_spread(ev, modes, nev, nmodes, t, tags, rng)
    if any(v >= len(dev["t"]) for _, _, v in dev["triples"]):
        return None   # a spreading value behind eraseFrom: adjustTrajectory reads an erased sample (undefined in the reference)
    assert np.array_equal(dev["t"], out["t"])
    assert np.array_equal(dev["x"][:, 0], out["tags"].astype(float))
    assert (dev["will_truncate"], dev["will_spread"]) == (out["will_truncate"], out["will_spread"])
    assert dev["post_event_indices"] == out["post_event_indices"]
    # the same strategy on the toPrimalSolution inputs, against the Python restatement
    prim = R.to_primal_solution(t, event, np.zeros((len(t), 1)), u[:, :1])
    py = R.trajectory_spread(R.ModeSchedule(list(ev), list(modes)), R.ModeSchedule(list(nev), list(nmodes)), prim)
    assert np.array_equal(dev["u"][:, :1], np.asarray(py["u"]).reshape(-1, 1))
    ts = R.TrajectorySpreading().set(R.ModeSchedule(list(ev), list(modes)), R.ModeSchedule(list(nev), list(nmodes)), t)
    assert dev["triples"] == list(zip(ts.begin, ts.end, ts.value_idx))
    return dev


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_spreading_matches_the_oracle_on_the_reference_recipes(name):
    ev, modes, nev, nmodes, period, _ = CASES[name]
    ev, nev = [float(e) for e in ev], [float(e) for e in nev]
    t, tags, _, event_data = rollout(ev, modes, period)
    check_against_oracle(ev, modes, nev, nmodes, t, tags, event_data, np.random.default_rng(len(name)))


def random_pair(rng):
    n_ev = int(rng.integers(1, 7))
    ev = np.sort(rng.uniform(0.2, 2.8, n_ev)).tolist()
    modes = [int(m) for m in rng.integers(0, 4, n_ev + 1)]
    kind = int(rng.integers(0, 5))
    nev = np.sort(np.clip(np.array(ev) + rng.uniform(-0.3, 0.3, n_ev), 0.05, 2.95)).tolist()
    nmodes = list(modes)
    if kind == 1:      # the new schedule drops its first mode
        nev, nmodes = nev[1:], nmodes[1:]
    elif kind == 2:    # the tail changes
        nmodes[-1] = 9
    elif kind == 3:    # nothing matches
        nmodes = [m + 10 for m in nmodes]
    elif kind == 4:    # a matched event moves onto the final time
        nev[-1] = 2.95
    return ev, modes, nev, nmodes


def test_device_spreading_matches_the_oracle_on_random_schedule_changes():
    rng = np.random.default_rng(7)
    seen, skipped = set(), 0
    for _ in range(400):
        ev, modes, nev, nmodes = random_pair(rng)
        t0, tf = float(rng.uniform(0.0, 0.5)), float(rng.choice([rng.uniform(2.0, 3.0), 2.95]))
        t, tags, _, event_data = rollout(ev, modes, (t0, tf))
        dev = check_against_oracle(ev, modes, nev, nmodes, t, tags, event_data, rng)
        if dev is None:
            skipped += 1
            continue
        seen.add((dev["will_truncate"], dev["will_spread"], len(dev["t"]) == 0))
        if modes[bisect.bisect_right(ev, t[0])] != nmodes[bisect.bisect_right(nev, t[0])] and len(dev["t"]):
            seen.add("front")   # the first window modes differ and a later one matches: the front extension at t0 - 1e-4
    assert skipped < 40
    assert {(True, False, True), (True, True, False), (False, True, False), (False, False, False), "front"} <= seen, seen


@pytest.mark.parametrize("ptst", [0.0, 0.2])
def test_device_schedule_functions_match_both_restatements(ptst):
    """300 cycles 0.05 s apart from a cold walking start: the seed, then every cycle getModeSchedule(t0 - T, tf + T) and (one cycle in four,
    seeded) a random gait command through updateGaitSchedule -- the device functions, references.GaitSchedule and the C++ GaitSchedule hold
    identical event times and modes after every step"""
    model = model_loader.load_packaged_model()
    desc, names = abi.builder_desc(model)
    usable = [g for g in names if desc.gait_n_modes[names.index(g)] > 0]
    tmpl = lambda g: ([R.MODE_NAMES[m] for m in model["gaits"][g]["modeSequence"]], model["gaits"][g]["switchingTimes"])
    rng = np.random.default_rng(11)
    T = 1.1
    dev = emu.EmuGaitState(desc)
    dev.seed(names.index("walk"), 0.0, 0.0, T)
    py, cpp = R.GaitSchedule(phase_transition_stance_time=ptst), host_lib.HostGaitSchedule(ptst)
    for gs in (py, cpp):
        gs.insert_template(*tmpl("walk"), 0.0, 2 * T)
    last, changes = "walk", 0
    for c in range(300):
        t0 = 0.05 * c
        a = py.get_mode_schedule(t0 - T, t0 + 2 * T)
        b = cpp.get_mode_schedule(t0 - T, t0 + 2 * T)
        d = dev.state() if c == 0 else dev.get_mode_schedule(t0 - T, t0 + 2 * T)   # cycle 0: the seed is the first window
        assert d == b == (list(a.event_times), list(a.mode_sequence)), c
        if rng.random() < 0.25:
            g = usable[rng.integers(len(usable))]
            if g != last:
                py.update_gait(*tmpl(g), t0, t0 + T)
                cpp.update_gait(*tmpl(g), t0, t0 + T)
                assert dev.update_gait(names.index(g), t0, t0 + T, ptst) == 0
                last, changes = g, changes + 1
        assert dev.state() == cpp.state(), c
    assert changes > 30
