"""Per-instance resets of the device builder on the CPU harness (tests/emu/bld_emu.cu): the automatic predicate over synthetic rows and
statuses, the episode books and row replacement of builder_reset_kernel, and the warm grid pass with some instances flagged for a reset --
flagged instances equal a cold pass at the reset time (and the host restatement), the others equal the same warm pass without flags, bit for
bit."""
import numpy as np
import pytest

import bld_emu_lib as E
from wb_humanoid_mpc_b200 import abi, model_loader, references as R

NX, CNX = 58, 35
HORIZON, DT = 1.0, 1.0 / 64


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


def rows(n, cen):
    ref = np.zeros(n)
    ref[8 if cen else 2] = 0.75
    return ref


@pytest.mark.parametrize("cen", [False, True])
def test_each_reason_on_its_own(cen):
    n = CNX if cen else NX
    ref = rows(n, cen)
    h = 8 if cen else 2
    bounds = (0.15, 0.5, 0.4)
    assert E.reset_reason(ref, ref, max_dev=bounds, cen=cen) == 0
    assert E.reset_reason(ref, ref, requested=True, on=False, cen=cen) == 1
    assert E.reset_reason(ref, ref, on=False, on_solve=True, solve=1, cen=cen) == 0   # auto off: only requests
    x = ref.copy()
    x[n - 1] = np.nan
    assert E.reset_reason(x, ref, cen=cen) == 2
    x[n - 1] = np.inf
    assert E.reset_reason(x, ref, cen=cen) == 2
    assert E.reset_reason(ref, ref, on_solve=True, solve=2, cen=cen) == 3   # (whole-body status 2 counts)
    assert E.reset_reason(ref, ref, on_solve=False, solve=1, cen=cen) == 0
    assert E.reset_reason(ref, ref, on_rollout=True, rollout=2, cen=cen) == 4
    assert E.reset_reason(ref, ref, on_rollout=False, rollout=2, cen=cen) == 0
    for k, why in enumerate((5, 6, 7)):
        x = ref.copy()
        x[[h, h + 2, h + 3][k]] += 1.01 * bounds[k]
        assert E.reset_reason(x, ref, max_dev=bounds, cen=cen) == why
        x[[h, h + 2, h + 3][k]] = ref[[h, h + 2, h + 3][k]] - 1.01 * bounds[k]
        assert E.reset_reason(x, ref, max_dev=bounds, cen=cen) == why
        x[[h, h + 2, h + 3][k]] = ref[[h, h + 2, h + 3][k]] + 0.99 * bounds[k]
        assert E.reset_reason(x, ref, max_dev=bounds, cen=cen) == 0
        off = list(bounds)
        off[k] = 0.0   # a bound of 0 switches that test off
        x[[h, h + 2, h + 3][k]] += 10.0
        assert E.reset_reason(x, ref, max_dev=off, cen=cen) == 0


@pytest.mark.parametrize("cen", [False, True])
def test_indices_follow_the_family(cen):
    """the whole-body test reads x[2], x[4], x[5]; the centroidal one x[8], x[10], x[11]: a deviation in the other family's slots is ignored"""
    n = CNX if cen else NX
    ref = np.zeros(n)
    for j, why in zip((8, 10, 11) if cen else (2, 4, 5), (5, 6, 7)):
        x = ref.copy()
        x[j] = 1.0
        assert E.reset_reason(x, ref, max_dev=(0.5, 0.5, 0.5), cen=cen) == why
    for j in (2, 4, 5) if cen else (8, 10, 11):
        x = ref.copy()
        x[j] = 1.0
        assert E.reset_reason(x, ref, max_dev=(0.5, 0.5, 0.5), cen=cen) == 0


def test_precedence_is_the_order_of_the_reasons():
    ref = rows(NX, False)
    x = ref.copy()
    x[2] += 1.0
    x[4] += 1.0
    x[5] += 1.0
    kw = dict(on_solve=True, on_rollout=True, max_dev=(0.1, 0.1, 0.1), solve=1, rollout=2)
    assert E.reset_reason(x, ref, requested=True, **kw) == 1
    assert E.reset_reason(x, ref, **kw) == 3
    assert E.reset_reason(x, ref, **{**kw, "solve": 0}) == 4
    assert E.reset_reason(x, ref, **{**kw, "solve": 0, "rollout": 0}) == 5
    assert E.reset_reason(x, ref, **{**kw, "solve": 0, "rollout": 0, "max_dev": (0, 0.1, 0.1)}) == 6
    assert E.reset_reason(x, ref, **{**kw, "solve": 0, "rollout": 0, "max_dev": (0, 0, 0.1)}) == 7
    x[0] = np.nan
    assert E.reset_reason(x, ref, **kw) == 2
    assert E.reset_reason(x, ref, requested=True, **kw) == 1


def test_reset_kernel_replaces_rows_and_keeps_the_books():
    B = 6
    rng = np.random.default_rng(3)
    reset = rng.normal(size=(B, NX))
    books = E.new_books(B)
    x0 = rng.normal(size=(B, NX))
    E.reset_instances(x0, reset, books, warm=False, t0=0.25)   # a cold build: episode 0 at t0, nothing replaced
    assert books["episode"].tolist() == [0] * B and books["start"].tolist() == [0.25] * B and not books["rst"].any()
    x0[:, 2] = reset[:, 2]
    x0[3, 2] += 1.0   # height of instance 3
    before, sim = x0.copy(), rng.normal(size=(B, NX))
    sim0 = sim.copy()
    slot = np.array([5, 4, 3, 2, 1, 0])   # the last solve's slot order: its statuses are read per slot
    status = np.zeros(B, int)
    status[slot.tolist().index(1)] = 1   # instance 1 failed its solve
    req = np.zeros(B, np.uint8)
    req[4] = 1
    E.reset_instances(x0, reset, books, t0=1.0, on=True, on_solve=True, max_dev=(0.5, 0, 0), req=req, status=status, slot_inst=slot, sim_x=sim)
    want = {1: 3, 3: 5, 4: 1}
    assert books["reason"].tolist() == [want.get(i, 0) for i in range(B)]
    assert books["rst"].tolist() == [int(i in want) for i in range(B)]
    assert books["episode"].tolist() == [int(i in want) for i in range(B)]
    assert books["start"].tolist() == [1.0 if i in want else 0.25 for i in range(B)]
    assert books["last_length"].tolist() == [0.75 if i in want else 0.0 for i in range(B)]
    for i in range(B):
        assert np.array_equal(x0[i], reset[i] if i in want else before[i])
        assert np.array_equal(sim[i], reset[i] if i in want else sim0[i])
    # the next build without triggers: books stay, flags clear
    E.reset_instances(x0, reset, books, t0=1.5, on=True, max_dev=(0.5, 0, 0))
    assert not books["rst"].any() and not books["reason"].any() and books["episode"].tolist() == [int(i in want) for i in range(B)]


def _inputs(model, B, rng):
    x0 = np.tile(np.array(model["x_init"], float), (B, 1))
    x0[:, 2] = model["reference"]["defaultBaseHeight"]
    x0[:, :2] += rng.uniform(-0.05, 0.05, (B, 2))
    cmd = np.zeros((B, 4))
    cmd[:, 0] = rng.uniform(0.0, 0.4, B)
    cmd[:, 2] = 0.8
    return x0, cmd


@pytest.mark.parametrize("manager", [False, True])
def test_flagged_instances_restart_cold_and_the_others_are_untouched(model, manager):
    rng = np.random.default_rng(11 if manager else 7)
    B = 8
    names = abi.builder_desc(model)[1]
    md = abi.motion_desc(model, names, 0.0) if manager else None
    a = E.EmuBuilder(model, B, HORIZON, stateful=True, motion=md, reset=dict(on=False))   # (requested resets only)
    b = E.EmuBuilder(model, B, HORIZON, stateful=True, motion=md)
    x0, cmd = _inputs(model, B, rng)
    gaits = ["walk" if i % 2 else "stance" for i in range(B)]
    starts = rng.uniform(0.0, 0.5, B)
    for g in (a, b):
        g.build(0.0, x0, cmd, gaits, starts, warm=False)
    for c in range(1, 12):
        for g in (a, b):
            g.build(c * DT, x0, cmd, gaits, starts)
    t0 = 12 * DT
    flag = np.isin(np.arange(B), [0, 3, 6]).astype(np.uint8)
    rs_gaits = ["walk" if i % 3 else "trot" for i in range(B)]
    rs_off = rng.uniform(-0.4, 0.5, B)
    rs_x0, _ = _inputs(model, B, rng)
    xa = np.where(flag[:, None] == 1, rs_x0, x0)   # builder_reset_kernel has replaced the flagged rows
    a.set_reset_states(rs_x0, rs_gaits, rs_off)
    oa = a.build(t0, x0, cmd, gaits, starts, requests=flag)
    ob = b.build(t0, x0, cmd, gaits, starts)
    fresh = E.EmuBuilder(model, B, HORIZON, stateful=True, motion=abi.motion_desc(model, names, t0) if manager else None)   # a cold pass with every clock at t0
    oc = fresh.build(t0, rs_x0, cmd, rs_gaits, t0 + rs_off, warm=False)
    for i in range(B):
        src = oc if flag[i] else ob
        assert oa["schedules"][i] == src["schedules"][i] and oa["grids"][i] == src["grids"][i], i
        assert np.array_equal(oa["tt_time"][i], src["tt_time"][i]) and np.array_equal(oa["tt_state"][i], src["tt_state"][i]), i
        if flag[i]:
            assert oa["spr_len"][i] == 0
            host = R.build_instance(model, rs_x0[i], t0=t0, horizon=HORIZON, gait=rs_gaits[i], gait_start=t0 + rs_off[i], cmd=list(cmd[i]),
                                    episode_start=t0)
            assert np.max(np.abs(np.array(oa["grids"][i]) - host["t_nodes"])) <= 1e-12
            assert oa["schedules"][i][1] == host["mode_schedule"].mode_sequence
            assert np.max(np.abs(np.array(oa["schedules"][i][0]) - host["mode_schedule"].event_times)) <= 1e-12
        else:
            assert oa["spr_len"][i] == ob["spr_len"][i]
        if manager:
            if flag[i]:   # a fresh manager at the reset time: the row of the reset gait, lastChange = origin = t0, filter gain 0
                assert abi.MOTION_GAITS[oa["state"][i]] == rs_gaits[i]
                assert oa["last_change"][i] == t0 and oa["origin"][i] == t0 and not oa["filtered"][i].any()
            else:
                for k in ("state", "last_change", "origin", "filtered"):
                    assert np.array_equal(oa[k][i], ob[k][i]), k
                assert oa["origin"][i] == 0.0
    # one pass later the reset instances run warm again from their new episode, with the filter counting from the reset
    oa2 = a.build(t0 + DT, xa, cmd, gaits, starts)
    if manager:
        d = DT
        alpha = d / (d + 1 / (2 * np.pi * 5.0))
        scaled = np.clip(cmd, [-1, -1, 0.2, -1], [1, 1, 1, 1]) * [md.max_velocity_x, md.max_velocity_y, 1.0, md.max_rotation_velocity]
        for i in np.flatnonzero(flag):
            assert np.allclose(oa2["filtered"][i], alpha * scaled[i], rtol=0, atol=1e-15)
