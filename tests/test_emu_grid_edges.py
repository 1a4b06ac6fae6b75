"""The time grid at its edges, without a GPU: the recipes of tests/grid_edges.py put gait events exactly on an accumulated grid node or one ulp
to either side of it, at dtMin - ulp / dtMin / dtMin + ulp past the last node (the replace-or-keep test of timeDiscretizationWithEvents), 1.1 dtMin
before an event or after the last one (a stage about 3,500 times shorter than dt), at t0, at tf and within dtMin of tf, and two events less
than one grid step apart.  For both OCP families:

- the device builder (bldGridInstance and the node pass of wb_builder.cuh, on the CPU harness) equals the host restatement
  (references.build_instance) on every recipe and on all 14 templates of the device gait table: integer arrays exactly, floating-point arrays
  to 1e-12, cold and warm from a previous solution whose grid holds the sub-dt stage and a PreEvent/PostEvent pair;
- gait.info's "skip" template stays out of the device table;
- the K1 node blocks of the harness (all whole-body K1b schedules, the centroidal node) equal the oracle's raw blocks on the sub-dt stages and
  their neighbours, at each node's own interval duration.

tests/test_gpu_grid_edges.py runs the same recipes through the C ABI on the GPU."""
import numpy as np
import pytest

import bld_emu_lib
import emu_lib as emu
import grid_edges as ge
import oracle_lib as orc
from wb_humanoid_mpc_b200 import abi, references
from wb_humanoid_mpc_b200.solver import stack_instances

FLOAT_KEYS = ["x0", "x_init", "u_init", "t_nodes", "swing_ref", "impact_factor", "arm_phase", "x_ref"]
INT_KEYS = ["node_event", "contact_flags"]
KEYS = ["A", "B", "b", "Q", "S", "R", "q", "r", "C", "D", "e"]
FAMILIES = ("wb", "cen")


@pytest.fixture(scope="module", params=FAMILIES)
def family(request):
    return request.param


@pytest.fixture(scope="module")
def models():
    return {f: ge.load_model(f) for f in FAMILIES}


@pytest.fixture(scope="module")
def built(models):
    return {f: ge.recipes(f, models[f]) for f in FAMILIES}


def is_cen(model):
    return model.get("kind") == "centroidal"


def host_base_velocity(model, x):
    """Ab^-1 hbar of the centroidal state x: the oracle's flow map at u = 0 over the total mass"""
    return orc.CenOracle(model).flow_map(x, np.zeros(model["nu"]))[6:12] / sum(model["mass"])


def compare(dev, host_insts, what):
    ref = stack_instances(host_insts)
    assert dev["t_nodes"].shape == ref["t_nodes"].shape, (what, dev["t_nodes"].shape, ref["t_nodes"].shape)
    for k in INT_KEYS:
        assert np.array_equal(dev[k], ref[k]), (what, k)
    for k in FLOAT_KEYS:
        err = np.max(np.abs(dev[k] - ref[k]))
        assert err <= 1e-12 * max(1.0, np.max(np.abs(ref[k]))), (what, k, err)


def device_build(model, t0, horizon, x0s, gaits, starts, cmds, previous=None):
    r = bld_emu_lib.build_instances(model, t0, horizon, x0s, gaits, starts, cmds, previous=previous)
    assert not isinstance(r, int), r
    if not is_cen(model):
        return r, None
    dev, bv, padding = r
    assert padding == {"x_init": 0.0, "x_ref": 0.0}
    return dev, bv


def host_builds(model, x0s, cmds, t0, horizon, gait, start, prevs=None):
    out = []
    for b in range(len(x0s)):
        kw = dict(base_vel=host_base_velocity(model, x0s[b])) if is_cen(model) else {}
        # the host's "stance" is the default schedule (stance phases from 0.5), the device's the stance template tiled from gait_start = 0.5
        out.append(references.build_instance(model, x0s[b], t0=t0, horizon=horizon, gait=gait, gait_start=None if gait == "stance" else start, cmd=list(cmds[b]),
                                             previous=None if prevs is None else prevs[b], **kw))
    return out


def check_cold_and_warm(model, family, gait, start, t0, horizon, seed, warm_shifts, what):
    """cold build of two instances against the host, then warm builds at t0 + each shift from a made-up previous solution on the cold grid
    -> the cold build"""
    rng = np.random.default_rng(seed)
    B = 2
    x0s = np.array([ge.x0_of(model, rng) for _ in range(B)])
    h = model["reference"]["defaultBaseHeight"]
    cmds = np.array([[rng.uniform(-0.5, 1.0), rng.uniform(-0.3, 0.3), h, rng.uniform(-0.5, 0.5)] for _ in range(B)])
    first, _ = device_build(model, t0, horizon, x0s, [gait] * B, [start] * B, cmds)
    compare(first, host_builds(model, x0s, cmds, t0, horizon, gait, start), (what, "cold"))
    n, nx, nu = first["t_nodes"].shape[1], model["nx"], model["nu"]
    if is_cen(model):   # near the cold initial guess, momentum included
        xs = first["x_init"] + 0.05 * rng.normal(size=(B, n, nx))
    else:
        xs = rng.normal(size=(B, n, nx))
    us = rng.normal(size=(B, n - 1, nu))
    for shift in warm_shifts:
        t1 = t0 + shift
        prevs = [references.to_primal_solution(first["t_nodes"][b], first["node_event"][b], xs[b], us[b]) for b in range(B)]
        x1 = np.array([references.linear_interpolate(t1, p["t"], p["x"]) for p in prevs])
        dev, _ = device_build(model, t1, horizon, x1, [gait] * B, [start] * B, cmds,
                              previous=dict(t=first["t_nodes"], event=first["node_event"], x=xs, u=us))
        compare(dev, host_builds(model, x1, cmds, t1, horizon, gait, start, prevs), (what, "warm", shift))
    return first


def test_every_branch_is_hit_on_both_families(models, built):
    """each recipe reaches its own branch (asserted in grid_edges.recipes); together they reach every branch of the grid on both families"""
    msgs = [ge.format_counts(f, ge.branch_counts(built[f])) for f in FAMILIES]
    print("\n".join(msgs))
    for f in FAMILIES:
        total = ge.branch_counts(built[f])
        missing = [b for b in ge.BRANCHES if total[b] == 0]
        assert not missing, (f, missing, msgs)
        # the sub-dt stage of the short-stage recipes is a real stage of the grid: about 3,500 times shorter than dt
        for r, _ in built[f]:
            if r["branch"].startswith("short_stage"):
                inst = ge.build_host(models[f], r, np.array(models[f]["x_init"], float))
                k = ge.sub_dt_stages(inst)
                assert len(k) == 1, (ge.name(r), k)
                length = inst["t_nodes"][k[0] + 1] - inst["t_nodes"][k[0]]
                assert ge.DT_MIN < length < 1.2 * ge.DT_MIN, (ge.name(r), length)


@pytest.mark.parametrize("index", range(max(len(p) for p in ge.PLAN.values())))
def test_recipe_builds_match_the_host(models, built, family, index):
    """cold, and warm from a previous solution on the recipe's own grid: one warm build 0.4 of the shortest stage later (the new grid moves
    by less than dtMin, so nodes merge and the warm start interpolates inside the sub-dt stage), one a third of dt later"""
    model = models[family]
    r, _ = built[family][index]
    dt = ge.FAMILIES[family][1]
    t = ge.build_host(model, r, np.array(model["x_init"], float))["t_nodes"]
    short = min(b - a for a, b in zip(t, t[1:]) if b > a)
    first = check_cold_and_warm(model, family, r["gait"], r["gait_start"], r["t0"], r["horizon"], 100 + index, (0.4 * short, dt / 3), ge.name(r))
    if r["branch"].startswith("short_stage"):
        assert ge.sub_dt_stages(dict(t_nodes=first["t_nodes"][0])) and (first["node_event"][0] == 1).any()


@pytest.mark.parametrize("gait", ge.DEVICE_GAITS)
def test_every_device_template_builds_like_the_host(models, family, gait):
    """all 14 templates of the device table, seven of which no other builder or parity test names, at two phases each, cold and warm"""
    model = models[family]
    horizon = ge.FAMILIES[family][2]
    dt = ge.FAMILIES[family][1]
    for j, (start, t0) in enumerate(((-0.23, 0.0125), (0.31, 0.2))):
        start = 0.5 if gait == "stance" else start
        check_cold_and_warm(model, family, gait, start, t0, horizon, 7 * j + len(gait), (dt / 3, 0.27), (family, gait, start))


def test_skip_stays_out_of_the_device_table(models):
    """gait.info's skip template has a decreasing switching time (0.75 -> 0.08): tiled, its events would not increase.  The device table leaves
    it out (no modes, so b200sqp_build_instances refuses it by name and b200sqp_set_builder refuses the template itself); every other template
    is in the table with its own modes and times."""
    for f in FAMILIES:
        model = models[f]
        desc, names = abi.builder_desc(model)
        g = model["gaits"]["skip"]
        times = g["switchingTimes"]
        assert any(b <= a for a, b in zip(times, times[1:]))
        assert desc.gait_n_modes[names.index("skip")] == 0
        for name in ge.DEVICE_GAITS + (ge.SHORT_FLIGHT,):
            i = names.index(name)
            tg = model["gaits"][name]
            assert desc.gait_n_modes[i] == len(tg["modeSequence"]), name
            assert [desc.gait_switching_times[i][j] for j in range(len(tg["switchingTimes"]))] == [float(v) for v in tg["switchingTimes"]], name
        # what the reference's GaitSchedule would make of it: an event list that goes backwards
        gs = references.GaitSchedule()
        gs.insert_template([references.MODE_NAMES[m] for m in g["modeSequence"]], times, 0.0, 2.0)
        ev = gs.ms.event_times
        assert any(b < a for a, b in zip(ev, ev[1:]))


def interval_duration(inst, k):
    """getIntervalDuration: a post-event node starts and a pre-event node ends weakEpsilon inside the interval"""
    t, ev = inst["t_nodes"], inst["node_event"]
    return (t[k + 1] - (ge.WEAK_EPS if ev[k + 1] == 1 else 0.0)) - (t[k] + (ge.WEAK_EPS if ev[k] == 2 else 0.0))


def test_node_blocks_on_sub_dt_stages_match_the_oracle(models, built, family):
    """the K1 node of the harness on every sub-dt stage of the recipes and on the stages next to it (the event's PostEvent stage included), at
    the node's own interval duration (about 1.1e-5 s): RK4 over the short step, the dt-scaled cost and the projection.  Raw blocks 1e-9 relative
    to the oracle; the whole-body node in all three K1b schedules."""
    model = models[family]
    rng = np.random.default_rng(21)
    seen = 0
    worst = {}
    for r, _ in built[family]:
        inst = ge.build_host(model, r, ge.x0_of(model, rng), cmd=[0.3, 0.05, model["reference"]["defaultBaseHeight"], 0.1])
        short = ge.sub_dt_stages(inst)
        if not short:
            continue
        inst["x_init"] = inst["x_init"] + 0.01 * rng.normal(size=inst["x_init"].shape)
        o = orc.CenOracle(model) if is_cen(model) else orc.WbOracle(model)
        inst["u_init"] = inst["u_init"] + 1.0 * rng.normal(size=inst["u_init"].shape)
        o.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
        o.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], abi.default_settings(model, sqp_iteration=1), keep_raw=True)
        raw = o.last_raw_blocks(len(inst["t_nodes"]))
        ks = sorted({j for k in short for j in (k - 2, k - 1, k, k + 1, k + 2) if 0 <= j < len(inst["t_nodes"]) - 1 and inst["node_event"][j] != 1})
        for k in ks:
            dt = interval_duration(inst, k)
            args = (inst["x_init"][k], inst["u_init"][k], inst["x_init"][k + 1], inst["x_ref"][k], dt, inst["contact_flags"][k], inst["swing_ref"][k],
                    inst["impact_factor"][k], inst["arm_phase"][k])
            outs = [emu.cen_node(o.desc, o.cdesc, *args)] if is_cen(model) else [emu.lq_node(o.desc, *args, mode=m) for m in (0, 1, 2)]
            for mode, e in enumerate(outs):
                assert e["raw"]["nc"] == raw[k]["nc"], (ge.name(r), k)
                for key in KEYS:
                    d = np.max(np.abs(e["raw"][key] - raw[k][key])) / max(1e-12, np.max(np.abs(raw[k][key]))) if raw[k][key].size else 0.0
                    worst[key] = max(worst.get(key, 0.0), d)
                    assert d < 1e-9, (ge.name(r), k, dt, mode, key, d)
                assert abs(e["raw"]["c"] - raw[k]["c"]) < 1e-9 * max(1.0, abs(raw[k]["c"])), (ge.name(r), k, mode)
            seen += k in short
    print(f"{family}: {seen} sub-dt stages; largest relative differences " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))
    assert seen >= 3


def test_oracle_qp_on_sub_dt_stages_matches_extended_precision(models, built, family):
    """the oracle's QP step and gains on the recipes with a stage of about dtMin, against the Riccati recursion in np.longdouble
    (test_gpu_qp_shapes.riccati_ref) of the oracle's own stage blocks, projected with its LU: the oracle stays accurate where the dt-scaled
    input Hessian of the short stage is nearly singular, so it is a sound yardstick for the GPU there (tests/test_gpu_grid_edges.py)"""
    from test_gpu_qp_shapes import riccati_ref

    model = models[family]
    st = abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1)
    seen = 0
    for i, (r, _) in enumerate(built[family]):
        inst = ge.build_host(model, r, ge.x0_of(model, np.random.default_rng(300 + i)), cmd=[0.3, 0.05, model["reference"]["defaultBaseHeight"], 0.1])
        if not ge.sub_dt_stages(inst):
            continue
        o = orc.CenOracle(model) if is_cen(model) else orc.WbOracle(model)
        o.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
        res = o.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], st, keep_raw=True)
        P, p = o.last_value_function(np.zeros_like(inst["x_init"]))
        data, n_in, proj = ge.projected_qp(model, inst, o.last_raw_blocks(len(inst["t_nodes"])), P[-1], p[-1], st.reg_prim)
        ref = riccati_ref(*data, inst["x0"] - inst["x_init"][0], n_in, st.reg_prim)
        assert ref is not None, ge.name(r)
        for key, got, want in zip(("dx", "du", "K"), (res["dx"], res["du"], res["K"]), ge.to_input_space(ref, n_in, proj, model["nu"])):
            d = ge.rel_ld(got, want)
            assert d < 1e-11, (ge.name(r), key, d)
        seen += 1
    assert seen >= 3
