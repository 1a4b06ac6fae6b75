"""The time-grid edges of tests/grid_edges.py through the C ABI on the GPU, for both OCP families (tests/test_emu_grid_edges.py runs the
builder part on the CPU harness):

- all recipes of a family in one fleet build (their node counts differ, so the fleet regroups them; 17 copies of one recipe make a group
  above the cluster limit, so that group's K2 runs the two-kernel Riccati): every instance's device build equals the host build, and every
  instance's solve equals its alone-solve at the tolerances of tests/test_gpu_batch_paths.py;
- every recipe alone against the oracle (with the measured exceptions SUB_DT_CONDITIONING and PIVOT_TIES): raw LQ blocks 1e-9 relative, the accepted step bit for bit, step type and convergence code, log fields,
  x, u and K at the family tolerances of tests/test_gpu_wb.py (flight and single-support gaits) and tests/test_gpu_cen_ocp.py, one SQP iteration
  for every recipe and three for those with a sub-dt stage or an event on t0 / tf; the accepted step satisfies the linearised dynamics and
  projected constraints on every stage, the sub-dt and event stages included;
- on the recipes with a stage of about dtMin, the QP split from the LQ: the GPU's and the oracle's step and gains against the np.longdouble
  Riccati of their own stage blocks (1e-10), and the two extended-precision solutions against each other (printed: the sensitivity of the QP
  to the rounding of its blocks);
- the MRT joint actions and the policy roll-out at an event, weakEpsilon to either side of it and inside a sub-dt stage;
- gait.info's "skip" template is refused by b200sqp_set_builder and by b200sqp_build_instances."""
import ctypes as C
import time

import numpy as np
import pytest

import grid_edges as ge
import mrt_ref
import oracle_lib as orc
import rollout_ref
from test_gpu_batch_paths import cluster_limit, compare_first_iteration
from wb_humanoid_mpc_b200 import abi, references
from wb_humanoid_mpc_b200.lib import B200SqpError

pytestmark = pytest.mark.gpu
FAMILIES = ("wb", "cen")
KEYS = ["A", "B", "b", "Q", "S", "R", "q", "r", "C", "D", "e"]
INST_KEYS = ["x0", "x_init", "u_init", "t_nodes", "node_event", "contact_flags", "swing_ref", "impact_factor", "arm_phase", "x_ref"]
INT_KEYS = ["node_event", "contact_flags"]
# (x, u, K, log fields) relative tolerances: the whole-body values of test_flight_and_single_support_gaits_match_oracle (the recipes run flight and
# one-leg gaits), the centroidal ones of test_gpu_cen_ocp.test_sqp_matches_oracle
TOL = {"wb": (1e-7, 1e-6, 1e-5, 1e-7), "cen": (1e-6, 1e-6, 1e-5, 1e-6)}
THREE_ITERATIONS = ("short_stage_before_event", "short_stage_after_event", "gap_dtmin_plus_ulp", "event_at_t0", "event_at_tf")
# Whole-body recipes whose QP is ill-conditioned at the sub-dt stage.  test_sub_dt_qp_split_against_extended_precision measured on an H100:
# the GPU's and the oracle's Riccati each solve their own projected blocks to 1.1e-12 of the np.longdouble recursion (riccati_ref), and the
# blocks agree to 6e-15, but the exact QP solutions of the two block sets differ by 8.4e-5 (du) and 3.7e-4 (K) on the walk recipe: the
# rounding of the blocks alone moves the exact solution that far (the Armijo metric, which follows the LU's particular solution, differs by
# 0.2 there).  Over three iterations the measured differences to the oracle are x 5.0e-7, u 2.4e-4, K 5.0e-4, the step norm |du| (log field
# 11) 4.2e-5, and from the second iteration on the merit, cost and constraint terms that follow the iterate (fields 0, 1, 4, 5, 7) 3.5e-4.
# These recipes get about twice the measured values for those quantities; every other log field, the step sizes, step types and convergence
# codes keep the family's tolerances.
SUB_DT_CONDITIONING = {"wb-short_stage_before_event-walk", "wb-short_stage_before_event-right_leg"}
CONDITIONING_TOL = dict(x=1e-6, u=5e-4, K=1e-3, log={11: 1e-4, 0: 1e-3, 1: 1e-3, 4: 1e-3, 5: 1e-3, 7: 1e-3})
# Whole-body recipes where the complete-pivoting LU resolves exact pivot ties the other way (the PIVOT_TIES treatment of
# test_gpu_penalty_branches.py): on fast_run with an event one ulp before a node the Armijo metric, which follows the particular solution, was
# measured 2.5e-2 apart on the first iteration and the merit and cost after the step (log fields 4, 5) 1.9e-7 apart; those two fields get 1e-6.
PIVOT_TIES = {"wb-event_ulp_before_node-fast_run": {4: 1e-6, 5: 1e-6}}
COPIES = 17   # copies of one recipe in the fleet: one group above the cluster limit of an H100 (132 SMs // 8 = 16)
_ORACLE, _INST = {}, {}


def rel(a, b):
    return np.max(np.abs(a - b)) / max(1e-9, np.max(np.abs(b))) if b.size else 0.0


def is_cen(model):
    return model.get("kind") == "centroidal"


@pytest.fixture(scope="module")
def models():
    return {f: ge.load_model(f) for f in FAMILIES}


@pytest.fixture(scope="module")
def built(models):
    return {f: ge.recipes(f, models[f]) for f in FAMILIES}


def cmd_of(model, i):
    return [0.3 - 0.05 * (i % 3), 0.05 * ((i % 5) - 2), model["reference"]["defaultBaseHeight"], 0.1 * ((i % 4) - 1.5)]


def instance(model, family, i, r):
    """recipe r as a host-built instance (cached: the oracle solves key on it)"""
    key = (family, i)
    if key not in _INST:
        _INST[key] = ge.build_host(model, r, ge.x0_of(model, np.random.default_rng(300 + i)), cmd=cmd_of(model, i))
    return _INST[key]


def oracle(model, family, i, inst, iters):
    key = (family, i, iters)
    if key not in _ORACLE:
        o = orc.CenOracle(model) if is_cen(model) else orc.WbOracle(model)
        o.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
        st = abi.default_settings(model, sqp_iteration=iters, use_feedback_policy=1)
        t = time.perf_counter()
        res = o.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], st, keep_raw=iters == 1)
        res["seconds"] = time.perf_counter() - t
        if iters == 1:
            res["raw"] = o.last_raw_blocks(len(inst["t_nodes"]))
        _ORACLE[key] = res
    return _ORACLE[key]


def new_solver(model, iters, raw=False):
    from wb_humanoid_mpc_b200.solver import B200SqpSolver

    return B200SqpSolver(model, abi.default_settings(model, sqp_iteration=iters, use_feedback_policy=1), capture_raw_blocks=raw)


@pytest.mark.parametrize("family", FAMILIES)
def test_all_recipes_in_one_fleet(models, built, family):
    """one fleet build of every recipe and 17 more instances of one sub-dt recipe: device build = host build, and each instance's one-iteration
    solve equals its alone-solve (B = 1, cluster kernel) on the same uploaded arrays: step, step type and convergence code exactly, the rest
    1e-9 relative (the two-kernel Riccati adds reg_prim in another order)"""
    from test_gpu_fleet import fleet_of

    model = models[family]
    recs = [r for r, _ in built[family]]
    sub = next(r for r in recs if r["branch"] == "short_stage_before_event")
    recs = recs + [sub] * COPIES
    B = len(recs)
    rng = np.random.default_rng(17)
    x0s = np.array([ge.x0_of(model, rng) for _ in range(B)])
    cmds = np.array([cmd_of(model, b) for b in range(B)])
    s = new_solver(model, 1)
    fl = fleet_of(s)
    n = fl.build_instances(ge.T0, recs[0]["horizon"], x0s, [r["gait"] for r in recs], [r["gait_start"] for r in recs], cmds)
    dev = fl.download_instances()
    counts = {int(v): int((n == v).sum()) for v in np.unique(n)}
    assert len(counts) >= 3 and max(counts.values()) > cluster_limit(), counts
    for b, r in enumerate(recs):
        kw = dict(base_vel=np.zeros(6)) if is_cen(model) else {}
        h = references.build_instance(model, x0s[b], t0=ge.T0, horizon=r["horizon"], gait=r["gait"], gait_start=r["gait_start"], cmd=list(cmds[b]), **kw)
        assert n[b] == len(h["t_nodes"]), (ge.name(r), n[b], len(h["t_nodes"]))
        m = n[b]
        for k in INST_KEYS:
            d = dev[k][b] if k == "x0" else dev[k][b][: m - 1] if k == "u_init" else dev[k][b][:m]
            if k in INT_KEYS:
                assert np.array_equal(d, h[k]), (ge.name(r), k)
            else:
                assert np.max(np.abs(d - h[k])) <= 1e-12 * max(1.0, np.max(np.abs(h[k]))), (ge.name(r), k)
    fl.solve()
    sol = fl.primal_solution()
    assert not sol["status"].any()
    alone = new_solver(model, 1)
    worst = dict(log=0.0, x=0.0, u=0.0, K=0.0)
    for b in range(B):
        m = n[b]
        inst = {k: (dev[k][b] if k == "x0" else dev[k][b][: m - 1] if k == "u_init" else dev[k][b][:m]) for k in INST_KEYS}
        o = alone.run([inst])
        one = {k: sol[k][b: b + 1] for k in ("log", "n_iter", "status")}
        one.update(x=sol["x"][b: b + 1, :m], u=sol["u"][b: b + 1, : m - 1], K=sol["K"][b: b + 1, : m - 1])
        w = compare_first_iteration(one, [o], 1e-9)
        worst = {k: max(worst[k], w[k]) for k in worst}
    print(f"{family}: fleet groups {counts}; largest relative differences to the alone-solves {worst}")
    if is_cen(model):
        return
    # the group above the cluster limit, solved again in a plain handle: one more launch per SQP iteration than a one-kernel K2 (the
    # two-kernel Riccati ran), and bit for bit the fleet's solve of those instances
    from test_gpu_batch_paths import assert_k2_path
    from test_gpu_fleet import KEYS as FLEET_KEYS, per_group_plain

    big = max(counts, key=counts.get)
    idx, plain = per_group_plain(model, fl, dev, iters=1, use_feedback_policy=1)[big]
    assert len(idx) > cluster_limit() and FLEET_KEYS == INST_KEYS
    assert_k2_path(plain, model, plain.settings, True)
    ref = plain.primal_solution()
    assert np.array_equal(sol["x"][idx][:, :big], ref["x"]) and np.array_equal(sol["u"][idx][:, : big - 1], ref["u"])
    assert np.array_equal(sol["K"][idx][:, : big - 1], ref["K"]) and np.array_equal(sol["log"][idx], ref["log"])


@pytest.mark.parametrize("family", FAMILIES)
def test_every_recipe_alone_matches_the_oracle(models, built, family):
    model = models[family]
    tx, tu, tk, tl = TOL[family]
    worst = dict(blocks=0.0, x=0.0, u=0.0, K=0.0, log=0.0)
    misses = []   # every recipe runs before the outputs are judged, so that a failure reports all recipes that miss
    t_oracle = 0.0
    for i, (r, _) in enumerate(built[family]):
        inst = instance(model, family, i, r)
        n = len(inst["t_nodes"])
        for iters in (1, 3) if r["branch"] in THREE_ITERATIONS else (1,):
            s = new_solver(model, iters, raw=iters == 1)
            sol = s.run([inst])
            ref = oracle(model, family, i, inst, iters)
            t_oracle += ref["seconds"]
            what = (ge.name(r), iters)
            name = ge.name(r)
            log_tol = dict(CONDITIONING_TOL["log"]) if name in SUB_DT_CONDITIONING else {}
            log_tol.update(PIVOT_TIES.get(name, {}))
            assert not sol["status"].any(), what
            nit = len(ref["log"])
            assert sol["n_iter"][0] == nit, what
            for it in range(nit):
                g, o = sol["log"][0, it], ref["log"][it]
                assert g[8] == o[8], (what, it, "step", g[8], o[8])
                assert int(g[9]) == int(o[9]) and int(g[13]) == int(o[13]), (what, it)
                for j in (0, 1, 2, 3, 4, 5, 6, 7, 10, 11):
                    d = abs(g[j] - o[j]) / max(1.0, abs(o[j]))
                    worst["log"] = max(worst["log"], d)
                    if d > log_tol.get(j, tl):
                        misses.append((what, it, "log", j, d))
                # the Armijo metric depends on the particular solution of the pivoting LU (test_gpu_wb.py): its sign
                assert np.sign(g[12]) == np.sign(o[12]), (what, it)
            for key, tol in (("x", tx), ("u", tu), ("K", tk)):
                d = rel(sol[key][0], ref[key])
                worst[key] = max(worst[key], d)
                if d >= (CONDITIONING_TOL[key] if name in SUB_DT_CONDITIONING else tol):
                    misses.append((what, key, d))
            if iters != 1:
                continue
            raw = s.raw_stage_blocks()
            nx = model["nx"]
            alpha = sol["log"][0, 0, 8]
            assert alpha > 0
            dx = (sol["x"][0] - inst["x_init"]) / alpha
            du = (sol["u"][0] - inst["u_init"]) / alpha
            assert np.allclose(dx[0], inst["x0"] - inst["x_init"][0], atol=1e-9), what
            for k in range(n - 1):
                g, o = orc.unpack_raw_blocks(raw[0, k], nx, model["nu"]), ref["raw"][k]
                assert g["nc"] == o["nc"], (what, k)
                for key in KEYS:
                    d = rel(g[key], o[key])
                    worst["blocks"] = max(worst["blocks"], d)
                    assert d < 1e-9, (what, k, key, d)
                # the accepted step satisfies the linearised dynamics and the projected constraints of every stage
                if inst["node_event"][k] == 1:
                    assert np.max(np.abs(dx[k] + g["b"] - dx[k + 1])) < 1e-8, (what, k)
                    continue
                assert np.max(np.abs(g["A"] @ dx[k] + g["B"] @ du[k] + g["b"] - dx[k + 1])) < 1e-7, (what, k)
                assert np.max(np.abs(g["C"] @ dx[k] + g["D"] @ du[k] + g["e"])) < 1e-6, (what, k)
    print(f"{family}: largest relative differences to the oracle {worst}; oracle solves {t_oracle:.1f} s")
    for m in misses:
        print("miss", *m)
    assert not misses, f"{len(misses)} misses (printed)"


def policy_times(inst):
    """an event, weakEpsilon before and after it, and the middle of the sub-dt stage that ends at it"""
    k = ge.sub_dt_stages(inst)[0]
    t = inst["t_nodes"]
    te = float(t[k + 1])
    return [te, te - ge.WEAK_EPS, te + ge.WEAK_EPS, 0.5 * (float(t[k]) + te)]


@pytest.mark.parametrize("family", FAMILIES)
def test_policy_at_the_grid_edges(models, built, family):
    """b200sqp_joint_actions against mrt_ref.joint_action and (whole-body) b200sqp_rollout_policy against rollout_ref.rollout_policy, after a
    solve of each recipe that ends a sub-dt stage at an event"""
    model = models[family]
    wb = orc.WbOracle(ge.load_model("wb"))
    rng = np.random.default_rng(8)
    for i, (r, _) in enumerate(built[family]):
        if r["branch"] != "short_stage_before_event":
            continue
        inst = instance(model, family, i, r)
        s = new_solver(model, 1)
        sol = s.run([inst])
        plan = dict(t_nodes=inst["t_nodes"], node_event=inst["node_event"], contact_flags=inst["contact_flags"], x=sol["x"][0], u=sol["u"][0])
        K = sol["K"][0]
        for t in policy_times(inst):
            base = np.array([mrt_ref.interpolate(t, plan["t_nodes"], plan["x"])])
            rs = mrt_ref.random_robot_states(rng, 1, model["nj"], base=base[:, 6:] if is_cen(model) else base)
            dev = s.joint_actions(t, rs)
            ref = mrt_ref.joint_action(model, wb, t, robot_state=rs[0], plan=plan, K=K)
            what = (ge.name(r), t)
            assert np.max(np.abs(dev["x"][0] - ref["x"])) < 1e-12, what
            for k in ("q_des", "qd_des", "u"):
                d = float(np.max(np.abs(dev[k][0] - ref[k])) / max(1e-300, np.max(np.abs(ref[k]))))
                assert d < 1e-12 or (not np.any(dev[k][0]) and not np.any(ref[k])), (what, k, d)
            assert np.max(np.abs(dev["tau"][0] - ref["tau"])) < 1e-9 * max(1.0, np.abs(ref["tau"]).max()), what
            assert dev["mode"][0] == ref["mode"], what
            if is_cen(model):
                continue
            i0, a = rollout_ref.time_segment(t, list(plan["t_nodes"]))
            xs = (a * plan["x"][i0] + (1 - a) * plan["x"][i0 + 1])[None].copy()
            xs[:, 29:35] += rng.normal(0.0, 0.2, (1, 6))
            dr = s.rollout_policy(t, 1.0 / 80.0, x_start=xs)
            rr = rollout_ref.rollout_policy(wb.flow_map, plan, t, 1.0 / 80.0, xs[0], K=K)
            assert dr["status"][0] == rr["status"] == 0, what
            assert tuple(dr["n_steps"][0]) == (rr["accepted"], rr["rejected"], rr["calls"]), what
            assert dr["mode"][0] == rr["mode"], what
            for k in ("x", "u"):
                d = float(np.max(np.abs(dr[k][0] - rr[k])) / max(1e-300, np.max(np.abs(rr[k]))))
                assert d < 1e-12, (what, k, d)


def test_skip_is_refused(models):
    """a builder table that holds gait.info's skip template (switching times 0.75 -> 0.08) is refused, and so is a build that names the skip
    entry of the packaged table (left out: no modes)"""
    from wb_humanoid_mpc_b200 import lib as L

    model = models["wb"]
    s = new_solver(model, 1)
    desc, names = abi.builder_desc(model)
    g = names.index("skip")
    tmpl = model["gaits"]["skip"]
    desc.gait_n_modes[g] = len(tmpl["modeSequence"])
    for j, m in enumerate(tmpl["modeSequence"]):
        desc.gait_modes[g][j] = references.MODE_NAMES[m]
    for j, t in enumerate(tmpl["switchingTimes"]):
        desc.gait_switching_times[g][j] = float(t)
    assert L.lib().b200sqp_set_builder(s._h, C.byref(desc)) == L.EINVAL
    x0 = ge.x0_of(model, np.random.default_rng(1))[None]
    with pytest.raises(B200SqpError) as e:
        s.build_instances(0.0, 1.1, x0, ["skip"], [0.0], [cmd_of(model, 0)])
    assert e.value.code == L.EINVAL and "gait table" in str(e.value)


@pytest.mark.parametrize("family", FAMILIES)
def test_sub_dt_qp_split_against_extended_precision(models, built, family):
    """the QP half and the LQ half of the solve on every recipe with a stage of about dtMin, first SQP iteration: the GPU's step and gains
    against the np.longdouble Riccati (test_gpu_qp_shapes.riccati_ref) of the GPU's own captured stage blocks, projected with the oracle's LU;
    the same for the oracle's; and the two extended-precision solutions against each other, which measures how far the difference between
    the GPU's and the oracle's blocks moves the exact solution of the QP."""
    from test_gpu_qp_shapes import riccati_ref

    model = models[family]
    st = abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1)
    nx, nu = model["nx"], model["nu"]
    out = []
    for i, (r, _) in enumerate(built[family]):
        inst = instance(model, family, i, r)
        if not ge.sub_dt_stages(inst):
            continue
        n = len(inst["t_nodes"])
        s = new_solver(model, 1, raw=True)
        sol = s.run([inst])
        graw = [orc.unpack_raw_blocks(v, nx, nu) for v in s.raw_stage_blocks()[0]]
        o = orc.CenOracle(model) if is_cen(model) else orc.WbOracle(model)
        o.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
        res = o.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], st, keep_raw=True)
        P, p = o.last_value_function(np.zeros_like(inst["x_init"]))
        dx0 = inst["x0"] - inst["x_init"][0]
        refs = {}
        for side, raw in (("gpu", graw), ("oracle", o.last_raw_blocks(n))):
            data, n_in, proj = ge.projected_qp(model, inst, raw, P[-1], p[-1], st.reg_prim)
            ref = riccati_ref(*data, dx0, n_in, st.reg_prim)
            assert ref is not None, (ge.name(r), side)
            refs[side] = ge.to_input_space(ref, n_in, proj, nu)
        alpha = sol["log"][0, 0, 8]
        gpu = ((sol["x"][0] - inst["x_init"]) / alpha, (sol["u"][0] - inst["u_init"]) / alpha, sol["K"][0])
        row = {"recipe": ge.name(r)}
        for key, a, b, c, d in zip(("dx", "du", "K"), gpu, refs["gpu"], (res["dx"], res["du"], res["K"]), refs["oracle"]):
            row[key] = (ge.rel_ld(a, b), ge.rel_ld(c, d), ge.rel_ld(b, d))
        out.append(row)
    for row in out:
        print("split", row["recipe"], "(GPU vs its longdouble, oracle vs its longdouble, longdouble GPU blocks vs oracle blocks):",
              {k: tuple(f"{v:.1e}" for v in row[k]) for k in ("dx", "du", "K")})
    assert len(out) >= 3
    for row in out:
        for key in ("dx", "du", "K"):
            assert row[key][0] < 1e-10 and row[key][1] < 1e-10, (row["recipe"], key, row[key])
