"""The soft-constraint penalties where they act, on the GPU through the C ABI, whole-body and centroidal: the recipes of
tests/test_penalty_branches.py (foot collision and joint limits in both polynomial pieces, the knee pair alone, a flight node, the relaxed
branches of the friction cone and the contact-moment rows, exact thresholds, large base rotations) against the oracle; per-instance penalty
gains that move an instance into another branch; and the recipes inside a batch above the cluster limit against their alone-solves.

Tolerances are those of the parity tests: raw LQ blocks 1e-9 relative; accepted step bit for bit, step type and convergence code equal;
log fields, x, u 1e-7 and K 1e-6 relative (tests/test_gpu_wb.py) on the whole-body path, 1e-6 / 1e-6 / 1e-5 on the centroidal path
(tests/test_gpu_cen_ocp.py).  The Armijo metric is compared tightly on the first iteration and by sign afterwards (its value depends on the
particular solution the complete-pivoting LU picks, see test_gpu_wb.py::test_sqp_end_to_end_matches_oracle)."""
from collections import Counter

import numpy as np
import pytest

import oracle_lib as orc
from test_emu_gains import model_gains, model_with_gains
from test_gpu_batch_paths import assert_k2_path, cluster_limit, compare_first_iteration, solve_alone
from test_penalty_branches import (Geometry, _copy, base_instance, build_recipes, cross_legs, edge_moments, format_counts, is_cen,
                                   joints_at_limits, unload_feet)
from wb_humanoid_mpc_b200 import abi, model_loader

pytestmark = pytest.mark.gpu

KEYS = ["A", "B", "b", "Q", "S", "R", "q", "r", "C", "D", "e"]
LOG_J = (0, 1, 2, 3, 4, 5, 6, 7, 10, 11)


def rel(a, b):
    return np.max(np.abs(a - b)) / max(1e-9, np.max(np.abs(b))) if b.size else 0.0


@pytest.fixture(scope="module", params=["g1_wb", "g1_centroidal"])
def model(request):
    return model_loader.load_packaged_model() if request.param == "g1_wb" else model_loader.load_packaged_model(request.param)


@pytest.fixture(scope="module")
def built(model):
    return build_recipes(model, Geometry(model))


@pytest.fixture
def default_dispatch(monkeypatch):
    monkeypatch.delenv("B200SQP_NO_CLUSTER", raising=False)
    monkeypatch.delenv("B200SQP_K2_LEGACY", raising=False)


def tolerances(model, name):
    """(log, x, u, K) relative tolerances.  On the recipes of PIVOT_TIES the LU's exact pivot ties may resolve either way, which changes the
    conditioning of the projected QP (test_gpu_wb.py::test_flight_and_single_support_gaits_match_oracle allows u 1e-6 and K 1e-5 for the
    same reason); with the ankles on their limits the merit after the step was measured 1.8e-7 apart, so these recipes get the centroidal
    tolerances."""
    if is_cen(model):
        return 1e-6, 1e-6, 1e-6, 1e-5
    if name in PIVOT_TIES:   # a tie resolved the other way changes the conditioning of the projected QP: the centroidal tolerances
        return 1e-6, 1e-6, 1e-6, 1e-5
    return 1e-7, 1e-7, 1e-7, 1e-6


# Recipes where the complete-pivoting LU may pick another particular solution on each side: exact ties among the largest entries of D at
# their double-stance nodes (measured on the oracle's blocks: four equal entries with the base rotated, with the ankles on their limits, and
# in the gain probe), and the symmetric crossed legs of the flight and rotated-collision recipes (as for the symmetric gaits of
# test_gpu_wb.py::test_flight_and_single_support_gaits_match_oracle).  The Armijo metric depends on that choice
# (test_gpu_wb.py::test_sqp_end_to_end_matches_oracle) and is compared by sign there, on the first iteration too.  Every other log field, the
# accepted step, x, u and K keep their tolerances.
PIVOT_TIES = {"collision_flight", "rotated_contact", "rotated_collision", "exact_thresholds", "gain probe"}


def new_solver(model, st, **kw):
    from wb_humanoid_mpc_b200.solver import B200SqpSolver

    return B200SqpSolver(model, st, **kw)


def oracle_solve(model, inst, st, keep_raw=False):
    o = orc.CenOracle(model) if is_cen(model) else orc.WbOracle(model)
    o.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
    res = o.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], st, keep_raw=keep_raw)
    if keep_raw:
        res["raw"] = o.last_raw_blocks(len(inst["t_nodes"]))
    return res


_ORACLE = {}


def cached_oracle(model, key, inst, st, keep_raw=False):
    """one oracle solve per (family, recipe, gain set, iterations)"""
    key = (model["name"], model.get("centroidalModelType"), *key, st.sqp_iteration, keep_raw)
    if key not in _ORACLE:
        _ORACLE[key] = oracle_solve(model, inst, st, keep_raw)
    return _ORACLE[key]


def by_node_count(built):
    groups = {}
    for name, inst, _ in built:
        groups.setdefault(len(inst["t_nodes"]), []).append((name, inst))
    return groups.values()


def nx_of(model):
    return model["nx"]


def compare_blocks(model, raw_gpu, ref_raw, what, worst):
    nx = nx_of(model)
    for k in range(len(ref_raw)):
        g, o = orc.unpack_raw_blocks(raw_gpu[k], nx, 35), ref_raw[k]
        assert g["nc"] == o["nc"], (what, k)
        for key in KEYS:
            d = rel(g[key], o[key])
            worst[key] = max(worst[key], d)
            assert d < 1e-9, (what, k, key, d)


def compare_solve(model, sol, b, ref, name, worst, first_only=False, recipe=None):
    recipe = name if recipe is None else recipe
    tl, tx, tu, tk = tolerances(model, recipe)
    nit = 1 if first_only else len(ref["log"])
    if not first_only:
        assert sol["n_iter"][b] == nit, (name, sol["n_iter"][b], nit)
    for it in range(nit):
        g, o = sol["log"][b, it], ref["log"][it]
        assert g[8] == o[8], (name, "step size", it, g[8], o[8])
        assert int(g[9]) == int(o[9]) and int(g[13]) == int(o[13]), (name, it, g[9], o[9], g[13], o[13])
        for j in LOG_J:
            d = abs(g[j] - o[j]) / max(1.0, abs(o[j]))
            worst["log"] = max(worst["log"], d)
            assert d <= tl, (name, it, j, g[j], o[j])
        if it == 0 and recipe not in PIVOT_TIES:
            assert abs(g[12] - o[12]) <= tl * max(1.0, abs(o[12])), (name, it, g[12], o[12])
        else:
            assert np.sign(g[12]) == np.sign(o[12]), (name, it, g[12], o[12])
    for key, t in (("x", tx), ("u", tu), ("K", tk)):
        d = rel(sol[key][b], ref[key])
        worst[key] = max(worst[key], d)
        assert d < t, (name, key, d)


def report(title, worst):
    print(f"\n[{title}] largest relative differences: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))


# ---- 1. the recipes against the oracle ---------------------------------------------------------------------------------------------------------

def test_lq_blocks_match_oracle(model, built):
    """raw LQ blocks of every stage of every recipe, first iteration, 1e-9 relative"""
    st = abi.default_settings(model, sqp_iteration=1)
    worst = Counter()
    for group in by_node_count(built):
        s = new_solver(model, st, capture_raw_blocks=True)
        s.run([inst for _, inst in group])
        raw = s.raw_stage_blocks()
        for b, (name, inst) in enumerate(group):
            compare_blocks(model, raw[b], cached_oracle(model, (name,), inst, st, keep_raw=True)["raw"], name, worst)
    report(f"{model['name']} raw blocks", worst)


@pytest.mark.parametrize("iters", [1, 4])
def test_sqp_matches_oracle(model, built, iters):
    """one and four SQP iterations of every recipe: accepted steps bit for bit, step types and convergence codes, log fields, x, u, K"""
    st = abi.default_settings(model, sqp_iteration=iters, use_feedback_policy=1)
    worst = Counter()
    for group in by_node_count(built):
        sol = new_solver(model, st).run([inst for _, inst in group])
        assert not sol["status"].any()
        for b, (name, inst) in enumerate(group):
            compare_solve(model, sol, b, cached_oracle(model, (name,), inst, st), name, worst)
    report(f"{model['name']} SQP, {iters} iteration(s)", worst)


# ---- 2. per-instance penalty gains ---------------------------------------------------------------------------------------------------------------

# (label, {gain field: factor on the model's value}); the first set is the model's own
GAIN_CHANGES = [("model", {}), ("jlim_delta", {"jlim_delta": 2.0}), ("jlim_mu", {"jlim_mu": 3.0}), ("coll_delta", {"coll_delta": 2.0}),
                ("coll_radii", {"coll_r_foot": 1.3, "coll_r_knee": 1.3}), ("coll_mu", {"coll_mu": 3.0}), ("fric_delta", {"fric_delta": 2.0}),
                ("fric_mu", {"fric_mu": 3.0}), ("momxy_delta", {"momxy_delta": 2.0}), ("momxy_mu", {"momxy_mu": 3.0})]
# the penalty whose branch a set moves (mu-only sets keep the branches)
GAIN_TERM = {"jlim_delta": "joint_limits", "coll_delta": "collision", "coll_radii": "collision", "fric_delta": "friction", "momxy_delta": "moment"}


def gain_probe(model):
    """one state near every threshold: legs crossed slightly, joints ramped around delta of their limits, an unloaded foot, moments near the
    edge of the foot; each delta or radius of GAIN_CHANGES moves some of its rows into another branch"""
    geo = Geometry(model)
    inst = cross_legs(model, _copy(base_instance(model, "walk", 0.5 if is_cen(model) else 0.8)), 0.04, 0.14)
    inst = joints_at_limits(model, inst)
    return edge_moments(model, geo, unload_feet(model, geo, inst, 10.0, 40.0), 0.0, 0.08)


def test_per_instance_penalty_gains_match_the_oracle_of_their_model(model):
    """one batch, one state, a different penalty gain set per instance: each instance against the oracle of the model carrying its gains (raw
    blocks, one SQP iteration); the branch counts of each delta / radius set differ from the model's, and every set changes the solution"""
    inst = gain_probe(model)
    base = model_gains(model)
    sets = []
    for label, change in GAIN_CHANGES:
        g = {k: np.array(v, copy=True) for k, v in base.items()}
        for k, f in change.items():
            g[k] = g[k] * f
        sets.append((label, g))
    cnt0 = Geometry(model).counts(inst)
    print("\n" + format_counts("gains: model", cnt0))
    for label, g in sets[1:]:
        if label in GAIN_TERM:
            cnt = Geometry(model_with_gains(model, g)).counts(inst)
            print(format_counts(f"gains: {label}", cnt))
            term = GAIN_TERM[label]
            assert {k: v for k, v in cnt.items() if k[0] == term} != {k: v for k, v in cnt0.items() if k[0] == term}, label
    from wb_humanoid_mpc_b200.solver import stack_instances

    st = abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1)
    s = new_solver(model, st, capture_raw_blocks=True)
    B = len(sets)
    s.upload(stack_instances([inst] * B))
    s.set_gains(np.arange(B), {k: np.stack([np.asarray(g[k]) for _, g in sets]) for k in abi.GAIN_FIELDS})
    s.solve()
    sol = s.primal_solution()
    raw = s.raw_stage_blocks()
    assert not sol["status"].any()
    worst = Counter()
    for b, (label, g) in enumerate(sets):
        m = model_with_gains(model, g)
        ref = cached_oracle(m, ("gains", label), inst, st, keep_raw=True)
        compare_blocks(m, raw[b], ref["raw"], label, worst)
        compare_solve(m, sol, b, ref, label, worst, recipe="gain probe")
        if b:
            assert not np.array_equal(sol["x"][b], sol["x"][0]) and not np.array_equal(raw[b], raw[0]), label
    report(f"{model['name']} per-instance penalty gains", worst)


# ---- 3. above the cluster limit ---------------------------------------------------------------------------------------------------------------

def test_recipes_in_a_large_batch_match_their_alone_solves(model, built, default_dispatch):
    """the recipes of one node count mixed with nominal instances in a batch above the cluster limit (two-kernel K2): the raw blocks of every
    recipe bit for bit those of its alone-solve (K1 runs one CTA per node and instance); the first iteration against the alone-solve as in
    test_gpu_batch_paths.py::test_production_batch_matches_the_alone_solves, where the two-kernel K2 adds the regularisation in another order
    and forms symmetric entries once.  That test allows 1e-9 on nominal instances; here the penalty Hessians (collision mu = 1500 on J'J,
    relaxed-barrier curvature mu / delta^2) worsen the conditioning of the Riccati recursion, which amplifies the same round-off to a few
    1e-8, so the parity tolerance of the oracle comparisons, 1e-7, applies."""
    group = max(by_node_count(built), key=len)
    B = cluster_limit() + 1
    recipes_ = [inst for _, inst in group]
    rng_seeds = iter(range(100, 100 + B))
    insts = []
    for b in range(B):   # recipes spread over the batch, nominal walk instances between them
        insts.append(recipes_[b // 2] if b % 2 == 0 and b // 2 < len(recipes_) else None)
    for b in range(B):
        if insts[b] is None:
            insts[b] = base_instance(model, "walk", 0.5 if is_cen(model) else 0.8, seed=next(rng_seeds))
    assert all(len(i["t_nodes"]) == len(recipes_[0]["t_nodes"]) for i in insts)
    st = abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1)
    s = new_solver(model, st, capture_raw_blocks=True)
    sol = s.run(insts)
    assert_k2_path(s, model, st, True)
    assert not sol["status"].any()
    raw = s.raw_stage_blocks()
    alone, _ = solve_alone(model, st, insts, raw=True)
    picks = [b for b in range(B) if b % 2 == 0 and b // 2 < len(recipes_)]
    assert len(picks) == len(recipes_)
    for b in picks:
        assert np.array_equal(raw[b], alone[b]["raw"][0]), b
    worst = compare_first_iteration({k: v[picks] for k, v in sol.items()}, [alone[b] for b in picks], 1e-7)
    report(f"{model['name']} B={B}, two-kernel K2 against alone", worst)
