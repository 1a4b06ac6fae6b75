"""The filter line search and the convergence checks under line-search settings other than the defaults, without a GPU.

Every recipe of RECIPES is one behaviour of SqpSolver::takeStep / FilterLinesearch::acceptStep / checkConvergence (SqpSolver.cpp:484-602):
each branch of the filter test (CONSTRAINT, COST with the Armijo test deciding, DUAL), each way the back-tracking ends (an accepted step, the
deltaTol early exit, running past alpha_min), each convergence code and their precedence, and ladders longer than 32 trials.  Here the fast
CPU arm (oracle/fast/wb_fast.cu, bench.py's timed CPU leg) is checked against the checker oracle on every recipe, and every recipe is checked
to produce the behaviour it is named for, so that tests/test_gpu_line_search.py compares the GPU with a CPU-checked expectation.  The trial
count of a ladder, and the settings the library rejects, are checked through b200sqp_line_search_trials, which needs no device."""
import ctypes as C
import math

import numpy as np
import pytest

import oracle_lib as orc
from test_oracle_late_trials import bench_instance
from wb_humanoid_mpc_b200 import abi, lib, model_loader
from wb_humanoid_mpc_b200.solver import stack_instances

CONSTRAINT, DUAL, COST, ZERO = 1, 2, 3, 4                     # StepType
ITERATIONS, STEPSIZE, METRICS, PRIMAL = 1, 2, 3, 4            # sqp::Convergence

# every trial takes the CONSTRAINT branch (g1 > g_max = 0) and would need g1 < (1 - gamma_c) g0 = 0: the whole ladder is rejected
FORCED = dict(g_max=0.0, gamma_c=1.0, delta_tol=0.0)


def ladder(alpha_decay, alpha_min):
    """the step sizes SqpSolver::takeStep tries (SqpSolver.cpp:527-565): alpha = 1 (a do-while), then alpha *= alpha_decay while >= alpha_min"""
    out, a = [], 1.0
    while True:
        out.append(a)
        a *= alpha_decay
        if not a >= alpha_min:
            return out


RECIPES = {
    # the whole ladder rejected: a zero step after 42 / 88 trials (more than the 32 an earlier enqueue served)
    "ladder42": dict(FORCED, sqp_iteration=2, alpha_decay=0.8),
    "ladder88": dict(FORCED, sqp_iteration=2, alpha_decay=0.9),
    # a long ladder whose step is accepted past the 32nd trial (the pushed instance of wb_instances)
    "late88": dict(sqp_iteration=1, alpha_decay=0.9),
    # ladders that end exactly on alpha_min: 0.125 = 0.5^3 (4 trials), 0.5^14 (15), 0.7^4 by repeated multiplication (5)
    "boundary_half_3": dict(FORCED, sqp_iteration=2, alpha_decay=0.5, alpha_min=0.125),
    "boundary_half_14": dict(FORCED, sqp_iteration=2, alpha_decay=0.5, alpha_min=0.5 ** 14),
    "boundary_07_4": dict(FORCED, sqp_iteration=2, alpha_decay=0.7, alpha_min=ladder(0.7, 0.2)[4]),
    # alpha_min >= 1: the do-while still tries alpha = 1 once
    "one_trial_1": dict(sqp_iteration=2, g_max=1e3, alpha_min=1.0),
    "one_trial_15": dict(sqp_iteration=2, g_max=1e3, alpha_min=1.5),
    # deltaTol early exit: alpha_decay^j max(|dx|, |du|) < 100 after 2-4 rejected trials (|du| is 200-550 at a bench cold start)
    "delta_exit": dict(FORCED, sqp_iteration=2, delta_tol=100.0),
    # a zero step with a large deltaTol converges by STEPSIZE, which precedes PRIMAL
    "stepsize_not_primal": dict(FORCED, sqp_iteration=3, delta_tol=1e3),
    # the three branches of the filter test (a cold start has g0 > 1: the default g_max = 1e-2 always gives CONSTRAINT)
    "constraint": dict(sqp_iteration=1, g_max=1e-8),
    "dual": dict(sqp_iteration=1, g_max=1e3),
    "cost": dict(sqp_iteration=1, g_max=1e3, g_min=1e3),
    "cost_armijo05": dict(sqp_iteration=1, g_max=1e3, g_min=1e3, armijo_factor=0.5),
    # convergence codes
    "metrics": dict(sqp_iteration=3, cost_tol=1e9, g_min=1e3),
    "primal": dict(sqp_iteration=3, g_max=1e3, cost_tol=0.0, delta_tol=1e3),
    # instances of one batch converge at different iterations with different codes
    "mixed_wb": dict(sqp_iteration=4, g_max=1e3, g_min=1e3, cost_tol=0.1),
    "mixed_cen": dict(sqp_iteration=4, g_max=1e3, cost_tol=0.0, delta_tol=10.0),
}
WB_RECIPES = [r for r in RECIPES if r != "mixed_cen"]
CEN_RECIPES = [r for r in RECIPES if r not in ("mixed_wb", "late88")]

LATE = (9, 5.0)   # seed, push of the instance that accepts only at 0.9^33 under "late88"


def settings(model, recipe):
    return abi.default_settings(model, use_feedback_policy=1, **RECIPES[recipe])


def pushed_instance(model, seed, push):
    """bench.py's distribution with the joint and base velocities of the initial state pushed by up to +-push"""
    inst = dict(bench_instance(model, seed, 0.5))
    nx = model["nx"]
    x0 = inst["x0"].copy()
    x0[nx // 2:] += push * np.random.default_rng(1000 + seed).uniform(-1.0, 1.0, nx - nx // 2)
    inst["x0"] = x0
    return inst


def wb_instances(model):
    """four cold starts of bench.py's distribution (in "mixed_wb" they converge after 1, 2, 3 and 4 iterations) and the pushed instance"""
    return [bench_instance(model, s, 0.5) for s in (3, 0, 6, 1)] + [pushed_instance(model, *LATE)]


def trial_index(step, st):
    """j with step == alpha_decay^j on the recipe's ladder (bit for bit), or None"""
    lad = ladder(st.alpha_decay, st.alpha_min)
    return lad.index(step) if step in lad else None


def assert_recipe(recipe, st, log, n_iter, family):
    """the recipe produced the behaviour it is named for; log [B][sqp_iteration][16], n_iter [B] of one batch"""
    B = len(n_iter)
    rows = [log[b, it] for b in range(B) for it in range(n_iter[b])]
    assert all(1 <= n_iter[b] <= st.sqp_iteration for b in range(B)), n_iter
    for r in rows:   # every accepted step lies on the ladder, every zero step is a ZERO step
        assert (r[8] == 0 and r[9] == ZERO) or (trial_index(r[8], st) is not None and r[9] in (CONSTRAINT, DUAL, COST)), (recipe, r[8:14])
    first = [log[b, 0] for b in range(B)]
    types = {int(r[9]) for r in first}
    if recipe in ("ladder42", "ladder88", "delta_exit", "stepsize_not_primal") or recipe.startswith("boundary"):
        assert all(n == 1 for n in n_iter) and all(r[9] == ZERO and r[13] == STEPSIZE for r in first), (recipe, [r[8:14] for r in first])
        assert all(r[2] + r[3] > 0 for r in first)   # g0 > 0, so that g1 < (1 - gamma_c) g0 = 0 is impossible
    if recipe == "late88":   # (the pushed instance)
        assert any(r[9] == CONSTRAINT and trial_index(r[8], st) >= 32 and r[8] < 0.9 ** 32 for r in first), [r[8:14] for r in first]
    if recipe.startswith("one_trial"):
        assert all(r[8] in (0.0, 1.0) for r in first)
        if recipe == "one_trial_15":
            assert all(r[13] == STEPSIZE for r in first)
        if family == "cen":
            assert any(r[8] == 1.0 for r in first)
    if recipe == "constraint":
        assert types == {CONSTRAINT}
    if recipe == "dual":
        assert types == {DUAL}
    if recipe == "cost":
        assert types == {COST}
    if recipe == "cost_armijo05":
        assert COST in types and types <= {COST, ZERO}
    if recipe == "metrics":
        assert all(n == 1 and r[13] == METRICS and r[8] > 0 for n, r in zip(n_iter, first))
    if recipe == "primal":
        assert all(r[13] == (PRIMAL if r[8] == 1.0 else STEPSIZE) for r in first)
        if family == "cen":
            assert any(r[13] == PRIMAL for r in first)
    if recipe.startswith("mixed"):
        ends = {(int(n_iter[b]), int(log[b, n_iter[b] - 1, 13])) for b in range(B)}
        assert len({n for n, _ in ends}) >= 2 and len({c for _, c in ends}) >= 2, ends


def delta_exit_trials(dxn, dun, st):
    """trials of a rejected ladder that the deltaTol early exit ends (SqpSolver.cpp:554-561)"""
    n, a = 1, 1.0
    while True:
        a *= st.alpha_decay
        if (a * dxn < st.delta_tol and a * dun < st.delta_tol) or not a >= st.alpha_min:
            return n
        n += 1


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


def line_search_trials(st):
    n = C.c_int32(-1)
    rc = lib.lib().b200sqp_line_search_trials(C.byref(st), C.byref(n))
    return rc, n.value


# ---- the ladder and the settings the library accepts ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("decay", [0.05, 0.1, 0.25, 0.5, 0.7, 0.8, 0.9, 0.95, 0.9523, 0.99])
@pytest.mark.parametrize("amin", [1e-300, 1e-9, 1e-4, 0.5 ** 14, 0.125, 0.2, 0.5, 0.99, 1.0, 1.5, 1e30])
def test_trial_count_is_the_reference_loop(model, decay, amin):
    st = abi.default_settings(model, alpha_decay=decay, alpha_min=amin)
    n = len(ladder(decay, amin))
    rc, got = line_search_trials(st)
    if n <= lib_max_trials():
        assert rc == 0 and got == n, (decay, amin, rc, got, n)
    else:
        assert rc == lib.EINVAL and b"B200SQP_MAX_LS_TRIALS" in lib.lib().b200sqp_last_error()


def lib_max_trials():
    import re
    from pathlib import Path

    text = (Path(__file__).resolve().parents[1] / "include" / "b200sqp.h").read_text()
    return int(re.search(r"#define B200SQP_MAX_LS_TRIALS\s+(\d+)", text).group(1))


def test_ladder_boundaries(model):
    """repeated multiplication decides the boundary, as on the device: 0.5^3 and 0.7^4 are on their ladders, their next-lower doubles not"""
    assert line_search_trials(abi.default_settings(model))[1] == 14   # the default settings
    for decay, j in ((0.5, 3), (0.5, 14), (0.7, 4), (0.9, 87)):
        a = ladder(decay, 1e-300)[j]
        assert line_search_trials(abi.default_settings(model, alpha_decay=decay, alpha_min=a))[1] == j + 1
        assert line_search_trials(abi.default_settings(model, alpha_decay=decay, alpha_min=math.nextafter(a, 2.0)))[1] == j
    assert 0.7 ** 4 != ladder(0.7, 0.2)[4]   # (the power is not the product the loop forms)
    assert line_search_trials(abi.default_settings(model, alpha_decay=0.95))[1] == 180
    for name in RECIPES:
        st = settings(model, name)
        assert line_search_trials(st) == (0, len(ladder(st.alpha_decay, st.alpha_min)))
    assert [line_search_trials(settings(model, r))[1] for r in ("ladder42", "ladder88", "boundary_half_3", "boundary_half_14", "boundary_07_4",
                                                                "one_trial_1", "one_trial_15")] == [42, 88, 4, 15, 5, 1, 1]


INVALID = [dict(alpha_decay=0.0), dict(alpha_decay=1.0), dict(alpha_decay=-0.5), dict(alpha_decay=1.5), dict(alpha_min=0.0), dict(alpha_min=-1e-4),
           dict(alpha_decay=0.999), dict(alpha_decay=0.96), dict(sqp_iteration=0), dict(sqp_iteration=1001)] + \
          [{f: v} for f in ("delta_tol", "cost_tol", "alpha_decay", "alpha_min", "gamma_c", "g_max", "g_min", "armijo_factor")
           for v in (math.nan, math.inf, -math.inf)]


@pytest.mark.parametrize("over", INVALID, ids=lambda o: ",".join(f"{k}={v}" for k, v in o.items()))
def test_invalid_settings_are_rejected(model, over):
    st = abi.default_settings(model, **over)
    assert line_search_trials(st) == (lib.EINVAL, -1)
    assert lib.lib().b200sqp_last_error().startswith(b"line_search_trials: ")


def test_global_step_serves_32_candidates(model):
    assert line_search_trials(abi.default_settings(model, global_step=1, alpha_decay=0.8, alpha_min=1e-3)) == (0, 31)
    assert line_search_trials(abi.default_settings(model, global_step=1, alpha_decay=0.8, alpha_min=1e-4)) == (lib.EINVAL, -1)
    assert b"global-step" in lib.lib().b200sqp_last_error()
    assert line_search_trials(abi.default_settings(model, global_step=0, alpha_decay=0.8, alpha_min=1e-4)) == (0, 42)


def test_create_rejects_the_settings_before_touching_a_device(model):
    """b200sqp_create / b200sqp_cen_create check the settings first: EINVAL and no handle, on any machine"""
    cm = model_loader.load_packaged_model("g1_centroidal")
    L = lib.lib()
    for over in (dict(alpha_decay=1.0), dict(alpha_min=math.nan), dict(global_step=1, alpha_decay=0.9)):
        h = C.c_void_p()
        st = abi.default_settings(model, **over)
        assert L.b200sqp_create(C.byref(abi.model_desc(model)), C.byref(st), 0, C.byref(h)) == lib.EINVAL and not h
        assert L.b200sqp_last_error().startswith(b"create: ")
        st = abi.default_settings(cm, **over)
        assert L.b200sqp_cen_create(C.byref(abi.model_desc(cm)), C.byref(abi.cen_desc(cm)), C.byref(st), 0, C.byref(h)) == lib.EINVAL and not h
        assert L.b200sqp_last_error().startswith(b"cen_create: ")


# ---- the recipes on the fast CPU arm against the checker oracle ----------------------------------------------------------------------------

def oracle_solve(model, inst, st):
    wb = orc.WbOracle(model)
    wb.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
    return wb.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], st)


def rel(a, b):
    return np.max(np.abs(a - b)) / max(1e-9, np.max(np.abs(b))) if b.size else 0.0


@pytest.mark.parametrize("recipe", WB_RECIPES)
def test_recipe_fast_arm_matches_checker_oracle(model, recipe):
    insts = wb_instances(model)
    st = settings(model, recipe)
    out = orc.fast_wb_sqp_batch(model, stack_instances(insts), st, threads=len(insts))
    for b, inst in enumerate(insts):
        ref = oracle_solve(model, inst, st)
        nit = len(ref["log"])
        assert out["n_iter"][b] == nit, (b, out["n_iter"][b], nit)
        for it in range(nit):
            g, o = out["log"][b, it], ref["log"][it]
            assert g[8] == o[8] and g[9] == o[9] and g[13] == o[13], (b, it, g[8:14], o[8:14])
            for j in (0, 1, 2, 3, 4, 5, 6, 7, 10, 11):
                assert abs(g[j] - o[j]) <= 1e-7 * max(1.0, abs(o[j])), (b, it, j, g[j], o[j])
        assert rel(out["x"][b], ref["x"]) < 1e-7 and rel(out["u"][b], ref["u"]) < 1e-6
    assert_recipe(recipe, st, out["log"], out["n_iter"], "wb")
    if recipe == "delta_exit":   # the early exit, not alpha_min, ends these ladders, after 2-4 trials
        dflt = orc.fast_wb_sqp_batch(model, stack_instances(insts), abi.default_settings(model, g_max=1e3), threads=len(insts))
        for b in range(len(insts)):
            step = dflt["log"][b, 0, 8]
            n = delta_exit_trials(dflt["log"][b, 0, 10] / step, dflt["log"][b, 0, 11] / step, st)
            assert 2 <= n < len(ladder(st.alpha_decay, st.alpha_min)) and (n <= 4 or b == len(insts) - 1), (b, n)   # (the pushed one: 7)


def test_recipes_reach_every_branch_and_code(model):
    """over the recipes: every step type and every convergence code of the whole-body solver, and an instance accepting past trial 32"""
    insts = wb_instances(model)
    types, codes = set(), set()
    for recipe in WB_RECIPES:
        st = settings(model, recipe)
        out = orc.fast_wb_sqp_batch(model, stack_instances(insts), st, threads=len(insts))
        for b in range(len(insts)):
            for it in range(out["n_iter"][b]):
                types.add(int(out["log"][b, it, 9]))
                codes.add(int(out["log"][b, it, 13]))
    assert types == {CONSTRAINT, DUAL, COST, ZERO} and codes >= {ITERATIONS, STEPSIZE, METRICS}, (types, codes)
