"""The filter line search and the convergence checks on the GPU (through the C ABI) under the recipes of tests/test_oracle_line_search.py,
against the checker oracle, on whole-body and centroidal handles (both share accept_kernel and evalTrial).

Each recipe runs at a batch the cluster K2 kernel serves and at one batch above the cluster limit (the two-kernel Riccati, and the sparse
rollout_kernel launches of trial >= 3); the large batch tiles the small one, so every instance is compared with the oracle solve of its own
initial guess.  The accepted step sizes, step types, convergence codes and iteration counts match bit for bit; the log rows and the primal
trajectory at the tolerances of tests/test_gpu_wb.py (whole body) and tests/test_gpu_cen_ocp.py (centroidal).  The Armijo metric is compared
on the first iteration only: past it, an exact tie in the complete-pivoting LU may move it by ~3e-4 (DESIGN.md section 2); the recipes whose
decisions the Armijo test takes (cost, cost_armijo05) run one iteration, and mixed_wb's later decisions were checked not to sit on such a tie.
Each handle first solves the batch in reverse order, so that log rows an earlier solve wrote must not reappear past n_iter."""
import math

import numpy as np
import pytest

from test_gpu_batch_paths import cluster_limit, new_solver
from test_gpu_cen_ocp import make_instance
from test_gpu_cen_ocp import oracle_solve as cen_oracle_solve
from test_gpu_wb import oracle_solve as wb_oracle_solve
from test_gpu_wb import rel
from test_oracle_line_search import (CEN_RECIPES, COST, CONSTRAINT, DUAL, INVALID, ITERATIONS, METRICS, PRIMAL, STEPSIZE, WB_RECIPES,
                                     ZERO, assert_recipe, ladder, line_search_trials, settings, wb_instances)
from wb_humanoid_mpc_b200 import abi, lib, model_loader

pytestmark = pytest.mark.gpu

TOL = {"wb": 1e-7, "cen": 1e-6}


@pytest.fixture(scope="module")
def models():
    return {"wb": model_loader.load_packaged_model(), "cen": model_loader.load_packaged_model("g1_centroidal")}


_INSTANCES = {}


def instances(models, family):
    if family not in _INSTANCES:
        if family == "wb":
            _INSTANCES[family] = wb_instances(models["wb"])
        else:
            rng = np.random.default_rng(3)
            _INSTANCES[family] = [make_instance(models["cen"], rng, "stance", 0.5, None),
                                  make_instance(models["cen"], rng, "walk", 0.5, [0.3, 0.0, 0.7925, 0.1])]
    return _INSTANCES[family]


_ORACLE = {}


def oracle(models, family, recipe, i):
    key = (family, recipe, i)
    if key not in _ORACLE:
        solve = wb_oracle_solve if family == "wb" else cen_oracle_solve
        _ORACLE[key] = solve(models[family], instances(models, family)[i], settings(models[family], recipe))
    return _ORACLE[key]


_COVERAGE = {"wb": (set(), set()), "cen": (set(), set())}


@pytest.mark.parametrize("size", ["cluster", "above_cluster"])
@pytest.mark.parametrize("family,recipe", [("wb", r) for r in WB_RECIPES] + [("cen", r) for r in CEN_RECIPES])
def test_recipe_matches_oracle(models, family, recipe, size):
    model = models[family]
    base = instances(models, family)
    B = len(base) if size == "cluster" else cluster_limit() + 1
    insts = [base[b % len(base)] for b in range(B)]
    st = settings(model, recipe)
    s = new_solver(model, st)
    s.run(insts[::-1])
    sol = s.run(insts)
    assert not sol["status"].any()
    tol = TOL[family]
    for b in range(B):
        ref = oracle(models, family, recipe, b % len(base))
        nit = len(ref["log"])
        assert sol["n_iter"][b] == nit, (b, sol["n_iter"][b], nit)
        for it in range(nit):
            g, o = sol["log"][b, it], ref["log"][it]
            assert g[8] == o[8] and g[9] == o[9] and g[13] == o[13], (b, it, g[8:14], o[8:14])
            for j in (0, 1, 2, 3, 4, 5, 6, 7, 10, 11):
                assert abs(g[j] - o[j]) <= tol * max(1.0, abs(o[j])), (b, it, j, g[j], o[j])
            if it == 0:
                assert abs(g[12] - o[12]) <= tol * max(1.0, abs(o[12])), (b, g[12], o[12])
        assert not sol["log"][b, nit:].any(), (b, nit)   # rows this solve did not write are zeros
        assert rel(sol["x"][b], ref["x"]) < tol and rel(sol["u"][b], ref["u"]) < tol
    assert_recipe(recipe, st, sol["log"], sol["n_iter"], family)
    types, codes = _COVERAGE[family]
    for b in range(B):
        types.update(int(v) for v in sol["log"][b, : sol["n_iter"][b], 9])
        codes.update(int(v) for v in sol["log"][b, : sol["n_iter"][b], 13])


@pytest.mark.parametrize("family", ["wb", "cen"])
def test_recipes_reached_every_step_type_and_code(models, family):
    """(runs after test_recipe_matches_oracle in file order) every step type and convergence code was reached on the GPU"""
    types, codes = _COVERAGE[family]
    if not types:
        pytest.skip("test_recipe_matches_oracle did not run")
    assert types == {CONSTRAINT, DUAL, COST, ZERO}, types
    assert codes >= {ITERATIONS, STEPSIZE, METRICS} | ({PRIMAL} if family == "cen" else set()), codes


@pytest.mark.parametrize("family", ["wb", "cen"])
@pytest.mark.parametrize("recipe", ["ladder88", "boundary_half_3", "boundary_07_4", "one_trial_15"])
def test_whole_ladder_is_enqueued(models, family, recipe):
    """each SQP iteration enqueues one roll-out and one accept_kernel per trial of the ladder: 14 with the default settings"""
    model = models[family]
    st = settings(model, recipe)
    n = len(ladder(st.alpha_decay, st.alpha_min))
    assert line_search_trials(st) == (0, n)
    launches = []
    for s_ in (st, abi.default_settings(model, use_feedback_policy=1, sqp_iteration=st.sqp_iteration)):
        s = new_solver(model, s_)
        s.run(instances(models, family)[:1])
        launches.append(s.launch_count())
    assert launches[0] - launches[1] == 2 * (n - 14) * st.sqp_iteration, (launches, n)


@pytest.mark.parametrize("family", ["wb", "cen"])
def test_invalid_settings_create_nothing(models, family):
    model = models[family]
    L = lib.lib()
    for over in INVALID + [dict(global_step=1, alpha_decay=0.9)]:
        with pytest.raises(lib.B200SqpError) as e:
            new_solver(model, abi.default_settings(model, **over))
        assert e.value.code == lib.EINVAL, over
        assert b"create: " in L.b200sqp_last_error()


@pytest.mark.parametrize("family", ["wb", "cen"])
def test_global_step_ladder(models, family):
    """the global-step mode walks the trials of the back-tracking ladder (at most 32): alpha = 1 even with alpha_min > 1"""
    model = models[family]
    for over, n in ((dict(alpha_decay=0.8, alpha_min=1e-3), 31), (dict(alpha_min=1.5), 1), ({}, 14)):
        st = abi.default_settings(model, global_step=1, **over)
        s = new_solver(model, st)
        lad = s.global_ladder()
        assert len(lad) == n and list(lad) == ladder(st.alpha_decay, st.alpha_min)
    s.run(instances(models, family)[:1])
    stats, chosen = s.global_stats()
    assert len(stats) >= 1 and math.isfinite(stats[0, 2])
