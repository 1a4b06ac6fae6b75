"""The whole-body and centroidal SQP on the code paths that only run at large batch sizes (GPU, through the C ABI).

K2 dispatch depends on the batch (b200sqp.cu launch_riccati): the 4-CTA cluster kernel runs while B * 4 * 2 <= #SMs (B <= 16 on an H100);
above that the whole-body sizes run riccati_wb.cuh's riccati_bwd_kernel + riccati_fwd_kernel, which the parity tests of tests/test_gpu_wb.py
(B <= 8) never reach.  From the fourth line-search trial on, rollout_kernel gathers several instances per CTA row (gridDim.y = ceil(B / 16)).

Reference for the large batches: the same instance solved alone (B = 1, cluster kernel).  K1 runs one CTA per (node, instance), so in the first
SQP iteration both solves see bit-identical LQ blocks and LU pivots, and only K2's arithmetic differs (riccati_wb.cuh adds reg_prim in another
order and computes symmetric entries once): 1e-9 relative.  Instances of one batch never interact (no cross-instance reduction outside the
global-step mode), so permuting the batch permutes every output bit for bit."""
import numpy as np
import pytest

import oracle_lib as orc
from test_gpu_wb import make_instances, oracle_solve, rel
from test_oracle_late_trials import assert_late_trial_case, late_trial_batch, late_trial_rows, late_trial_settings
from wb_humanoid_mpc_b200 import abi, model_loader, references

pytestmark = pytest.mark.gpu

OUT_KEYS = ("x", "u", "K", "log", "n_iter", "status")
LOG_J = (0, 1, 2, 3, 4, 5, 6, 7, 10, 11, 12)   # performance indices, norms and the Armijo metric of an iteration log


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


@pytest.fixture(scope="module")
def cmodel():
    return model_loader.load_packaged_model("g1_centroidal")


@pytest.fixture(params=["cluster", "two_kernel", "generic"])
def k2_mode(request, monkeypatch):
    """the three K2 variants of the whole-body sizes, forced for any batch (launch_riccati reads the variables on every launch)"""
    monkeypatch.setenv("B200SQP_NO_CLUSTER", "0" if request.param == "cluster" else "1")
    monkeypatch.setenv("B200SQP_K2_LEGACY", "1" if request.param == "generic" else "0")
    return request.param


@pytest.fixture
def default_dispatch(monkeypatch):
    monkeypatch.delenv("B200SQP_NO_CLUSTER", raising=False)
    monkeypatch.delenv("B200SQP_K2_LEGACY", raising=False)


def cluster_limit():
    """largest batch that launch_riccati gives to the cluster kernel (RC = 4 SMs per instance, at most half of the SMs)"""
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count // 8


def new_solver(model, st, **kw):
    from wb_humanoid_mpc_b200.solver import B200SqpSolver

    return B200SqpSolver(model, st, **kw)


_ONE_KERNEL_LAUNCHES = {}


def one_kernel_launches(model, st):
    """launch count of a solve whose K2 is one kernel (generic variant forced), for the same settings; the count does not depend on the
    instances (the whole back-tracking ladder is enqueued every iteration)"""
    key = (model.get("kind"), st.sqp_iteration, st.create_value_function, st.alpha_decay, st.alpha_min)
    if key not in _ONE_KERNEL_LAUNCHES:
        if model.get("kind") == "centroidal":
            from test_gpu_cen_ocp import make_instance

            inst = make_instance(model, np.random.default_rng(0), "stance", 0.2, None)
        else:
            inst = make_instances(model, np.random.default_rng(0), [("stance", 0.2, None)])[0]
        with pytest.MonkeyPatch.context() as mp:
            mp.setenv("B200SQP_NO_CLUSTER", "1")
            mp.setenv("B200SQP_K2_LEGACY", "1")
            s = new_solver(model, st)
            s.run([inst])
            _ONE_KERNEL_LAUNCHES[key] = s.launch_count()
    return _ONE_KERNEL_LAUNCHES[key]


def assert_k2_path(solver, model, st, two_kernel):
    """the two-kernel Riccati adds exactly one launch per SQP iteration to the launches of the cluster or generic kernel"""
    extra = solver.launch_count() - one_kernel_launches(model, st)
    assert extra == (st.sqp_iteration if two_kernel else 0), (extra, st.sqp_iteration, two_kernel)


def bench_batch(model, B, horizon):
    """bench.py build_batch (rank 0, gait walk): SEED 1234, perturbed initial states, random velocity commands, cold start"""
    rng = np.random.default_rng(1234)
    nj = model["nj"]
    lo, hi = np.array(model["q_lower"]), np.array(model["q_upper"])
    insts = []
    for _ in range(B):
        x0 = np.array(model["x_init"], float)
        x0[2] = model["reference"]["defaultBaseHeight"]
        x0[0:3] += rng.uniform(-0.02, 0.02, 3)
        x0[3:6] += rng.uniform(-0.05, 0.05, 3)
        x0[6:6 + nj] = np.clip(x0[6:6 + nj] + rng.uniform(-0.1, 0.1, nj), lo + 0.05, hi - 0.05)
        x0[6 + nj:] += rng.uniform(-0.2, 0.2, 6 + nj)
        cmd = [rng.uniform(-0.5, 1.0), rng.uniform(-0.3, 0.3), model["reference"]["defaultBaseHeight"], rng.uniform(-0.5, 0.5)]
        insts.append(references.build_instance(model, x0, t0=0.0, horizon=horizon, gait="walk", cmd=cmd))
    return insts


def solve_alone(model, st, insts, value_function=False, raw=False):
    """every instance solved on its own (B = 1: the cluster kernel), in one handle; -> (list of per-instance outputs, launch count)"""
    s = new_solver(model, st, capture_raw_blocks=raw)
    outs = []
    for inst in insts:
        o = s.run([inst])
        if value_function:
            o["P"], o["p"] = s.value_function()
        if raw:
            o["raw"] = s.raw_stage_blocks()
        outs.append(o)
    return outs, s.launch_count()


def assert_permutation_bitwise(model, st, insts, sol, seed, value_function=None):
    """the batch solved again in a shuffled order: every output of every instance bit for bit"""
    perm = np.random.default_rng(seed).permutation(len(insts))
    s = new_solver(model, st)
    sp = s.run([insts[i] for i in perm])
    for key in OUT_KEYS:
        if key in sol:
            assert np.array_equal(sp[key], sol[key][perm]), key
    if value_function is not None:
        Pp, pp = s.value_function()
        assert np.array_equal(Pp, value_function[0][perm]) and np.array_equal(pp, value_function[1][perm])


def compare_first_iteration(sol, alone, tol):
    """batch solve against the alone-solves, first SQP iteration: same step, step type and convergence code; log fields, x, u, K at tol.
    Returns the largest relative difference of each quantity."""
    worst = dict(log=0.0, x=0.0, u=0.0, K=0.0)
    for b, o in enumerate(alone):
        g, r = sol["log"][b, 0], o["log"][0, 0]
        assert g[8] == r[8] and int(g[9]) == int(r[9]) and int(g[13]) == int(r[13]), (b, g[8:14], r[8:14])
        assert sol["n_iter"][b] == o["n_iter"][0] and sol["status"][b] == o["status"][0]
        for j in LOG_J:
            worst["log"] = max(worst["log"], abs(g[j] - r[j]) / max(1.0, abs(r[j])))
        for key in ("x", "u", "K"):
            worst[key] = max(worst[key], rel(sol[key][b], o[key][0]))
    assert max(worst.values()) < tol, worst
    return worst


# ---- 1. whole-body SQP against the checker oracle under every K2 variant ------------------------------------------------------------------

_ORACLE = {}


def cached_oracle(model, key, inst, st):
    """the checker oracle does not depend on the K2 variant: one solve per instance and settings"""
    if key not in _ORACLE:
        _ORACLE[key] = oracle_solve(model, inst, st)
    return _ORACLE[key]


@pytest.mark.parametrize("iters", [1, 4])
def test_sqp_matches_oracle_under_every_k2_variant(model, k2_mode, iters):
    """tests/test_gpu_wb.py::test_sqp_end_to_end_matches_oracle (same instances and tolerances) with the K2 variant forced"""
    insts = make_instances(model, np.random.default_rng(2), [("stance", 1.1, None), ("stance", 1.1, [0.3, 0.1, 0.7925, 0.0]),
                                                             ("walk", 1.1, [0.4, 0.0, 0.7925, 0.1])])
    st = abi.default_settings(model, sqp_iteration=iters, use_feedback_policy=1)
    s = new_solver(model, st)
    sol = s.run(insts)
    assert_k2_path(s, model, st, k2_mode == "two_kernel")
    assert not sol["status"].any()
    for b, inst in enumerate(insts):
        ref = cached_oracle(model, ("e2e", b, iters), inst, st)
        nit = len(ref["log"])
        assert sol["n_iter"][b] == nit
        for it in range(nit):
            g, o = sol["log"][b, it], ref["log"][it]
            assert g[8] == o[8], ("step size", b, it, g[8], o[8])
            assert int(g[9]) == int(o[9]) and int(g[13]) == int(o[13])
            for j in (0, 1, 2, 3, 4, 5, 6, 7, 10, 11):
                assert abs(g[j] - o[j]) <= 1e-7 * max(1.0, abs(o[j])), (b, it, j, g[j], o[j])
            if it == 0:   # the Armijo metric depends on the LU's pivot order, which near-ties may flip after the first iteration
                assert abs(g[12] - o[12]) <= 1e-7 * max(1.0, abs(o[12])), (b, it, g[12], o[12])
            else:
                assert np.sign(g[12]) == np.sign(o[12])
        assert rel(sol["x"][b], ref["x"]) < 1e-7
        assert rel(sol["u"][b], ref["u"]) < 1e-7
        assert rel(sol["K"][b], ref["K"]) < 1e-6


def test_flight_gait_matches_oracle_under_every_k2_variant(model, k2_mode):
    """a run gait (flight phases: both feet swing) with the tolerances of test_gpu_wb.py::test_flight_and_single_support_gaits_match_oracle"""
    inst = make_instances(model, np.random.default_rng(13), [("run", 1.1, [0.3, 0.0, 0.7925, 0.1])])[0]
    assert (0, 0) in {tuple(c) for c in inst["contact_flags"]}
    st = abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1)
    s = new_solver(model, st)
    sol = s.run([inst])
    assert_k2_path(s, model, st, k2_mode == "two_kernel")
    ref = cached_oracle(model, ("run",), inst, st)
    assert not sol["status"].any()
    g, o = sol["log"][0, 0], ref["log"][0]
    assert g[8] == o[8] and int(g[9]) == int(o[9])
    for j in (0, 1, 2, 3, 4, 5, 6, 7, 10, 11):
        assert abs(g[j] - o[j]) <= 1e-7 * max(1.0, abs(o[j])), (j, g[j], o[j])
    assert np.sign(g[12]) == np.sign(o[12])
    assert rel(sol["x"][0], ref["x"]) < 1e-7
    assert rel(sol["u"][0], ref["u"]) < 1e-6
    assert rel(sol["K"][0], ref["K"]) < 1e-5


# ---- 2. skip flags and the value function --------------------------------------------------------------------------------------------------

def test_converged_instances_keep_their_qp_outputs_under_every_k2_variant(model, k2_mode):
    """tests/test_gpu_wb.py::test_value_function_of_instances_converging_at_different_iterations with the K2 variant forced; in addition the
    instance that converges first has the gains K and the re-centred cost-to-go (P, p) of the iteration it converged in, bit for bit: a solve
    capped at that iteration gives the same arrays (K2 must skip the converged instance in the later iterations of the batch)."""
    insts = make_instances(model, np.random.default_rng(16), [("walk", 0.3, [0.4, 0.0, 0.7925, 0.1])])
    x_nom = np.array(model["x_init"], float)
    x_nom[2] = model["reference"]["defaultBaseHeight"]
    insts.insert(0, references.build_instance(model, x_nom, t0=0.0, horizon=0.3, gait="stance", cmd=None))
    st = abi.default_settings(model, sqp_iteration=10, create_value_function=1, use_feedback_policy=1)
    s = new_solver(model, st)
    sol = s.run(insts)
    assert_k2_path(s, model, st, k2_mode == "two_kernel")
    P, p = s.value_function()
    n_iter = [int(v) for v in sol["n_iter"]]
    assert len(set(n_iter)) > 1, n_iter   # the case this test is about
    for b, inst in enumerate(insts):
        key = ("vf", b)
        if key not in _ORACLE:
            wb = orc.WbOracle(model)
            wb.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
            ref = wb.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], st)
            x_lin = ref["x"] - ref["log"][-1][8] * ref["dx"]   # linearisation trajectory of the instance's last iteration
            _ORACLE[key] = (len(ref["log"]), *wb.last_value_function(x_lin))
        nit, Po, po = _ORACLE[key]
        assert sol["n_iter"][b] == nit
        assert rel(P[b], Po) < 1e-6, (b, rel(P[b], Po))
        assert rel(p[b], po) < 1e-5, (b, rel(p[b], po))
    first = min(range(len(insts)), key=lambda b: n_iter[b])
    assert n_iter[first] < st.sqp_iteration
    st_cap = abi.default_settings(model, sqp_iteration=n_iter[first], create_value_function=1, use_feedback_policy=1)
    sc = new_solver(model, st_cap)
    cap = sc.run(insts)
    Pc, pc = sc.value_function()
    assert cap["n_iter"][first] == n_iter[first]
    assert np.array_equal(cap["K"][first], sol["K"][first])
    assert np.array_equal(Pc[first], P[first]) and np.array_equal(pc[first], p[first])
    assert np.array_equal(cap["x"][first], sol["x"][first]) and np.array_equal(cap["u"][first], sol["u"][first])


# ---- 3. production-size batch, default dispatch ---------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def production(model):
    """the benchmarked configuration (walk, horizon 3.5 s, cold start, one SQP iteration) at B = max(48, cluster limit + 1), solved in one
    batch (two-kernel K2) and every instance alone (cluster K2)"""
    with pytest.MonkeyPatch.context() as mp:
        mp.delenv("B200SQP_NO_CLUSTER", raising=False)
        mp.delenv("B200SQP_K2_LEGACY", raising=False)
        B = max(48, cluster_limit() + 1)
        insts = bench_batch(model, B, 3.5)
        assert len(insts[0]["t_nodes"]) == 115
        st = abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1)
        s = new_solver(model, st)
        sol = s.run(insts)
        launches = s.launch_count()
        alone, alone_launches = solve_alone(model, st, insts)
        return dict(insts=insts, st=st, sol=sol, launches=launches, alone=alone, alone_launches=alone_launches)


def test_production_batch_matches_the_alone_solves(model, production, default_dispatch):
    """3(a): instances of a 48-instance batch (two-kernel K2) against the same instances solved alone (cluster K2), 1e-9 relative"""
    B, st, sol = len(production["insts"]), production["st"], production["sol"]
    assert B > cluster_limit()
    # the two-kernel path ran in the batch (one launch more per iteration), a one-kernel path alone
    assert production["launches"] == one_kernel_launches(model, st) + st.sqp_iteration
    assert production["alone_launches"] == one_kernel_launches(model, st)
    assert not sol["status"].any()
    worst = compare_first_iteration(sol, production["alone"], 1e-9)
    print(f"\n[two-kernel vs cluster K2, whole-body B={B}, N=114] max relative differences: "
          + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


def test_production_batch_is_permutation_invariant(model, production, default_dispatch):
    """3(b): the batch solved in a shuffled order gives every instance's outputs bit for bit"""
    assert len(production["insts"]) > cluster_limit()
    assert_permutation_bitwise(model, production["st"], production["insts"], production["sol"], seed=48)


def test_production_batch_matches_the_fast_cpu_arm(model, production):
    """3(c): bench.py's parity check on the same inputs, for every instance: the same accepted step sizes, x within 1e-5 relative (instances
    whose complete-pivoting LU meets a pivot tie may be solved in another, equally valid, basis: ~1e-6, DESIGN.md section 2)"""
    import os

    from wb_humanoid_mpc_b200.solver import stack_instances

    sol = production["sol"]
    cpu = orc.fast_wb_sqp_batch(model, stack_instances(production["insts"]), production["st"], threads=max(1, min(16, os.cpu_count() or 1)))
    assert np.array_equal(sol["log"][:, 0, 8], cpu["log"][:, 0, 8])
    B = len(production["insts"])
    dx = np.abs(sol["x"] - cpu["x"]).reshape(B, -1).max(1) / np.abs(cpu["x"]).reshape(B, -1).max(1)
    print(f"\n[GPU vs fast CPU arm, B={B}] max relative difference of x: {dx.max():.2e} (median {np.median(dx):.2e})")
    assert dx.max() < 1e-5


def test_lq_blocks_do_not_depend_on_the_batch(model, production, default_dispatch):
    """3(d): the raw stage blocks of K1 (one CTA per node and instance) are bit for bit those of the alone-solve, at B = cluster limit + 4"""
    B = cluster_limit() + 4
    insts, st = production["insts"][:B], production["st"]
    s = new_solver(model, st, capture_raw_blocks=True)
    s.run(insts)
    assert_k2_path(s, model, st, True)
    raw = s.raw_stage_blocks()
    picks = [0, B // 2, B - 1]
    alone, _ = solve_alone(model, st, [insts[b] for b in picks], raw=True)
    for b, o in zip(picks, alone):
        assert np.array_equal(raw[b], o["raw"][0]), b


# ---- 4. late line-search trials: several instances per CTA row --------------------------------------------------------------------------

def test_late_trial_rollouts(model, default_dispatch):
    """the batch of tests/test_oracle_late_trials.py (B = 40, three CTA rows in the sparse roll-out launches): five instances of CTA row 1
    accept only at the fourth or fifth trial, a sixth exhausts the ladder (zero step), each at a different position along the row.  Against the
    alone-solves at 1e-9 and bitwise under permutation, as the production batch."""
    insts = late_trial_batch(model)
    st = late_trial_settings(model)
    B = len(insts)
    assert B > cluster_limit()
    s = new_solver(model, st)
    sol = s.run(insts)
    assert_k2_path(s, model, st, True)
    alphas = sol["log"][:, 0, 8]
    assert_late_trial_case(alphas, st.alpha_decay)
    by_row, zero = late_trial_rows(alphas, st.alpha_decay)
    print(f"\n[late trials, B={B}] instances accepted at trial >= 4 by CTA row: {by_row}; zero steps: {zero}")
    alone, _ = solve_alone(model, st, insts)
    compare_first_iteration(sol, alone, 1e-9)
    assert_permutation_bitwise(model, st, insts, sol, seed=40)


# ---- 5. several SQP iterations at a large batch --------------------------------------------------------------------------------------

def test_multi_iteration_large_batch(model, default_dispatch):
    """ten SQP iterations with the value function at B = cluster limit + 4; instances converge at different iterations (instances on their
    reference converge early, perturbed walking ones late).  Against the alone-solves: the same iteration counts and step sizes; after the
    first iteration round-off may flip an LU pivot tie, so the multi-iteration tolerances of tests/test_gpu_wb.py apply.  Bitwise under
    permutation."""
    B = cluster_limit() + 4
    assert B > cluster_limit()
    rng = np.random.default_rng(55)
    x_nom = np.array(model["x_init"], float)
    x_nom[2] = model["reference"]["defaultBaseHeight"]
    insts = []
    for b in range(B):
        if b % 3 == 0:
            insts.append(references.build_instance(model, x_nom, t0=0.0, horizon=0.3, gait="stance", cmd=None))
        else:
            insts += make_instances(model, rng, [("walk", 0.3, [0.1 * (b % 5), 0.0, 0.7925, 0.05 * (b % 3)])])
    st = abi.default_settings(model, sqp_iteration=10, create_value_function=1, use_feedback_policy=1)
    s = new_solver(model, st)
    sol = s.run(insts)
    assert_k2_path(s, model, st, True)
    P, p = s.value_function()
    assert not sol["status"].any()
    assert len(set(sol["n_iter"].tolist())) > 1, sol["n_iter"]
    alone, _ = solve_alone(model, st, insts, value_function=True)
    worst = dict(x=0.0, u=0.0, K=0.0, P=0.0, p=0.0)
    for b, o in enumerate(alone):
        assert sol["n_iter"][b] == o["n_iter"][0], b
        nit = int(o["n_iter"][0])
        assert np.array_equal(sol["log"][b, :nit, 8], o["log"][0, :nit, 8]), b
        for key, got in (("x", sol["x"][b]), ("u", sol["u"][b]), ("K", sol["K"][b]), ("P", P[b]), ("p", p[b])):
            worst[key] = max(worst[key], rel(got, o[key][0]))
    print(f"\n[ten iterations, B={B}, n_iter {sorted(set(sol['n_iter'].tolist()))}] max relative differences vs alone: "
          + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    assert worst["x"] < 1e-7 and worst["u"] < 1e-6 and worst["K"] < 1e-5 and worst["P"] < 1e-6 and worst["p"] < 1e-5, worst
    assert_permutation_bitwise(model, st, insts, sol, seed=10, value_function=(P, p))


# ---- 6. QP failure at the whole-body sizes ---------------------------------------------------------------------------------------------

def _failing_qp(Bn, bad, seed):
    from test_gpu_qp import _random_batch

    rng = np.random.default_rng(seed)
    nx, numax, N = 58, 23, 12
    pattern = rng.choice([21, 22, 23, 23, 0], size=(Bn, N)).astype(np.int32)
    pattern[bad, N // 2] = 23
    data, nu, dx0 = _random_batch(rng, Bn, N, nx, numax, pattern)
    data[5][bad, N // 2] = -100.0 * np.eye(numax)   # R indefinite at one stage of one instance
    return data, nu, dx0


def _check_failure(Bn, bad, seed):
    from wb_humanoid_mpc_b200.lib import B200SqpError
    from wb_humanoid_mpc_b200.qp import BatchedQp

    data, nu, dx0 = _failing_qp(Bn, bad, seed)
    qp = BatchedQp(Bn, 12, 58, 23)
    qp.upload(*data, dx0, nu)
    qp.solve()
    with pytest.raises(B200SqpError) as ei:
        qp.download()
    assert ei.value.code == -4
    sol = qp.download(raise_on_failure=False)
    assert sol["status"][bad] != 0
    A, Bm, b, Q, S, R, q, r = data
    for i in range(Bn):
        if i == bad:
            continue
        assert sol["status"][i] == 0, i
        ref = orc.riccati(A[i], Bm[i], b[i], Q[i], S[i], R[i], q[i], r[i], dx0[i], nu[i])
        for key in ("dx", "du", "K", "k", "P", "p"):
            assert rel(sol[key][i], ref[key]) < 1e-9, (i, key, rel(sol[key][i], ref[key]))


def test_qp_failure_at_whole_body_sizes_every_variant(k2_mode):
    """an indefinite R of one instance: that instance reports failure, download raises -4, the others still solve (1e-9 against the oracle)"""
    _check_failure(3, 1, 606)


def test_qp_failure_at_whole_body_sizes_large_batch(default_dispatch):
    Bn = cluster_limit() + 4
    assert Bn > cluster_limit()
    _check_failure(Bn, Bn - 3, 607)


# ---- 7. centroidal handles on the two-kernel path ----------------------------------------------------------------------------------------

def test_centroidal_sqp_matches_oracle_on_the_two_kernel_path(cmodel, monkeypatch):
    """forced two-kernel K2 at B = 3: the padded state rows 35..57 of the centroidal handle go through riccati_wb; parity with the centroidal
    oracle at the tolerances of tests/test_gpu_cen_ocp.py"""
    from test_gpu_cen_ocp import make_instance
    from test_gpu_cen_ocp import oracle_solve as cen_oracle_solve

    monkeypatch.setenv("B200SQP_NO_CLUSTER", "1")
    monkeypatch.setenv("B200SQP_K2_LEGACY", "0")
    rng = np.random.default_rng(72)
    insts = [make_instance(cmodel, rng, "walk", 0.6, [0.1 * i, 0.0, 0.7925, 0.1]) for i in range(3)]
    st = abi.default_settings(cmodel, sqp_iteration=3, use_feedback_policy=1)
    s = new_solver(cmodel, st)
    sol = s.run(insts)
    assert_k2_path(s, cmodel, st, True)
    assert not sol["status"].any()
    for b, inst in enumerate(insts):
        ref = cen_oracle_solve(cmodel, inst, st)
        nit = len(ref["log"])
        assert sol["n_iter"][b] == nit
        for it in range(nit):
            g, o = sol["log"][b, it], ref["log"][it]
            assert g[8] == o[8], ("step size", b, it, g[8], o[8])
            assert int(g[9]) == int(o[9]) and int(g[13]) == int(o[13])
            for j in (0, 1, 2, 3, 4, 5, 6, 7, 10, 11):
                assert abs(g[j] - o[j]) <= 1e-6 * max(1.0, abs(o[j])), (b, it, j, g[j], o[j])
        assert rel(sol["x"][b], ref["x"]) < 1e-6
        assert rel(sol["u"][b], ref["u"]) < 1e-6
        assert rel(sol["K"][b], ref["K"]) < 1e-5


def test_centroidal_large_batch_matches_the_alone_solves(cmodel, default_dispatch):
    """default dispatch above the cluster limit: every instance against its alone-solve at 1e-9 (first iteration), bitwise under permutation"""
    from test_gpu_cen_ocp import make_instance

    B = cluster_limit() + 8
    assert B > cluster_limit()
    rng = np.random.default_rng(73)
    insts = [make_instance(cmodel, rng, "walk", 1.0, [rng.uniform(-0.3, 0.6), rng.uniform(-0.2, 0.2), 0.7925, rng.uniform(-0.3, 0.3)],
                           momentum=bool(b % 2)) for b in range(B)]
    st = abi.default_settings(cmodel, sqp_iteration=1, use_feedback_policy=1)
    s = new_solver(cmodel, st)
    sol = s.run(insts)
    assert_k2_path(s, cmodel, st, True)
    assert not sol["status"].any()
    alone, _ = solve_alone(cmodel, st, insts)
    worst = compare_first_iteration(sol, alone, 1e-9)
    print(f"\n[two-kernel vs cluster K2, centroidal B={B}, N={len(insts[0]['t_nodes']) - 1}] max relative differences: "
          + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    assert_permutation_bitwise(cmodel, st, insts, sol, seed=73)


# ---- 8. fleet groups above the cluster limit ------------------------------------------------------------------------------------------

def test_fleet_groups_above_the_cluster_limit(model, default_dispatch):
    """a fleet whose two node-count groups (stance, run) both exceed the cluster limit: riccati_wb runs on views offset into the fleet-wide
    buffers; each group is bitwise the plain handle of the same instances (tests/test_gpu_fleet.py's rule)"""
    from test_gpu_builder import make_inputs
    from test_gpu_fleet import HORIZON, fleet_of, per_group_plain, solver

    lim = cluster_limit()
    B = 2 * (lim + 1)
    rng = np.random.default_rng(81)
    x0s, cmds = make_inputs(model, rng, B)
    gaits = ["stance" if b % 2 else "run" for b in range(B)]   # 36 and 38 nodes over 1.1 s
    starts = [0.5 if g == "stance" else 0.0 for g in gaits]
    kw = dict(iters=3, use_feedback_policy=1)
    fl = fleet_of(solver(model, **kw))
    n = fl.build_instances(0.0, HORIZON, x0s, gaits, starts, cmds)
    counts = {int(v): int((n == v).sum()) for v in np.unique(n)}
    assert sum(c > lim for c in counts.values()) >= 2, (counts, lim)
    dev = fl.download_instances()
    fl.solve()
    sol = fl.primal_solution()
    assert not sol["status"].any()
    for m, (idx, s) in per_group_plain(model, fl, dev, **kw).items():
        assert_k2_path(s, model, s.settings, len(idx) > lim)
        ref = s.primal_solution()
        assert np.array_equal(sol["x"][idx][:, :m], ref["x"]) and np.array_equal(sol["u"][idx][:, : m - 1], ref["u"])
        assert np.array_equal(sol["K"][idx][:, : m - 1], ref["K"])
        assert np.array_equal(sol["log"][idx], ref["log"]) and np.array_equal(sol["status"][idx], ref["status"])
        assert np.array_equal(sol["n_iter"][idx], ref["n_iter"])
