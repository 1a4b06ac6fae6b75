"""The batch of tests/test_gpu_batch_paths.py::test_late_trial_rollouts, checked on the fast CPU arm (oracle/fast/wb_fast.cu): its line
search runs past the third trial for instances that share a CTA row of the sparse roll-out launches, and one instance exhausts the ladder.

From the fourth trial on, the whole-body solver launches rollout_kernel with gridDim.y = ceil(B / 16): each CTA row gathers the instances
b = y, y + gridDim.y, ... that still search and rolls them out one after the other.  The case only occurs if the batch has instances that
accept late, so the precondition is asserted here, without a GPU; the GPU test asserts it again from the solver's own log."""
import numpy as np
import pytest

import oracle_lib as orc
from wb_humanoid_mpc_b200 import abi, model_loader, references
from wb_humanoid_mpc_b200.solver import stack_instances

LATE_B, LATE_HORIZON = 40, 1.1
# a gentler back-tracking (0.7 instead of 0.5) makes instances of the benchmark distribution accept at the fourth or fifth trial; the ladder
# 1, 0.7, 0.49, 0.343, 0.2401 ends above alpha_min = 0.2, so an instance that needs a smaller step takes a zero step
LATE_SETTINGS = dict(alpha_decay=0.7, alpha_min=0.2)


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


def bench_instance(model, seed, horizon, gait="walk"):
    """one instance of bench.py's distribution (perturbed initial state, random velocity command, cold start), drawn from its own seed"""
    rng = np.random.default_rng(seed)
    nj = model["nj"]
    lo, hi = np.array(model["q_lower"]), np.array(model["q_upper"])
    x0 = np.array(model["x_init"], float)
    x0[2] = model["reference"]["defaultBaseHeight"]
    x0[0:3] += rng.uniform(-0.02, 0.02, 3)
    x0[3:6] += rng.uniform(-0.05, 0.05, 3)
    x0[6:6 + nj] = np.clip(x0[6:6 + nj] + rng.uniform(-0.1, 0.1, nj), lo + 0.05, hi - 0.05)
    x0[6 + nj:] += rng.uniform(-0.2, 0.2, 6 + nj)
    cmd = [rng.uniform(-0.5, 1.0), rng.uniform(-0.3, 0.3), model["reference"]["defaultBaseHeight"], rng.uniform(-0.5, 0.5)]
    return references.build_instance(model, x0, t0=0.0, horizon=horizon, gait=gait, cmd=cmd)


def late_trial_seeds():
    """seeds 0..39, with the five seeds that accept at the fourth or fifth trial (2, 18, 25, 32, 36) and the one that takes a zero step (9)
    moved to b = 4, 7, ..., 19: all in CTA row 1 of the sparse launches and each at a different position along it, so that an instance
    stride other than gridDim.y misses some of them"""
    order = list(range(LATE_B))
    for seed, pos in ((2, 4), (18, 7), (25, 10), (32, 13), (36, 16), (9, 19)):
        i = order.index(seed)
        order[i], order[pos] = order[pos], order[i]
    return order


def late_trial_batch(model):
    return [bench_instance(model, s, LATE_HORIZON) for s in late_trial_seeds()]


def late_trial_settings(model, **over):
    return abi.default_settings(model, sqp_iteration=1, use_feedback_policy=1, **LATE_SETTINGS, **over)


def late_trial_rows(alphas, decay):
    """{CTA row of the sparse launches: [instances of that row accepted at trial >= 4]}, and the instances that took a zero step"""
    rows = (len(alphas) + 15) // 16
    late = [b for b, a in enumerate(alphas) if 0 < a <= decay ** 3 * (1 + 1e-12)]
    by_row = {}
    for b in late:
        by_row.setdefault(b % rows, []).append(b)
    return by_row, [b for b, a in enumerate(alphas) if a == 0]


def assert_late_trial_case(alphas, decay):
    """at least three CTA rows; a row other than 0 holds two or more late instances past its first position; some instance takes a zero step"""
    rows = (len(alphas) + 15) // 16
    assert rows >= 3
    by_row, zero = late_trial_rows(alphas, decay)
    assert any(r != 0 and len([b for b in v if b >= rows]) >= 2 for r, v in by_row.items()), by_row
    assert zero, alphas


def test_late_trial_batch_reaches_the_sparse_rollouts(model):
    st = late_trial_settings(model)
    out = orc.fast_wb_sqp_batch(model, stack_instances(late_trial_batch(model)), st, threads=4)
    alphas = out["log"][:, 0, 8]
    assert_late_trial_case(alphas, st.alpha_decay)
