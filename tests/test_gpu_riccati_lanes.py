"""riccati_bwd_kernel's two lanes (GPU, through the C ABI).  Above the SM count the backward sweep runs two instances in one CTA, instance c
beside instance c + ceil(B / 2), each on its own four GEMM warps, helper warp, barriers and shared memory; at or below the SM count it runs one
instance per CTA.  The lanes share no arithmetic, so every output of an instance is the same, bit for bit, whether it ran beside a partner or
alone: the reference here is the same instances solved in batches of at most the SM count (and more than the cluster kernel's limit), where
no CTA pairs two instances."""
import numpy as np
import pytest

from test_gpu_batch_paths import OUT_KEYS, make_instances, new_solver
from test_gpu_qp import _random_batch
from test_gpu_qp_shapes import _check, _refs
from wb_humanoid_mpc_b200 import abi, model_loader, references

pytestmark = pytest.mark.gpu

NX, NM, N = 58, 23, 6
QP_KEYS = ("dx", "du", "K", "k", "P", "p", "status")


@pytest.fixture
def default_dispatch(monkeypatch):
    monkeypatch.delenv("B200SQP_NO_CLUSTER", raising=False)
    monkeypatch.delenv("B200SQP_K2_LEGACY", raising=False)


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def unpaired_chunks(B):
    """[lo, hi) ranges of at most the SM count and more than the cluster limit (SMs / 8) instances each, covering 0..B"""
    sms = sm_count()
    size = -(-B // -(-B // sms))
    assert size > sms // 8, B
    return [(lo, min(B, lo + size)) for lo in range(0, B, size)]


def _problem(B, seed):
    """B whole-body-size QPs of N stages: nu = 0 at stage i % (N + 1) of instance i (none when that is N), so that the two lanes of a CTA
    reach their input-free stages at different points of the sweep; every fifth instance has a random nu per stage"""
    rng = np.random.default_rng(seed)
    pattern = np.full((B, N), NM, dtype=np.int32)
    for i in range(B):
        if i % (N + 1) < N:
            pattern[i, i % (N + 1)] = 0
        if i % 5 == 4:
            pattern[i] = rng.integers(0, NM + 1, N)
    return _random_batch(rng, B, N, NX, NM, pattern)


def _solve(data, nu, dx0, lo, hi):
    from wb_humanoid_mpc_b200.qp import BatchedQp

    qp = BatchedQp(hi - lo, N, NX, NM)
    try:
        qp.upload(*[d[lo:hi] for d in data], dx0[lo:hi], nu[lo:hi])
        qp.solve(keep_P=True)
        return qp.download(raise_on_failure=False)
    finally:
        qp.close()


@pytest.mark.parametrize("B", [17, 132, 133, 255, 256, 264, 265, 1024])
def test_paired_instances_match_unpaired_batches(B, default_dispatch):
    """every output of every instance equals, bit for bit, the same instance solved in a batch that pairs none; instance 1 has an
    indefinite R~ at one stage, which fails it alone (status 1), while its partner in the CTA and everything else solve as before.  Both lanes
    of the first and last CTA also match the extended-precision reference of tests/test_gpu_qp_shapes.py."""
    data, nu, dx0 = _problem(B, seed=B)
    nu[1, N // 2] = NM
    data[5][1, N // 2] = -100.0 * np.eye(NM)
    sol = _solve(data, nu, dx0, 0, B)
    expect = np.zeros(B, dtype=np.int32)
    expect[1] = 1
    assert sol["status"].tolist() == expect.tolist()
    for lo, hi in unpaired_chunks(B):
        ref = _solve(data, nu, dx0, lo, hi)
        for key in QP_KEYS:
            assert np.array_equal(sol[key][lo:hi], ref[key], equal_nan=True), (B, lo, hi, key)
    half = -(-B // 2) if B > sm_count() else 0
    picks = sorted({0, half, B - 1})
    sub = [d[picks] for d in data]
    refs = _refs(sub, nu[picks], dx0[picks])
    _check({k: sol[k][picks] for k in ("dx", "du", "K", "k", "P", "p")}, refs, f"B={B} instances {picks}")


def test_converged_instances_beside_active_ones(default_dispatch):
    """ten SQP iterations at B = SM count + 8 (70 CTAs of two lanes on an H100): instances on their reference converge early and are skipped
    by K2 from then on, beside walking partners that keep iterating.  Every output (iteration counts and the log of the iterations each
    instance ran, the last QP's gains, the value function) equals, bit for bit, the same instances solved in two handles of B / 2, where no
    CTA pairs two instances.  (The log rows past an instance's n_iter are never written: they hold whatever the device memory held.)"""
    model = model_loader.load_packaged_model()
    B = 2 * (sm_count() // 2 + 4)
    rng = np.random.default_rng(77)
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
    P, p = s.value_function()
    assert not sol["status"].any()
    half = B // 2
    pairs_mixed = sum(int(sol["n_iter"][c] != sol["n_iter"][c + half]) for c in range(half))
    assert pairs_mixed > 0, sol["n_iter"]
    for lo in (0, half):
        h = new_solver(model, st)
        ref = h.run(insts[lo:lo + half])
        Pr, pr = h.value_function()
        for key in OUT_KEYS:
            if key in sol and key != "log":
                assert np.array_equal(sol[key][lo:lo + half], ref[key]), (lo, key)
        for b in range(half):
            nit = int(ref["n_iter"][b])
            assert np.array_equal(sol["log"][lo + b, :nit], ref["log"][b, :nit]), (lo + b, nit)
        assert np.array_equal(P[lo:lo + half], Pr) and np.array_equal(p[lo:lo + half], pr), lo
