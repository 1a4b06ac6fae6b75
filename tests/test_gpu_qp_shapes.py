"""The batched QP (b200sqp_qp_*, BatchedQp) across the sizes its C ABI accepts, against the Riccati recursion restated in extended precision.

b200sqp_qp_create accepts 0 < nx <= 64 and 0 < nu_max <= 32 whenever both generic kernels fit one block's shared memory.  Every size other
than the whole-body (58, 23) runs through riccati_kernel<0, 0> (one CTA per instance) or riccati_cluster_kernel<0, 0> (a cluster of four), so
this file sweeps sizes chosen where those kernels can go wrong: the scratch [K | k] at the end of W (it overflowed into Y[0] at sizes with
nu_max close to or above nx), DMMA tiles cut at every edge, each branch of warp_chol_inverse, and the largest layouts.  Each is compared at
1e-10 (relative to max(1, |ref|)) with `riccati_ref`, HPIPM's unconstrained recursion as oracle_lib.riccati states it, here in np.longdouble
(a 64-bit mantissa on x86-64), so that the difference measured is the kernel's rounding alone.

The overflow only shows where a later stage is prefetched into Y[0] while [K | k] is formed, i.e. at a stage k >= 1 with N - 1 - k odd: the
sweep uses N >= 3 there; N = 1 and N = 2 run as stage edges of their own.  In the cluster kernel only the last CTA of a cluster writes the tail
of [K | k], and the overflow lands in the first columns of that CTA's Y[0], which it never reads (it uses its own column slice of S~ and the
gathered copy): the results go wrong only where the overflow reaches the slice, as at (3, 32).  Elsewhere it is latent, and
tests/test_emu_riccati_layout.py is what holds the layout.  The whole-body instantiations get the same stage edges (N = 1, 2,
nu = 0 on the first, the last or every stage, keep_P = 0) in all three of their K2 variants."""
import os

import numpy as np
import pytest

import oracle_lib as orc
from wb_humanoid_mpc_b200 import lib
from test_gpu_qp import _random_batch, k2_mode  # noqa: F401  (k2_mode: the fixture of the whole-body variants)

LD = np.longdouble
TOL = 1e-10
KEYS = ("dx", "du", "K", "k", "P", "p")

# (nx, nu_max): where [K | k] overflowed W (both variants / one-CTA only / cluster only); DMMA tile edges (M, N, K off multiples of 8 and 4);
# nu_max at both ends of every warp_chol_inverse branch (8 | 16 | 24 | 32); the largest accepted layouts; the sizes tested before
OVERFLOW_BOTH = [(4, 4), (12, 12), (28, 28), (3, 32), (16, 32), (9, 17)]
OVERFLOW_ONE_CTA = [(4, 1), (20, 16), (36, 32)]
OVERFLOW_CLUSTER = [(3, 3), (8, 8), (9, 9)]
TILE_EDGES = [(1, 1), (7, 3), (33, 25), (57, 24), (63, 1), (2, 5), (11, 9)]
CHOL_BRANCHES = [(40, 8), (24, 17), (13, 24), (47, 31)]
LARGEST = [(52, 32), (64, 15), (56, 24), (60, 20)]
BEFORE = [(3, 2), (35, 23), (58, 23)]
SIZES = OVERFLOW_BOTH + OVERFLOW_ONE_CTA + OVERFLOW_CLUSTER + TILE_EDGES + CHOL_BRANCHES + LARGEST + BEFORE
SIZE_IDS = [f"{nx}x{nm}" for nx, nm in SIZES]
# the sizes qp_create refuses because the cluster layout does not fit (the one-CTA layout alone would)
CLUSTER_TOO_BIG = [(57, 28), (58, 26), (58, 27), (58, 28), (59, 25), (59, 26), (59, 27), (59, 28), (60, 24), (60, 25), (60, 26), (60, 27)]


# ---- the reference -----------------------------------------------------------------------------------------------------------------------------
def _chol(R):
    """lower Cholesky factor by plain loops, None for a non-positive pivot"""
    n = R.shape[0]
    L = np.zeros_like(R)
    for j in range(n):
        d = R[j, j] - L[j, :j] @ L[j, :j]
        if not d > 0:
            return None
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (R[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def _solve_lower(L, Y):
    X = np.zeros_like(Y)
    for i in range(L.shape[0]):
        X[i] = (Y[i] - L[i, :i] @ X[:i]) / L[i, i]
    return X


def _solve_upper_t(L, Y):
    """L' X = Y"""
    X = np.zeros_like(Y)
    for i in reversed(range(L.shape[0])):
        X[i] = (Y[i] - L[i + 1:, i] @ X[i + 1:]) / L[i, i]
    return X


def riccati_ref(A, Bm, b, Q, S, R, q, r, dx0, nu, reg):
    """One instance (math layout, stage arrays padded to nu_max as BatchedQp takes them) in np.longdouble: P_N = Q_N + reg I; per stage
    Q~ = Q + A'PA + reg I, S~ = S + B'PA, R~ = R + B'PB + reg I, q~ = q + A'(Pb + p), r~ = r + B'(Pb + p); R~ = L L';
    K = -L^-T L^-1 S~, k = -L^-T L^-1 r~, P = Q~ - S~'R~^-1 S~, p = q~ - S~'R~^-1 r~; then the forward sweep from dx0.  None if some R~ is
    not positive definite."""
    A, Bm, b, Q, S, R, q, r, dx0 = (np.asarray(a, dtype=LD) for a in (A, Bm, b, Q, S, R, q, r, dx0))
    N, nx, nm = A.shape[0], A.shape[1], Bm.shape[2]
    reg = LD(reg)
    I = np.eye(nx, dtype=LD)
    P = np.zeros((N + 1, nx, nx), dtype=LD)
    p = np.zeros((N + 1, nx), dtype=LD)
    K = np.zeros((N, nm, nx), dtype=LD)
    k = np.zeros((N, nm), dtype=LD)
    P[N] = Q[N] + reg * I
    p[N] = q[N]
    for s in reversed(range(N)):
        m = int(nu[s])
        Pn, Ak, Bk = P[s + 1], A[s], Bm[s][:, :m]
        v = Pn @ b[s] + p[s + 1]
        PA = Pn @ Ak
        Qt = Q[s] + Ak.T @ PA + reg * I
        qt = q[s] + Ak.T @ v
        if m == 0:
            P[s], p[s] = 0.5 * (Qt + Qt.T), qt
            continue
        Rt = R[s][:m, :m] + Bk.T @ Pn @ Bk + reg * np.eye(m, dtype=LD)
        St = S[s][:m] + Bk.T @ PA
        rt = r[s][:m] + Bk.T @ v
        L = _chol(Rt)
        if L is None:
            return None
        Ys, yr = _solve_lower(L, St), _solve_lower(L, rt)
        Pk = Qt - Ys.T @ Ys
        P[s], p[s] = 0.5 * (Pk + Pk.T), qt - Ys.T @ yr
        K[s, :m], k[s, :m] = -_solve_upper_t(L, Ys), -_solve_upper_t(L, yr)
    dx = np.zeros((N + 1, nx), dtype=LD)
    du = np.zeros((N, nm), dtype=LD)
    dx[0] = dx0
    for s in range(N):
        m = int(nu[s])
        du[s, :m] = K[s, :m] @ dx[s] + k[s, :m]
        dx[s + 1] = A[s] @ dx[s] + Bm[s][:, :m] @ du[s, :m] + b[s]
    return dict(dx=dx, du=du, K=K, k=k, P=P, p=p)


def _rel(a, ref):
    ref = np.asarray(ref, dtype=LD)
    return float(np.max(np.abs(np.asarray(a, dtype=LD) - ref)) / max(LD(1), np.max(np.abs(ref))))


# ---- problems and solves -----------------------------------------------------------------------------------------------------------------------
def _patterns(rng, N, nm):
    """one row of per-stage nu per instance: all nu_max; 0 on the first stage; 0 on the last stage; all 1; a random mix including 0"""
    rows = [np.full(N, nm), np.r_[0, np.full(N - 1, nm)], np.r_[np.full(N - 1, nm), 0], np.ones(N), rng.integers(0, nm + 1, N)]
    rows[4][rng.integers(0, N)] = 0
    return np.array(rows, dtype=np.int32)


def _problem(nx, nm, N, seed=0, pattern=None):
    rng = np.random.default_rng(seed * 100003 + nx * 100 + nm)
    pattern = _patterns(rng, N, nm) if pattern is None else np.asarray(pattern, dtype=np.int32)
    data, nu, dx0 = _random_batch(rng, len(pattern), N, nx, nm, pattern)
    return data, nu, dx0


def _refs(data, nu, dx0, reg=1e-12):
    A, Bm, b, Q, S, R, q, r = data
    return [riccati_ref(A[i], Bm[i], b[i], Q[i], S[i], R[i], q[i], r[i], dx0[i], nu[i], reg) for i in range(len(nu))]


def _set_variant(variant):
    """cluster: the 4-CTA cluster kernel (the default while B <= 16); one_cta: the one-CTA kernel (B200SQP_K2_LEGACY also keeps the whole-body
    sizes on it); natural: launch_riccati's own choice"""
    for key in ("B200SQP_NO_CLUSTER", "B200SQP_K2_LEGACY"):
        os.environ.pop(key, None)
    if variant == "cluster":
        os.environ["B200SQP_NO_CLUSTER"] = "0"
    elif variant == "one_cta":
        os.environ["B200SQP_NO_CLUSTER"] = "1"
        os.environ["B200SQP_K2_LEGACY"] = "1"


@pytest.fixture
def restore_env():
    saved = {k: os.environ.get(k) for k in ("B200SQP_NO_CLUSTER", "B200SQP_K2_LEGACY")}
    yield
    for k, v in saved.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


def _solve(data, nu, dx0, variant=None, reg=1e-12, keep_P=True):
    from wb_humanoid_mpc_b200.qp import BatchedQp

    if variant is not None:
        _set_variant(variant)
    Bn, N, nx, nm = data[1].shape
    qp = BatchedQp(Bn, N, nx, nm)
    try:
        qp.upload(*data, dx0, nu)
        qp.solve(reg_prim=reg, keep_P=keep_P)
        return qp.download(raise_on_failure=False)
    finally:
        qp.close()


def _check(sol, refs, label, instances=None, keys=KEYS):
    worst = 0.0
    for i in (range(len(refs)) if instances is None else instances):
        for key in keys:
            e = _rel(sol[key][i], refs[i][key])
            worst = max(worst, e)
            assert e < TOL, (label, i, key, e)
    print(f"{label}: largest difference {worst:.2e}")
    return worst


# ---- the reference against the oracle (no GPU) -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nx,nm", [(3, 2), (9, 17), (12, 12), (35, 23), (58, 23)], ids=lambda v: str(v))
@pytest.mark.parametrize("reg", [0.0, 1e-12, 1e-6])
def test_reference_agrees_with_the_oracle(nx, nm, reg):
    """the two restatements of the recursion pin each other: oracle_lib.riccati (double) and riccati_ref (extended precision)"""
    data, nu, dx0 = _problem(nx, nm, 5)
    A, Bm, b, Q, S, R, q, r = data
    refs = _refs(data, nu, dx0, reg)
    for i in range(len(nu)):
        o = orc.riccati(A[i], Bm[i], b[i], Q[i], S[i], R[i], q[i], r[i], dx0[i], nu[i], reg=reg)
        for key in KEYS:
            assert _rel(o[key], refs[i][key]) < TOL, (i, key, _rel(o[key], refs[i][key]))


# ---- the generic kernels across sizes --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("nx,nm", SIZES, ids=SIZE_IDS)
@pytest.mark.parametrize("variant", ["cluster", "one_cta"])
def test_size_against_extended_precision(variant, nx, nm, restore_env):
    """five instances at N = 7 and five at N = 3, one per stage pattern of _patterns (nu = nu_max; 0 on the first stage; 0 on the last;
    1 everywhere; a random mix including 0)"""
    for N, seed in ((7, 0), (3, 1)):
        data, nu, dx0 = _problem(nx, nm, N, seed)
        sol = _solve(data, nu, dx0, variant)
        assert not sol["status"].any(), sol["status"]
        _check(sol, _refs(data, nu, dx0), f"{variant} ({nx}, {nm}) N={N}")


@pytest.mark.gpu
@pytest.mark.parametrize("nx,nm", SIZES, ids=SIZE_IDS)
def test_variants_agree_bit_for_bit(nx, nm, restore_env):
    """the cluster kernel runs the one-CTA kernel's tile arithmetic, column slice by column slice, so every output agrees bit for bit; a solve
    with keep_P = 0 gives the same dx, du, K and k bits as one with keep_P = 1"""
    data, nu, dx0 = _problem(nx, nm, 7)
    one = _solve(data, nu, dx0, "one_cta")
    clu = _solve(data, nu, dx0, "cluster")
    for key in KEYS:
        assert np.array_equal(one[key], clu[key]), (key, np.abs(one[key] - clu[key]).max())
    for variant, full in (("one_cta", one), ("cluster", clu)):
        lean = _solve(data, nu, dx0, variant, keep_P=False)
        assert "P" not in lean
        for key in ("dx", "du", "K", "k"):
            assert np.array_equal(lean[key], full[key]), (variant, key)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 2, 3])
@pytest.mark.parametrize("nx,nm", [(4, 4), (3, 3), (36, 32), (9, 17), (64, 15)], ids=lambda v: str(v))
@pytest.mark.parametrize("variant", ["cluster", "one_cta"])
def test_short_horizons(variant, nx, nm, N, restore_env):
    data, nu, dx0 = _problem(nx, nm, N, seed=N)
    sol = _solve(data, nu, dx0, variant)
    assert not sol["status"].any()
    _check(sol, _refs(data, nu, dx0), f"{variant} ({nx}, {nm}) N={N}")


@pytest.mark.gpu
@pytest.mark.parametrize("nx,nm", [(12, 12), (36, 32), (9, 17), (7, 3)], ids=lambda v: str(v))
def test_natural_dispatch_above_the_cluster_threshold(nx, nm, restore_env):
    """B = 17 takes the one-CTA kernel by itself (B * 4 * 2 > 132 SMs): it matches the reference and the forced one-CTA solve bit for bit"""
    rng = np.random.default_rng(nx * 33 + nm)
    N, Bn = 7, 17
    pattern = np.vstack([_patterns(rng, N, nm)] * 4)[:Bn - 1]
    pattern = np.vstack([pattern, rng.integers(0, nm + 1, N)])
    data, nu, dx0 = _random_batch(rng, Bn, N, nx, nm, pattern)
    sol = _solve(data, nu, dx0, "natural")
    assert not sol["status"].any()
    _check(sol, _refs(data, nu, dx0), f"natural B=17 ({nx}, {nm})")
    forced = _solve(data, nu, dx0, "one_cta")
    for key in KEYS:
        assert np.array_equal(sol[key], forced[key]), key


@pytest.mark.gpu
@pytest.mark.parametrize("reg", [0.0, 1e-6])
@pytest.mark.parametrize("nx,nm", [(4, 4), (33, 25), (52, 32), (58, 23)], ids=lambda v: str(v))
@pytest.mark.parametrize("variant", ["cluster", "one_cta"])
def test_reg_prim(variant, nx, nm, reg, restore_env):
    """reg_prim is added to P_N, Q~ and R~: both values agree with the reference at the same reg, and 1e-6 moves the solution"""
    data, nu, dx0 = _problem(nx, nm, 7, seed=2)
    sol = _solve(data, nu, dx0, variant, reg=reg)
    assert not sol["status"].any()
    _check(sol, _refs(data, nu, dx0, reg), f"{variant} ({nx}, {nm}) reg={reg}")
    if reg:
        base = _solve(data, nu, dx0, variant, reg=0.0)
        assert not np.array_equal(base["P"], sol["P"])


@pytest.mark.gpu
@pytest.mark.parametrize("nx,nm", [(6, 5), (10, 12), (9, 20), (14, 30)], ids=lambda v: str(v))
@pytest.mark.parametrize("variant", ["cluster", "one_cta"])
def test_indefinite_input_hessian_fails_only_its_instance(variant, nx, nm, restore_env):
    """an indefinite R~ at a middle stage of instance 1 (nu_max in each branch of warp_chol_inverse) sets status 1 for that instance alone; the
    others still match the reference.  A NaN in b sets status 1 too."""
    from wb_humanoid_mpc_b200.lib import B200SqpError
    from wb_humanoid_mpc_b200.qp import BatchedQp

    N = 5
    data, nu, dx0 = _problem(nx, nm, N, pattern=np.full((4, N), nm))
    data[5][1, 2] = -100.0 * np.eye(nm)
    data[2][3, 1, nx - 1] = np.nan
    sol = _solve(data, nu, dx0, variant)
    assert sol["status"].tolist() == [0, 1, 0, 1]
    refs = _refs(data, nu, dx0)
    assert refs[1] is None
    _check(sol, refs, f"{variant} ({nx}, {nm}) failed instances 1, 3", instances=[0, 2])
    _set_variant(variant)
    qp = BatchedQp(4, N, nx, nm)
    qp.upload(*data, dx0, nu)
    qp.solve()
    with pytest.raises(B200SqpError) as ei:
        qp.download()
    assert ei.value.code == lib.EQP
    qp.close()


@pytest.mark.gpu
@pytest.mark.parametrize("nx,nm", CLUSTER_TOO_BIG, ids=[f"{nx}x{nm}" for nx, nm in CLUSTER_TOO_BIG])
def test_sizes_the_cluster_kernel_cannot_hold_are_refused(nx, nm):
    from wb_humanoid_mpc_b200.lib import B200SqpError
    from wb_humanoid_mpc_b200.qp import BatchedQp

    with pytest.raises(B200SqpError) as ei:
        BatchedQp(2, 3, nx, nm)
    assert ei.value.code == lib.EINVAL, str(ei.value)
    assert "shared memory" in str(ei.value)


# ---- the whole-body instantiations at the stage edges ------------------------------------------------------------------------------------------
WB_CASES = {
    "N1": (1, lambda N: np.full((4, N), 23)),
    "N2": (2, lambda N: np.full((4, N), 23)),
    "nu0_first": (6, lambda N: np.tile(np.r_[0, np.full(N - 1, 23)], (4, 1))),
    "nu0_last": (6, lambda N: np.tile(np.r_[np.full(N - 1, 23), 0], (4, 1))),
    "nu0_all": (5, lambda N: np.zeros((4, N))),
    "mixed": (9, lambda N: np.array([[23, 0, 21, 23, 0, 22, 23, 23, 0], [0, 23, 23, 0, 0, 23, 1, 23, 23], [23] * 9, [0] * 8 + [23]])),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(WB_CASES))
def test_whole_body_sizes_at_the_stage_edges(k2_mode, case):  # noqa: F811
    """(58, 23) in its three K2 variants: the prefetch edges of riccati_wb.cuh (the deferred P store at k > 0 and k < N - 1, the helper warp
    on a stage without R~), with keep_P = 0 giving the bits of keep_P = 1"""
    N, pat = WB_CASES[case]
    data, nu, dx0 = _problem(58, 23, N, seed=7, pattern=pat(N))
    sol = _solve(data, nu, dx0)
    assert not sol["status"].any()
    _check(sol, _refs(data, nu, dx0), f"{k2_mode} (58, 23) {case}")
    lean = _solve(data, nu, dx0, keep_P=False)
    for key in ("dx", "du", "K", "k"):
        assert np.array_equal(lean[key], sol[key]), key
    if case == "nu0_all":
        assert not sol["du"].any() and not sol["K"].any() and not sol["k"].any()
