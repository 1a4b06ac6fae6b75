"""Per-instance gains (b200sqp_set_gains*) on whole-body and centroidal handles, plain and fleets: gains set to the model's values change no
bit; an instance carrying a gain set is solved bit for bit as on a handle whose model description carries that set; gains follow each
instance through the fleet's regrouping, survive resets and cold builds of the same batch size and are dropped by another size; the device
path equals the host path and reports rejected rows; the error codes."""
import numpy as np
import pytest

from test_emu_gains import ACTIVE, model_with_gains, random_gains
from test_gpu_device_io import Case
from wb_humanoid_mpc_b200 import abi
from wb_humanoid_mpc_b200.lib import B200SqpError

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

EINVAL, ESTATE = -1, -5
KEYS = ("x", "u", "K", "log", "n_iter", "status")


def solve_cycles(case, cycles=1):
    """a cold build and cycles - 1 warm builds of the case, each solved; the plan of the last one"""
    n = case.build(0.0, case.x0s)
    case.h.solve()
    for c in range(1, cycles):
        case.build(c * 0.05, None, warm=True)
        case.h.solve()
    return case.h.primal_solution(with_gains=True, raise_on_failure=False), n


def rows(sol, idx):
    return {k: np.asarray(sol[k])[idx] for k in KEYS if k in sol}


def assert_same(a, b, what=""):
    for k in a:
        assert np.array_equal(a[k], b[k], equal_nan=True), (what, k)


def gain_sets(model, n, seed):
    rng = np.random.default_rng(seed)
    return [random_gains(model, rng, [k for k in ACTIVE if rng.uniform() < 0.25] if i else []) for i in range(n)]


def stacked(gs, assign):
    return {k: np.stack([np.asarray(gs[a][k]) for a in assign]) for k in abi.GAIN_FIELDS}


FAMS = ["wb", "cen"]


@pytest.mark.parametrize("fam", FAMS)
def test_model_values_change_no_bit(fam):
    ref = Case(fam, "plain", batch=16, feedback=True)
    want, _ = solve_cycles(ref, 3)
    case = Case(fam, "plain", batch=16, feedback=True)
    case.build(0.0, case.x0s)
    case.h.set_gains(np.arange(16), case.solver.default_gains())
    g = case.h.gains()
    assert g["custom"].all()
    got, _ = solve_cycles(case, 3)
    assert_same(rows(want, slice(None)), rows(got, slice(None)))


@pytest.mark.parametrize("fam,batch,nsets,iters", [("wb", 8, 8, 1), ("cen", 8, 8, 1), ("wb", 256, 4, 1), ("wb", 256, 4, 4)])
def test_each_instance_solves_as_the_model_carrying_its_gains(fam, batch, nsets, iters):
    model = Case(fam, "plain", batch=1).model
    gs = gain_sets(model, nsets, seed=batch + iters)
    assign = np.arange(batch) % nsets
    case = Case(fam, "plain", batch=batch, feedback=True)
    case.solver = type(case.solver)(case.model, abi.default_settings(case.model, sqp_iteration=iters, use_feedback_policy=1))
    case.h = case.solver
    case.build(0.0, case.x0s)
    case.h.set_gains(np.arange(batch), stacked(gs, assign))
    got, _ = solve_cycles(case, 2)
    back = case.h.gains()
    for s in range(nsets):
        ref = Case(fam, "plain", batch=batch, feedback=True)
        ref.model = model_with_gains(model, gs[s])
        ref.solver = type(case.solver)(ref.model, abi.default_settings(ref.model, sqp_iteration=iters, use_feedback_policy=1))
        ref.h = ref.solver
        want, _ = solve_cycles(ref, 2)
        idx = np.flatnonzero(assign == s)
        assert_same(rows(want, idx), rows(got, idx), f"set {s}")
        for k in abi.GAIN_FIELDS:
            assert np.array_equal(back[k][idx], np.broadcast_to(gs[s][k], back[k][idx].shape)), k


@pytest.mark.parametrize("fam", FAMS)
def test_fleet_gains_follow_their_instances(fam):
    B, nsets = 24, 4
    model = Case(fam, "fleet", batch=1).model
    gs = gain_sets(model, nsets, seed=5)
    assign = np.arange(B) % nsets
    case = Case(fam, "fleet", batch=B, feedback=True)
    case.build(0.0, case.x0s)
    case.h.set_gains(np.arange(B), stacked(gs, assign))
    got, _ = solve_cycles(case, 6)
    case.check_groups()
    back = case.h.gains()
    assert back["custom"].all()
    for k in abi.GAIN_FIELDS:
        assert np.array_equal(back[k], stacked(gs, assign)[k]), k
    for s in range(nsets):
        ref = Case(fam, "fleet", batch=B, feedback=True)
        ref.h.close()
        ref.model = model_with_gains(model, gs[s])
        from wb_humanoid_mpc_b200.solver import B200SqpFleet, B200SqpSolver

        ref.solver = B200SqpSolver(ref.model, abi.default_settings(ref.model, sqp_iteration=1, use_feedback_policy=1))
        ref.h = B200SqpFleet(ref.solver)
        want, _ = solve_cycles(ref, 6)
        idx = np.flatnonzero(assign == s)
        assert_same(rows(want, idx), rows(got, idx), f"set {s}")


def test_lifetimes():
    B = 8
    case = Case("wb", "plain", batch=B, feedback=True)
    case.solver.set_gait_schedule(True)
    case.build(0.0, case.x0s)
    gs = gain_sets(case.model, 2, seed=9)
    case.h.set_gains([1, 5], stacked(gs, [0, 1]))
    before = case.h.gains()
    assert before["custom"].tolist() == [0, 1, 0, 0, 0, 1, 0, 0]
    case.h.solve()
    case.solver.set_reset_states(case.x0s, case.gaits)
    case.h.request_resets(np.arange(B))   # (every instance: a plain handle needs one node count, and a reset restarts the schedule)
    case.build(0.05, None, warm=True)
    case.h.solve()
    assert case.solver.episodes()["reset"].all()
    after = case.h.gains()
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    case.build(0.0, case.x0s)   # a cold build of the same size keeps them
    after = case.h.gains()
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    # set_gains(idx, None) restores the model's values bit for bit
    ref = Case("wb", "plain", batch=B, feedback=True)
    want, _ = solve_cycles(ref, 2)
    case.h.set_gains([1, 5], None)
    assert not case.h.gains()["custom"].any()
    fresh = Case("wb", "plain", batch=B, feedback=True)
    fresh.build(0.0, fresh.x0s)
    fresh.h.set_gains([1, 5], stacked(gs, [0, 1]))
    fresh.h.set_gains([1, 5], None)
    got, _ = solve_cycles(fresh, 2)
    assert_same(rows(want, slice(None)), rows(got, slice(None)))
    # another batch size drops every gain set
    fresh.h.set_gains([3], gs[0])
    other = Case("wb", "plain", batch=B // 2, feedback=True)
    fresh.h.build_instances(0.0, fresh.horizon, other.x0s, other.gaits, other.starts, other.cmds)
    g = fresh.h.gains()
    assert g["custom"].shape == (B // 2,) and not g["custom"].any()


@pytest.mark.parametrize("kind", ["plain", "fleet"])
def test_device_path_equals_the_host_path(kind):
    B = 16
    model = Case("wb", kind, batch=1).model
    gs = gain_sets(model, 4, seed=13)
    assign = np.arange(B) % 4
    host = Case("wb", kind, batch=B, feedback=True)
    host.build(0.0, host.x0s)
    host.h.set_gains(np.arange(B), stacked(gs, assign))
    want, _ = solve_cycles(host, 3)
    dev = Case("wb", kind, batch=B, feedback=True)
    dev.build(0.0, dev.x0s)
    packed = abi.pack_gains(stacked(gs, assign))
    t = torch.zeros(packed.shape, dtype=torch.uint8, device="cuda")
    t.add_(torch.from_numpy(packed).cuda())   # written by a torch kernel on the current stream, read by the call on the same stream
    st = dev.h.set_gains_device(np.arange(B), t)
    got, _ = solve_cycles(dev, 3)
    assert st.cpu().tolist() == [0] * B
    assert_same(rows(want, slice(None)), rows(got, slice(None)))
    # rejected rows: status 1 / 2, those instances unchanged
    bad = stacked(gs, [0, 1, 2])
    bad["R_diag"][0][0] = 0.0
    bad["jlim_mu"][1] = np.nan
    before = dev.h.gains()
    st = dev.h.set_gains_device([4, 5, 6], torch.from_numpy(abi.pack_gains(bad)).cuda())
    assert st.cpu().tolist() == [2, 1, 0]
    after = dev.h.gains()
    for k in abi.GAIN_FIELDS:
        assert np.array_equal(after[k][[4, 5]], before[k][[4, 5]]), k
        assert np.array_equal(after[k][6], np.asarray(gs[2][k])), k


def test_error_codes():
    from wb_humanoid_mpc_b200.solver import B200SqpFleet, B200SqpSolver

    case = Case("wb", "plain", batch=4)
    d = case.solver.default_gains()
    with pytest.raises(B200SqpError) as e:
        case.h.set_gains([0], d)   # no batch yet
    assert e.value.code == ESTATE
    with pytest.raises(B200SqpError) as e:
        case.h.gains()
    assert e.value.code == ESTATE
    case.build(0.0, case.x0s)
    for idx, g in (([4], d), ([-1], d), ([1, 1], None)):
        with pytest.raises(B200SqpError) as e:
            case.h.set_gains(idx, g)
        assert e.value.code == EINVAL
    for k, v in (("R_diag", 0.0), ("Q_diag", -1.0), ("fric_delta", 0.0), ("coll_mu", np.inf), ("final_cost_active", 2)):
        bad = {kk: np.array(vv, copy=True) for kk, vv in d.items()}
        if bad[k].ndim:
            bad[k][0] = v
        else:
            bad[k] = np.array(v)
        with pytest.raises(B200SqpError) as e:
            case.h.set_gains([0], bad)
        assert e.value.code == EINVAL, k
    assert not case.h.gains()["custom"].any()   # nothing was applied
    with pytest.raises(B200SqpError) as e:
        case.h.set_gains_device([9], torch.from_numpy(abi.pack_gains(d, 1)).cuda())
    assert e.value.code == EINVAL
    s = B200SqpSolver(case.model, abi.default_settings(case.model, sqp_iteration=1))
    s._ensure_builder()
    s.build_instances(0.0, case.horizon, case.x0s, case.gaits, case.starts, case.cmds)
    fl = B200SqpFleet(s)
    with pytest.raises(B200SqpError) as e:
        s.set_gains([0], d)   # the handle entry points while a fleet is attached
    assert e.value.code == ESTATE
    with pytest.raises(B200SqpError) as e:
        s.gains()
    assert e.value.code == ESTATE
    fl.close()
