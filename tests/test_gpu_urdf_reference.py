"""The real launches against the extended-precision Lagrangian of the URDF (tests/urdf_lagrange.py): wb_torque_kernel through
b200sqp_joint_torques and cen_flow_kernel through b200sqp_centroidal_flow_map on every state recipe of test_urdf_reference.py, and the node
kernels of whole-body and centroidal handles (raw b and e of b200sqp_download_stage_blocks, which = 0) with recipe states on stance, left,
right and flight nodes.  Tolerances are those of test_urdf_reference.py; reference values are computed once per module."""
from __future__ import annotations

import numpy as np
import pytest
from mpmath import mp, mpf

import urdf_lagrange as U
import oracle_lib as orc
from test_penalty_branches import _copy, base_instance, interval_duration, stage_nodes
from test_urdf_reference import (PAYLOAD, PAYLOAD_RECIPES, cen_foot_gains, cen_state, close, foot_gains, payload_model, qddb_scale,
                                 recipes)
from wb_humanoid_mpc_b200 import abi, centroidal, model_loader
from wb_humanoid_mpc_b200.solver import joint_torques

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


@pytest.fixture(scope="module")
def cmodel():
    return model_loader.load_packaged_model("g1_centroidal")


@pytest.fixture(scope="module")
def g1():
    return U.G1.from_files()


def _values(g, model, names=None):
    out = {}
    for name, x, u in recipes(model):
        if names is None or name in names:
            d = g.dynamics(x, u)
            out[name] = dict(x=x, u=u, **{k: U.to_float(d[k]) for k in ("M", "tau", "qddb")})
    return out


@pytest.fixture(scope="module")
def ref(model, g1):
    return _values(g1, model)


@pytest.fixture(scope="module")
def payload_ref(model):
    return _values(U.G1.from_files(payloads=[PAYLOAD]), model, PAYLOAD_RECIPES)


def _tiled(ref, count):
    names = list(ref)
    idx = [names[i % len(names)] for i in range(count)]
    return idx, np.stack([ref[n]["x"] for n in idx]), np.stack([ref[n]["u"] for n in idx])


@pytest.mark.parametrize("which", ["packaged", "payload"])
def test_joint_torque_kernel_against_reference(model, ref, payload_ref, which):
    """tau and qddb of every recipe at counts 1, 127, 128, 129, 1000 (128-thread blocks: the last block partial); a sample's outputs are
    bit-identical wherever it sits in the batch"""
    m, r = (model, ref) if which == "packaged" else (payload_model(model), payload_ref)
    first = {}
    worst = {}
    for count in (1, 127, 128, 129, 1000):
        idx, x, u = _tiled(r, count)
        tau, qddb = joint_torques(m, x, u)
        for i, name in enumerate(idx):
            sc = qddb_scale(name, r[name])
            dt, okt = close(tau[i], r[name]["tau"], sc)
            dq, okq = close(qddb[i], r[name]["qddb"], sc)
            assert okt and okq, (which, count, i, name, dt, dq)
            worst[name] = max(worst.get(name, 0.0), dt, dq)
            if name in first:
                assert np.array_equal(first[name][0], tau[i]) and np.array_equal(first[name][1], qddb[i]), (which, count, i, name)
            else:
                first[name] = (tau[i].copy(), qddb[i].copy())
    print(f"wb_torque_kernel ({which}) against the reference: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))


def test_centroidal_model_shares_the_tree(model, cmodel):
    for k in ("joint_names", "parent", "joint_R", "joint_p", "joint_axis", "mass", "com", "inertia", "frame_body", "frame_p"):
        assert cmodel[k] == model[k], k


@pytest.fixture(scope="module")
def cen_ref(model, g1):
    out = {}
    for name, x, u in recipes(model):
        xc = cen_state(g1, x)
        uc = np.concatenate([u[:12], x[g1.nv + 6:]])
        out[name] = dict(x=xc, u=uc, xdot=U.to_float(g1.cen_flow_map(xc, uc)))
    return out


def test_cen_flow_kernel_against_reference(cmodel, cen_ref):
    worst = {}
    for count in (1, 33):
        names = list(cen_ref)
        idx = [names[i % len(names)] for i in range(count)]
        xd = centroidal.flow_map(cmodel, np.stack([cen_ref[n]["x"] for n in idx]), np.stack([cen_ref[n]["u"] for n in idx]), derivatives=False)
        for i, name in enumerate(idx):
            d, ok = close(xd[i], cen_ref[name]["xdot"])
            worst[name] = max(worst.get(name, 0.0), d)
            assert ok, (count, i, name, d)
    print("cen_flow_kernel against the reference: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))


@pytest.mark.parametrize("name", ["nominal", "pitch_-1.2", "rates_20", "yaw_-100"])
def test_cen_flow_kernel_jacobian_along_directions(cmodel, g1, cen_ref, name):
    """dfdx dx + dfdu du against central differences of the reference's centroidal flow map (step 1e-12 at 40 digits)"""
    r = cen_ref[name]
    _, A, B = centroidal.flow_map(cmodel, r["x"][None], r["u"][None])
    rng = np.random.default_rng(9)
    for _ in range(3):
        dx, du = rng.uniform(-1, 1, len(r["x"])), rng.uniform(-1, 1, len(r["u"]))
        with mp.workdps(g1.r.dps):
            h = g1.r.h
            sh = lambda z, d, s: [mpf(float(a)) + s * h * mpf(float(b)) for a, b in zip(z, d)]
            fp = g1.cen_flow_map(sh(r["x"], dx, 1), sh(r["u"], du, 1))
            fm = g1.cen_flow_map(sh(r["x"], dx, -1), sh(r["u"], du, -1))
            fd = U.to_float([(a - b) / (2 * h) for a, b in zip(fp, fm)])
        d, ok = close(A[0] @ dx + B[0] @ du, fd)
        assert ok, (name, d)


# ---- the node kernels of a handle: raw b and e of the first LQ approximation -----------------------------------------------------------------
# (recipe, contact flags of its node): stance, left, right and flight nodes at the extreme states
NODE_CASES = [("pitch_+1.5", (1, 1)), ("yaw_-100", (1, 0)), ("base_+1000_-1000", (0, 1)), ("below_lower", (0, 0)), ("rates_20", (1, 1)),
              ("above_upper", (1, 0))]
SWING = np.array([[0.03, 0.2, -1.0], [0.05, -0.1, 0.5]])


def _node_instance(model, states):
    """a walk instance whose stage nodes 2, 5, 8, ... carry (x, u, contact) of `states`; every such node is followed by a non-event node,
    whose state is left as built (it only enters the defect as x_next).  -> (instance, node indices)"""
    inst = _copy(base_instance(model, "walk", 0.8))
    inst["contact_flags"], inst["swing_ref"] = inst["contact_flags"].copy(), inst["swing_ref"].copy()
    st = set(stage_nodes(inst))
    nodes = [k for k in sorted(st) if k + 1 in st and k % 3 == 2][:len(states)]
    assert len(nodes) == len(states)
    for k, (x, u, contact) in zip(nodes, states):
        inst["x_init"][k], inst["u_init"][k] = x, u
        inst["contact_flags"][k] = contact
        inst["swing_ref"][k] = SWING
    return inst, nodes


def _raw_blocks(model, inst):
    from wb_humanoid_mpc_b200.solver import B200SqpSolver, stack_instances

    s = B200SqpSolver(model, abi.default_settings(model, sqp_iteration=1), capture_raw_blocks=True)
    s.upload(stack_instances([inst]))
    s.solve()
    return s.raw_stage_blocks()[0]


def test_wb_node_kernels_against_reference(model, g1, ref):
    """raw b (RK4 defect) and e (ZeroAcceleration / ZeroWrench / SwingLegVertical values) of the whole-body node kernels"""
    r = {n: (x, u) for n, x, u in recipes(model)}
    inst, nodes = _node_instance(model, [(*r[n], c) for n, c in NODE_CASES])
    raw = _raw_blocks(model, inst)
    for (name, contact), k in zip(NODE_CASES, nodes):
        x, u = r[name]
        b = U.to_float(g1.rk4_defect(x, u, inst["x_init"][k + 1], interval_duration(inst, k)))
        e = U.to_float(g1.eq_constraints(x, u, contact, SWING, foot_gains()))
        got = orc.unpack_raw_blocks(raw[k], model["nx"], model["nu"])
        sc = qddb_scale(name, {"M": ref[name]["M"]})
        db, okb = close(got["b"], b, sc)
        de, oke = close(got["e"], e, sc)
        print(f"K1 whole-body {name} {contact}: b {db:.1e}, e {de:.1e}")
        assert okb and oke, (name, k, db, de)


def test_cen_node_kernels_against_reference(model, cmodel, g1, cen_ref):
    """raw b (RK4 defect of the centroidal flow map) and e (ZeroWrench / NormalVelocity / ZeroVelocity values) of the centroidal node
    kernels"""
    inst, nodes = _node_instance(cmodel, [(cen_ref[n]["x"], cen_ref[n]["u"], c) for n, c in NODE_CASES])
    raw = _raw_blocks(cmodel, inst)
    for (name, contact), k in zip(NODE_CASES, nodes):
        x, u = cen_ref[name]["x"], cen_ref[name]["u"]
        b = U.to_float(g1.cen_rk4_defect(x, u, inst["x_init"][k + 1], interval_duration(inst, k)))
        e = U.to_float(g1.cen_eq_constraints(x, u, contact, SWING, cen_foot_gains()))
        got = orc.unpack_raw_blocks(raw[k], cmodel["nx"], cmodel["nu"])
        db, okb = close(got["b"], b)
        de, oke = close(got["e"], e)
        print(f"K1 centroidal {name} {contact}: b {db:.1e}, e {de:.1e}")
        assert okb and oke, (name, k, db, de)
