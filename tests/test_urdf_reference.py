"""The G1 model description, the CPU oracle and the kernels' arithmetic against an extended-precision Lagrangian of the URDF itself.

tests/urdf_lagrange.py restates the reference's dynamics from the URDF semantics Pinocchio implements, link by link and without welding, in
mpmath at 40 digits.  A model description that is wrong but self-consistent (a mis-composed rpy, a fold that loses a rotation, an axis in
the wrong frame) passes the identity and finite-difference tests of test_oracle_wb.py; it does not pass these.

Tolerance: |got - ref| <= 1e-11 max(1, |ref|_inf) per quantity; on the recipes near the ZYX singularity the base-acceleration bound is
multiplied by cond(M_bb_ang), the 3x3 block computeBaseAcceleration inverts.  The largest measured differences are printed per recipe.
"""
from __future__ import annotations

import numpy as np
import pytest
from mpmath import mp, mpf

import emu_lib as emu
import oracle_lib as orc
import urdf_lagrange as U
from test_oracle_wb import rand_input, rand_state
from wb_humanoid_mpc_b200 import model_loader, references

TOL = 1e-11


@pytest.fixture(scope="module")
def model():
    return model_loader.load_packaged_model()


@pytest.fixture(scope="module")
def cmodel():
    return model_loader.load_packaged_model("g1_centroidal")


@pytest.fixture(scope="module")
def wb(model):
    return orc.WbOracle(model)


@pytest.fixture(scope="module")
def g1():
    return U.G1.from_files()


def close(got, ref, scale=1.0):
    """max |got - ref| / max(1, |ref|_inf) and whether it is within TOL * scale"""
    got, ref = np.asarray(got, float), np.asarray(ref, float)
    d = float(np.max(np.abs(got - ref)) / max(1.0, np.max(np.abs(ref)))) if ref.size else 0.0
    return d, d <= TOL * scale


# ---- states ------------------------------------------------------------------------------------------------------------------------
def recipes(model):
    """[(name, x, u, property it is named for)] of the whole-body state / input layout"""
    nj, nv = model["nj"], 6 + model["nj"]
    mg = sum(model["mass"]) * 9.81
    x0 = np.array(model["x_init"], float)
    x0[2] = model["reference"]["defaultBaseHeight"]
    wc2, wc1 = references.weight_compensating_input(model, (1, 1)), references.weight_compensating_input(model, (1, 0))
    lo, hi = np.array(model["q_lower"]), np.array(model["q_upper"])
    out = [("nominal", x0, wc2, lambda x, u: np.all(x[nv:] == 0) and abs(u[2] + u[8] - mg) < 1e-9)]

    def rnd(seed, scale=1.0):
        rng = np.random.default_rng(seed)
        return rand_state(model, rng, scale), rand_input(model, rng)

    x, u = rnd(11)
    out.append(("random_1x", x, u, lambda x, u: np.any(x[nv:] != 0)))
    x, u = rnd(12, 3.0)
    out.append(("random_3x", x, u, lambda x, u: np.max(np.abs(x[nv:])) > 0.5))
    for i, (label, val) in enumerate([("pitch", 1.2), ("pitch", -1.2), ("pitch", 1.5), ("pitch", -1.5), ("pitch", 1.5707), ("roll", 1.0),
                                      ("roll", -1.0), ("yaw", np.pi), ("yaw", -np.pi), ("yaw", 40.0), ("yaw", -100.0)]):
        x, u = rnd(20 + i)
        k = {"yaw": 3, "pitch": 4, "roll": 5}[label]
        x[k] = val
        out.append((f"{label}_{val:+g}", x, u, lambda x, u, k=k, val=val: x[k] == val))
    for i, (px, py) in enumerate([(1e3, -1e3), (-1e3, 1e3)]):
        x, u = rnd(40 + i)
        x[0:3] = [px, py, 0.8]
        out.append((f"base_{px:+g}_{py:+g}", x, u, lambda x, u, p=(px, py): tuple(x[0:2]) == p))
    for i, (label, q) in enumerate([("q_lower", lo), ("q_upper", hi), ("below_lower", lo - 0.2), ("above_upper", hi + 0.2)]):
        x, u = rnd(50 + i)
        x[6:nv] = q
        out.append((label, x, u, lambda x, u, q=q: np.array_equal(x[6:nv], q)))
    x, u = rnd(60)
    x[nv + 6:] = 20.0 * np.where(np.arange(nj) % 2 == 0, 1.0, -1.0)
    x[nv + 3:nv + 6] = [5.0, -5.0, 5.0]
    out.append(("rates_20", x, u, lambda x, u: np.max(np.abs(x[nv + 6:])) == 20.0 and np.max(np.abs(x[nv + 3:nv + 6])) == 5.0))
    x, u = rnd(61)
    u[:12] = 0.0
    out.append(("flight", x, u, lambda x, u: not np.any(u[:12])))
    x, u = rnd(62)
    u[:12] = wc2[:12]
    out.append(("double_support", x, u, lambda x, u: abs(u[2] - u[8]) < 1e-9 and abs(u[2] + u[8] - mg) < 1e-9))
    x, u = rnd(63)
    u[:12] = wc1[:12]
    out.append(("single_support", x, u, lambda x, u: abs(u[2] - mg) < 1e-9 and not np.any(u[6:12])))
    x, u = rnd(64)
    u[:12] = 0.0
    u[2], u[8] = 1.5 * mg, 1.5 * mg
    u[0], u[7] = 0.3 * mg, -0.2 * mg
    u[3:6], u[9:12] = [50.0, -50.0, 50.0], [-50.0, 50.0, -50.0]
    out.append(("wrench_3x_torque_50", x, u, lambda x, u: abs(u[2] + u[8] - 3 * mg) < 1e-9 and np.max(np.abs(u[3:6])) == 50.0))
    for name, x, u, prop in out:
        assert prop(x, u), name
    return [(n, x, u) for n, x, u, _ in out]


def cen_state(g1, x):
    """centroidal (x, u) of a whole-body state: normalized momentum h/m of the reference's A_g at (q, qd)"""
    nv = g1.nv
    A, _ = g1.centroidal_map(x[:nv])
    with mp.workdps(g1.r.dps):
        h = [sum(a * mpf(float(v)) for a, v in zip(row, x[nv:])) / g1.r.total_mass for row in A]
    return np.concatenate([U.to_float(h), x[:nv]])


# ---- reference values, once per module ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref(model, g1):
    out = {}
    for name, x, u in recipes(model):
        d = g1.dynamics(x, u)
        feet = g1.foot_state(x, d["xdot"][g1.nv:])
        A, G = g1.centroidal_map(x[:g1.nv])
        xc = cen_state(g1, x)
        uc = np.concatenate([u[:12], x[g1.nv + 6:]])
        out[name] = dict(x=x, u=u, xc=xc, uc=uc, Ag=U.to_float(A), com=U.to_float(G), cen_xdot=U.to_float(g1.cen_flow_map(xc, uc)),
                         feet=[U.to_float(f) for f in feet], **{k: U.to_float(v) for k, v in d.items()})
    return out


# a 3 kg box with off-diagonal inertia on the torso (body 15, child of waist_pitch_joint)
PAYLOAD = (15, 3.0, [0.1, -0.05, 0.3], [[0.02, 0.003, -0.001], [0.003, 0.03, 0.002], [-0.001, 0.002, 0.04]])
PAYLOAD_RECIPES = ("random_1x", "pitch_-1.2", "wrench_3x_torque_50")


def payload_model(model):
    """the model description of a payload record: add_payload (the loader's composite arithmetic) -> with_robot_params"""
    nb = model["nj"] + 1
    params = dict(mass=np.array(model["mass"]), com=np.array(model["com"]), inertia=np.array(model["inertia"]).reshape(nb, 9))
    return model_loader.with_robot_params(model, model_loader.add_payload(params, *PAYLOAD))


@pytest.fixture(scope="module")
def payload_ref(model):
    """reference values of the payload robot: the box as an extra fixed link of the URDF tree"""
    g = U.G1.from_files(payloads=[PAYLOAD])
    out = {}
    for name, x, u in recipes(model):
        if name in PAYLOAD_RECIPES:
            d = g.dynamics(x, u)
            out[name] = dict(x=x, u=u, **{k: U.to_float(v) for k, v in d.items()})
    return out


def cond_ang(r):
    return float(np.linalg.cond(r["M"][3:6, 3:6]))


def qddb_scale(name, r):
    """near the ZYX singularity the base-acceleration bound is cond(M_bb_ang) * 1e-15 (about 4.5 float64 epsilons per unit of condition)
    where that exceeds TOL: 3e-6 at pitch 1.5707 (cond 3.1e9, measured 1.7e-7); every other recipe keeps TOL"""
    return max(1.0, cond_ang(r) * 1e-15 / TOL) if name.startswith("pitch") else 1.0


# ---- 1. known answers for the reference itself -------------------------------------------------------------------------------------
def _link(name, m, xyz="0 0 0", rpy="0 0 0", I=(0.01, 0, 0, 0.01, 0, 0.01)):
    ixx, ixy, ixz, iyy, iyz, izz = I
    return (f'<link name="{name}"><inertial><origin xyz="{xyz}" rpy="{rpy}"/><mass value="{m}"/>'
            f'<inertia ixx="{ixx}" ixy="{ixy}" ixz="{ixz}" iyy="{iyy}" iyz="{iyz}" izz="{izz}"/></inertial></link>')


def _joint(name, parent, child, kind="revolute", xyz="0 0 0", rpy="0 0 0", axis="0 1 0"):
    return (f'<joint name="{name}" type="{kind}"><origin xyz="{xyz}" rpy="{rpy}"/><parent link="{parent}"/><child link="{child}"/>'
            f'<axis xyz="{axis}"/></joint>')


def _robot(*parts):
    return '<robot name="t">' + "".join(parts) + "</robot>"


def _mpv(v):
    return [mpf(repr(float(a))) for a in v]


def test_reference_double_pendulum_closed_form():
    """a planar double pendulum about y: the joint block of M and nle (base at rest) is the textbook M, C qd and g"""
    m1, m2, l1, c1, c2, I1, I2 = 1.3, 0.7, 0.5, 0.2, 0.3, 0.02, 0.011
    txt = _robot(_link("base", 5.0), _link("l1", m1, f"0 0 {-c1}", I=(0.05, 0, 0, I1, 0, 0.03)), _link("l2", m2, f"0 0 {-c2}", I=(0.04, 0, 0, I2, 0, 0.02)),
                 _joint("j1", "base", "l1"), _joint("j2", "l1", "l2", xyz=f"0 0 {-l1}"))
    r = U.Robot(txt, ["j1", "j2"])
    rng = np.random.default_rng(0)
    for _ in range(3):
        th, thd = rng.uniform(-2, 2, 2), rng.uniform(-3, 3, 2)
        q = np.concatenate([rng.uniform(-1, 1, 3), [0, 0, 0], th])
        qd = np.concatenate([np.zeros(6), thd])
        with mp.workdps(r.dps):
            M = U.to_float(r.mass_matrix(_mpv(q)))[6:, 6:]
            nle = U.to_float(r.nle(_mpv(q), _mpv(qd)))[6:]
        c, s, g = np.cos(th[1]), np.sin(th[1]), 9.81
        M_ref = np.array([[I1 + I2 + m1 * c1 ** 2 + m2 * (l1 ** 2 + c2 ** 2 + 2 * l1 * c2 * c), I2 + m2 * (c2 ** 2 + l1 * c2 * c)],
                          [I2 + m2 * (c2 ** 2 + l1 * c2 * c), I2 + m2 * c2 ** 2]])
        hh = m2 * l1 * c2 * s
        Cqd = np.array([-hh * (2 * thd[0] * thd[1] + thd[1] ** 2), hh * thd[0] ** 2])
        grav = np.array([(m1 * c1 + m2 * l1) * g * np.sin(th[0]) + m2 * c2 * g * np.sin(th.sum()), m2 * c2 * g * np.sin(th.sum())])
        assert np.allclose(M, M_ref, rtol=0, atol=1e-14)
        assert np.allclose(nle, Cqd + grav, rtol=0, atol=1e-13)


def test_reference_floating_body_zyx_rate_map():
    """one free body with off-diagonal inertia and an inertial rpy: M = diag(m 1, E' R I R' E) with E the ZYX rate map, and
    nle = (0, 0, m g, ...) at rest"""
    m, I, rpy = 2.5, np.array([[0.3, 0.02, -0.01], [0.02, 0.2, 0.03], [-0.01, 0.03, 0.1]]), (0.3, -0.4, 1.1)
    txt = _robot(_link("b", m, "0 0 0", " ".join(map(str, rpy)), I=(I[0, 0], I[0, 1], I[0, 2], I[1, 1], I[1, 2], I[2, 2])))
    r = U.Robot(txt, [])
    z, y, x = 0.7, -0.9, 0.4
    q = [1.0, -2.0, 3.0, z, y, x]

    def rx(a):
        return np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])

    def ry(a):
        return np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])

    def rz(a):
        return np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])

    Rb, Rin = rz(z) @ ry(y) @ rx(x), rz(rpy[2]) @ ry(rpy[1]) @ rx(rpy[0])
    E = np.column_stack([[0, 0, 1], rz(z) @ [0, 1, 0], rz(z) @ ry(y) @ [1, 0, 0]])
    Iw = Rb @ Rin @ I @ Rin.T @ Rb.T
    with mp.workdps(r.dps):
        M = U.to_float(r.mass_matrix(_mpv(q)))
        nle = U.to_float(r.nle(_mpv(q), _mpv(np.zeros(6))))
    assert np.allclose(M[:3, :3], m * np.eye(3), atol=1e-15) and np.allclose(M[:3, 3:], 0, atol=1e-15)
    assert np.allclose(M[3:, 3:], E.T @ Iw @ E, rtol=0, atol=1e-14)
    assert np.allclose(nle, [0, 0, m * 9.81, 0, 0, 0], atol=1e-13)


def test_reference_fixed_link_equals_link_merged_by_hand():
    """a massive link behind a fixed joint with a three-angle rpy and its own inertial rpy == one link carrying the composite inertia"""
    m1, m2 = 1.7, 0.9
    I1, I2 = np.diag([0.03, 0.02, 0.01]), np.array([[0.02, 0.004, -0.002], [0.004, 0.015, 0.001], [-0.002, 0.001, 0.01]])
    c1, c2 = np.array([0.01, -0.02, 0.05]), np.array([0.03, 0.01, -0.04])
    jp, jrpy, irpy = np.array([0.1, -0.05, 0.2]), (0.27931, 5.4949e-05, -0.00019159), (0.4, -0.3, 0.2)

    def R(rpy):
        r, p, y = rpy
        rx = np.array([[1, 0, 0], [0, np.cos(r), -np.sin(r)], [0, np.sin(r), np.cos(r)]])
        ry = np.array([[np.cos(p), 0, np.sin(p)], [0, 1, 0], [-np.sin(p), 0, np.cos(p)]])
        rz = np.array([[np.cos(y), -np.sin(y), 0], [np.sin(y), np.cos(y), 0], [0, 0, 1]])
        return rz @ ry @ rx

    s = lambda v: " ".join(repr(float(a)) for a in v)
    sixI = lambda I: (I[0, 0], I[0, 1], I[0, 2], I[1, 1], I[1, 2], I[2, 2])
    leg = [_link("leg", 0.8, "0 0 -0.2"), _joint("hip", "pelvis", "leg", xyz="0 0.1 -0.1", axis="1 0 0")]
    welded = _robot(_link("pelvis", m1, s(c1), I=sixI(I1)), _link("box", m2, s(c2), s(irpy), I=sixI(I2)),
                    _joint("weld", "pelvis", "box", "fixed", s(jp), s(jrpy)), *leg)
    Rj = R(jrpy)
    c2p, I2p = Rj @ c2 + jp, Rj @ R(irpy) @ I2 @ R(irpy).T @ Rj.T
    m = m1 + m2
    c = (m1 * c1 + m2 * c2p) / m
    shift = lambda I, mm, d: I + mm * (d @ d * np.eye(3) - np.outer(d, d))
    Ic = shift(I1, m1, c1 - c) + shift(I2p, m2, c2p - c)
    merged = _robot(_link("pelvis", m, s(c), I=sixI(Ic)), *leg)
    rng = np.random.default_rng(1)
    q, qd = rng.uniform(-1, 1, 7), rng.uniform(-2, 2, 7)
    out = []
    for txt in (welded, merged):
        r = U.Robot(txt, ["hip"])
        with mp.workdps(r.dps):
            out.append((U.to_float(r.mass_matrix(_mpv(q))), U.to_float(r.nle(_mpv(q), _mpv(qd)))))
    assert np.allclose(out[0][0], out[1][0], rtol=0, atol=1e-14)
    assert np.allclose(out[0][1], out[1][1], rtol=0, atol=1e-13)


def test_reference_unaligned_non_unit_axis():
    """a revolute axis (1, 2, 2) (norm 3) behind a rotated joint origin: the joint's M entry is a' I a + m |a x r|^2 about the unit axis
    in the joint frame, and the non-unit axis describes the same robot as its normalised copy"""
    m, c, I = 1.1, np.array([0.2, -0.1, 0.3]), np.array([[0.03, 0.001, 0.002], [0.001, 0.02, -0.003], [0.002, -0.003, 0.01]])
    s = lambda v: " ".join(repr(float(a)) for a in v)
    six = (I[0, 0], I[0, 1], I[0, 2], I[1, 1], I[1, 2], I[2, 2])
    out = []
    for axis in ("1 2 2", s(np.array([1, 2, 2]) / 3.0)):
        txt = _robot(_link("b", 3.0), _link("l", m, s(c), I=six), _joint("j", "b", "l", xyz="0.1 0.2 0.3", rpy="0.5 -0.2 0.9", axis=axis))
        r = U.Robot(txt, ["j"])
        q = [0.3, 0.1, -0.2, 0.4, 0.2, -0.3, 0.8]
        with mp.workdps(r.dps):
            out.append(U.to_float(r.mass_matrix(_mpv(q))))
    a = np.array([1, 2, 2]) / 3.0
    assert abs(out[0][6, 6] - (a @ I @ a + m * np.sum(np.cross(a, c) ** 2))) < 1e-14
    assert np.allclose(out[0], out[1], rtol=0, atol=1e-14)


def test_reference_error_at_two_precisions(model, g1):
    """the reference shows its own error: (40 digits, h = 1e-12) and (50 digits, h = 1e-15) agree to 1e-18 relative"""
    g2 = g1.at(*U.SECONDARY)
    for name, x, u in [r for r in recipes(model) if r[0] in ("random_3x", "pitch_+1.5")]:
        a, b = g1.dynamics(x, u), g2.dynamics(x, u)
        for key in ("nle", "qddb", "tau"):
            with mp.workdps(60):
                d = max(abs(p - q) for p, q in zip(a[key], b[key])) / max(1, max(abs(p) for p in b[key]))
            assert d <= 1e-18, (name, key, d)
        fa, fb = g1.foot_state(x, U.to_float(a["xdot"])[g1.nv:]), g2.foot_state(x, U.to_float(a["xdot"])[g1.nv:])
        for c in range(2):
            for key in ("alin", "aang"):
                with mp.workdps(60):
                    d = max(abs(p - q) for p, q in zip(fa[c][key], fb[c][key])) / max(1, max(abs(p) for p in fb[c][key]))
                assert d <= 1e-18, (name, c, key, d)


# ---- 2. the model description and the oracle against the reference -----------------------------------------------------------------
def test_joint_order_and_total_mass(model, g1):
    names, fixed = U.g1_joint_order()
    assert model["joint_names"] == names and len(fixed) == 6
    assert abs(sum(model["mass"]) - float(g1.r.total_mass)) < 1e-12


def test_oracle_against_reference(model, wb, ref):
    worst = {}
    for name, r in ref.items():
        x, u, nv = r["x"], r["u"], wb.nj + 6
        M, nle = wb.crba_nle(x)
        tau, qddb = wb.joint_torques(x, u)
        a = np.random.default_rng(7).uniform(-3, 3, nv)
        feet, _ = wb.foot_state(x, u)
        Ag, com = wb.centroidal_map(x[:nv])
        sc = qddb_scale(name, r)
        checks = dict(M=close(M, r["M"]), nle=close(nle, r["nle"]), rnea=close(wb.rnea(x[:nv], x[nv:], a), r["M"] @ a + r["nle"]),
                      flow=close(wb.flow_map(x, u), r["xdot"], sc), tau=close(tau, r["tau"], sc), qddb=close(qddb, r["qddb"], sc),
                      Ag=close(Ag, r["Ag"]), com=close(com, r["com"]), cen_flow=close(wb.cen_flow_map(r["xc"], r["uc"]), r["cen_xdot"]))
        for c in range(2):
            for key in ("pos", "R", "oriErr", "vlin", "vang"):
                checks[f"{key}{c}"] = close(feet[c][key], r["feet"][c][key])
            for key in ("alin", "aang"):
                checks[f"{key}{c}"] = close(feet[c][key], r["feet"][c][key], sc)
        worst[name] = max(d for d, _ in checks.values())
        bad = {k: d for k, (d, ok) in checks.items() if not ok}
        assert not bad, (name, bad, cond_ang(r))
    print("oracle against the reference, largest difference per recipe: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))


def test_payload_model_against_reference(model, payload_ref):
    pm = payload_model(model)
    assert abs(sum(pm["mass"]) - sum(model["mass"]) - PAYLOAD[1]) < 1e-12
    o = orc.WbOracle(pm)
    for name, r in payload_ref.items():
        M, nle = o.crba_nle(r["x"])
        tau, qddb = o.joint_torques(r["x"], r["u"])
        sc = qddb_scale(name, r)
        checks = dict(M=close(M, r["M"]), nle=close(nle, r["nle"]), tau=close(tau, r["tau"], sc), qddb=close(qddb, r["qddb"], sc))
        tau_h, qddb_h = emu.joint_torques(o.desc, r["x"], r["u"])
        checks.update(tau_harness=close(tau_h, r["tau"], sc), qddb_harness=close(qddb_h, r["qddb"], sc))
        assert all(ok for _, ok in checks.values()), (name, checks)
        print(f"payload {name}: " + ", ".join(f"{k} {d:.1e}" for k, (d, _) in checks.items()))


def test_loader_fold_of_rotated_welded_links(model, tmp_path):
    """The G1's rotated welded links (d435, pitch 0.83 rad; mid360) carry no mass, so the packaged model cannot show whether the loader
    rotates a welded link's inertia.  This variant of the URDF gives d435_link an inertia with off-diagonal terms and an inertial rpy, and
    welds the left rubber hand behind a three-angle rpy; the loader's model of it must match the reference, which never welds."""
    text = U.G1_URDF.read_text()
    text = text.replace('<link name="d435_link"></link>', '<link name="d435_link"><inertial><origin xyz="0.02 -0.01 0.03" rpy="0.3 -0.5 0.7"/>'
                        '<mass value="0.4"/><inertia ixx="0.004" ixy="0.0005" ixz="-0.0003" iyy="0.002" iyz="0.0002" izz="0.001"/></inertial></link>')
    a = '<origin xyz="0.0415 0.003 0" rpy="0 0 0"/>\n    <parent link="left_wrist_yaw_link"/>'
    assert text.count(a) == 1 and text.count('<link name="d435_link"><inertial>') == 1
    text = text.replace(a, a.replace('rpy="0 0 0"', 'rpy="0.4 -0.3 0.6"'))
    urdf = tmp_path / "g1_variant.urdf"
    urdf.write_text(text)
    vm = model_loader.build_wb_model(urdf, U.G1_WB_TASK, U.G1_WB_REFERENCE)
    assert abs(sum(vm["mass"]) - sum(model["mass"]) - 0.4) < 1e-12
    names, _ = U.g1_joint_order()
    t = model_loader.parse_info(U.G1_WB_TASK)["contacts"]["contact_frame_translation"]
    g = U.G1(U.Robot(text, names, {"foot_l_contact": ("left_ankle_roll_link", [t[a] for a in "xyz"]),
                                   "foot_r_contact": ("right_ankle_roll_link", [t[a] for a in "xyz"])}))
    o = orc.WbOracle(vm)
    name, x, u = [r for r in recipes(model) if r[0] == "random_3x"][0]
    d = g.dynamics(x, u)
    M, nle = o.crba_nle(x)
    tau, qddb = o.joint_torques(x, u)
    checks = dict(M=close(M, U.to_float(d["M"])), nle=close(nle, U.to_float(d["nle"])), tau=close(tau, U.to_float(d["tau"])),
                  qddb=close(qddb, U.to_float(d["qddb"])))
    assert all(ok for _, ok in checks.values()), checks


def test_srbd_nominal_against_reference(model, g1):
    """model_loader.srbd_nominal (ccrba at (0_6, nominal joint angles)) against the reference's composite inertia of all URDF links"""
    qj = model["reference"]["defaultJointState"]
    got = model_loader.srbd_nominal(model, qj)
    with mp.workdps(g1.r.dps):
        Ig, G = g1.r.composite_inertia(_mpv(np.concatenate([np.zeros(6), qj])))
    assert close(got["inertia"], U.to_float(Ig))[1] and close(got["com_to_base"], -U.to_float(G))[1]


# ---- 3. the kernels' arithmetic on the CPU harness ---------------------------------------------------------------------------------
def test_harness_dyn_and_joint_torques_against_reference(wb, ref):
    worst = {}
    for name, r in ref.items():
        sc = qddb_scale(name, r)
        xd, _ = emu.dyn(wb.desc, r["x"], r["u"], False)
        tau, qddb = emu.joint_torques(wb.desc, r["x"], r["u"])
        checks = dict(flow=close(xd, r["xdot"], sc), tau=close(tau, r["tau"], sc), qddb=close(qddb, r["qddb"], sc))
        worst[name] = max(d for d, _ in checks.values())
        assert all(ok for _, ok in checks.values()), (name, checks)
    print("CPU harness against the reference: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))


@pytest.mark.parametrize("name", ["random_1x", "pitch_-1.2", "rates_20"])
def test_harness_dyn_jacobian_along_directions(model, wb, g1, ref, name):
    """the six dense rows of the flow-map Jacobian (d qddb / d(x, u)) along random directions against central differences of the
    reference in mpmath (step 1e-12 at 40 digits)"""
    r = ref[name]
    z0 = np.concatenate([r["x"], r["u"]])
    _, G = emu.dyn(wb.desc, r["x"], r["u"], True)
    rng = np.random.default_rng(3)
    nx = model["nx"]
    for _ in range(2):
        d = rng.uniform(-1, 1, len(z0))
        with mp.workdps(g1.r.dps):
            h = g1.r.h
            zp = [mpf(float(a)) + h * mpf(float(b)) for a, b in zip(z0, d)]
            zm = [mpf(float(a)) - h * mpf(float(b)) for a, b in zip(z0, d)]
            fp, fm = g1.dynamics(zp[:nx], zp[nx:])["qddb"], g1.dynamics(zm[:nx], zm[nx:])["qddb"]
            dd = U.to_float([(a - b) / (2 * h) for a, b in zip(fp, fm)])
        dist, ok = close(G @ d, dd, qddb_scale(name, r))
        assert ok, (name, dist)


GAINS = None


def foot_gains():
    global GAINS
    if GAINS is None:
        from wb_humanoid_mpc_b200.model_loader import parse_info

        GAINS = parse_info(U.G1_WB_TASK)["model_settings"]["foot_constraint"]
    return GAINS


LQ_CASES = [("nominal", (1, 1)), ("pitch_+1.5", (1, 0)), ("rates_20", (0, 1)), ("flight", (0, 0))]


@pytest.fixture(scope="module")
def lq_ref(ref, g1):
    """RK4 defect and equality-constraint values of the reference for the LQ_CASES nodes"""
    out = {}
    swing = np.array([[0.03, 0.2, -1.0], [0.05, -0.1, 0.5]])
    for name, contact in LQ_CASES:
        r = ref[name]
        xn = r["x"] + np.random.default_rng(5).uniform(-0.01, 0.01, len(r["x"]))
        out[name] = dict(xn=xn, swing=swing, contact=contact, dt=0.015,
                         b=U.to_float(g1.rk4_defect(r["x"], r["u"], xn, 0.015)),
                         e=U.to_float(g1.eq_constraints(r["x"], r["u"], contact, swing, foot_gains())))
    return out


def test_harness_lq_node_defect_and_constraints(model, wb, ref, lq_ref):
    """lq_node raw b (RK4 defect from four flow-map evaluations) and raw e (ZeroAcceleration / ZeroWrench / SwingLegVertical values)"""
    xref = np.array(model["x_init"], float)
    for name, contact in LQ_CASES:
        r, L = ref[name], lq_ref[name]
        sc = qddb_scale(name, r)
        e = emu.lq_node(wb.desc, r["x"], r["u"], L["xn"], xref, L["dt"], contact, L["swing"], [1.0, 1.0], 0.0)["raw"]
        db, okb = close(e["b"], L["b"], sc)
        de, oke = close(e["e"], L["e"], sc)
        print(f"{name}: b {db:.1e}, e {de:.1e}")
        assert okb and oke, (name, db, de)


CEN_CASES = [("nominal", (1, 1)), ("pitch_+1.5", (1, 0)), ("base_+1000_-1000", (0, 1)), ("yaw_-100", (0, 0))]
G1_CEN_TASK = U.GOLDEN / "robot_models/unitree_g1/g1_centroidal_mpc/config/mpc/task.info"


def cen_foot_gains():
    return model_loader.parse_info(G1_CEN_TASK)["model_settings"]["foot_constraint"]


def test_harness_cen_flow_against_reference(cmodel, ref):
    """cen_flow_kernel's value lane (cenFlowDual) on the host, every recipe.  With the base 1 km out its second moments about the world origin
    once cost 7 digits (6e-9); positions are now measured from the base."""
    co = orc.CenOracle(cmodel)
    worst = {}
    for name, r in ref.items():
        d, ok = close(emu.cen_flow(co.desc, co.cdesc, r["xc"], r["uc"]), r["cen_xdot"])
        worst[name] = d
        assert ok, (name, d)
    print("CPU harness cenFlowDual against the reference: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))


def test_harness_cen_node_defect_and_constraints(cmodel, ref, g1):
    """cen_node raw b (RK4 of the centroidal flow map) and raw e (ZeroWrench / NormalVelocity / ZeroVelocity values) on the centroidal model.
    The node path's kinematics (cenKinematics) form their second moments about the base position too: with the base 1 km out they had
    measured 1.7e-11 (6e-9 in cen_flow_kernel) about the world origin."""
    co = orc.CenOracle(cmodel)
    cx = cmodel["nx"]
    swing = np.array([[0.03, 0.2, -1.0], [0.05, -0.1, 0.5]])
    for name, contact in CEN_CASES:
        r = ref[name]
        xn = r["xc"] + np.random.default_rng(6).uniform(-0.01, 0.01, cx)
        b = U.to_float(g1.cen_rk4_defect(r["xc"], r["uc"], xn, 0.015))
        e_ref = U.to_float(g1.cen_eq_constraints(r["xc"], r["uc"], contact, swing, cen_foot_gains()))
        e = emu.cen_node(co.desc, co.cdesc, r["xc"], r["uc"], xn, np.array(cmodel["x_init"]), 0.015, contact, swing, [1.0, 1.0], 0.0)["raw"]
        db, okb = close(e["b"], b)
        de, oke = close(e["e"], e_ref)
        print(f"{name}: centroidal b {db:.1e}, e {de:.1e}")
        assert okb and oke, (name, db, de)
