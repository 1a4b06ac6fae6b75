"""An extended-precision reference of the G1 dynamics, restated from the URDF itself (test infrastructure only).

Independent of the product's model description: this module parses the URDF with its own code and never welds links.  Every link of the
URDF carries its own kinetic and potential energy, so the loader's fold of fixed links (and of payload records) is checked, not reused.
Only the boost INFO syntax of task.info is read with `model_loader.parse_info`.

Semantics restated (Pinocchio's URDF importer as createPinocchioModel.cpp uses it):
  * a joint origin is a translation followed by R = Rz(yaw) Ry(pitch) Rx(roll); an <inertial> origin likewise;
  * a revolute joint rotates about its normalised axis, expressed in the joint (child) frame;
  * revolute joints outside the MPC model (task.info fixedJointNames) are locked at 0;
  * the base is Translation then SphericalZYX: q_b = (p, yaw, pitch, roll), R_b = Rz Ry Rx, generalised velocity = dq/dt
    (createPinocchioModel.cpp:60-67); gravity (0, 0, -9.81);
  * contact frames: the ankle-roll joint frame translated by contact_frame_translation, identity rotation (createPinocchioModel.cpp:77-83);
  * wrenches act through LOCAL_WORLD_ALIGNED frame Jacobians, J^T F (DynamicsHelperFunctions.cpp:232-270).

Dynamics are the Euler-Lagrange equations of L = T - V in (q, dq/dt):
  M(q) from per-link Jacobians, nle = dM/dt qd - dT/dq + dV/dq (central differences in mpmath).
All arithmetic is mpmath at `dps` digits; `Robot.at` / `G1.at` rebuild the same robot at a second (digits, step) setting, so that a test
can show the reference's own error.
"""
from __future__ import annotations

import re
import xml.etree.ElementTree as ET
from pathlib import Path

from mpmath import mp, mpf

from wb_humanoid_mpc_b200.model_loader import parse_info

GOLDEN = Path(__file__).resolve().parent / "golden" / "g1_config"
G1_URDF = GOLDEN / "robot_models/unitree_g1/g1_description/urdf/g1_29dof.urdf"
G1_WB_TASK = GOLDEN / "robot_models/unitree_g1/g1_wb_mpc/config/mpc/task.info"
G1_WB_REFERENCE = GOLDEN / "robot_models/unitree_g1/g1_wb_mpc/config/command/reference.info"

# (digits, central-difference step): truncation ~ h^2, rounding ~ 10^-dps / h, both below 1e-20 relative
PRIMARY = (40, "1e-12")
SECONDARY = (50, "1e-15")
GRAVITY = "9.81"


# ---------------------------------------------------------------------------------------------------------------------------------------
# small mpmath linear algebra: 3-vectors as lists, 3x3 matrices as lists of rows
# ---------------------------------------------------------------------------------------------------------------------------------------
def _mm(A, B):
    return [[A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j] for j in range(3)] for i in range(3)]


def _mv(A, v):
    return [A[i][0] * v[0] + A[i][1] * v[1] + A[i][2] * v[2] for i in range(3)]


def _tr(A):
    return [[A[j][i] for j in range(3)] for i in range(3)]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _add(a, b):
    return [a[0] + b[0], a[1] + b[1], a[2] + b[2]]


def _sub(a, b):
    return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]


def _scale(s, a):
    return [s * a[0], s * a[1], s * a[2]]


def _eye():
    return [[mpf(1), mpf(0), mpf(0)], [mpf(0), mpf(1), mpf(0)], [mpf(0), mpf(0), mpf(1)]]


def rot_x(a):
    c, s = mp.cos(a), mp.sin(a)
    return [[mpf(1), mpf(0), mpf(0)], [mpf(0), c, -s], [mpf(0), s, c]]


def rot_y(a):
    c, s = mp.cos(a), mp.sin(a)
    return [[c, mpf(0), s], [mpf(0), mpf(1), mpf(0)], [-s, mpf(0), c]]


def rot_z(a):
    c, s = mp.cos(a), mp.sin(a)
    return [[c, -s, mpf(0)], [s, c, mpf(0)], [mpf(0), mpf(0), mpf(1)]]


def rpy_matrix(r, p, y):
    """URDF origin rotation: fixed-axis roll, pitch, yaw = Rz(y) Ry(p) Rx(r)"""
    return _mm(rot_z(y), _mm(rot_y(p), rot_x(r)))


def axis_angle(a, th):
    """rotation by th about the unit axis a (Rodrigues)"""
    c, s = mp.cos(th), mp.sin(th)
    C = 1 - c
    x, y, z = a
    return [[c + x * x * C, x * y * C - z * s, x * z * C + y * s],
            [y * x * C + z * s, c + y * y * C, y * z * C - x * s],
            [z * x * C - y * s, z * y * C + x * s, c + z * z * C]]


def solve(A, b):
    """Gaussian elimination with partial pivoting on mpf lists"""
    n = len(b)
    M = [list(A[i]) + [b[i]] for i in range(n)]
    for k in range(n):
        p = max(range(k, n), key=lambda i: abs(M[i][k]))
        M[k], M[p] = M[p], M[k]
        for i in range(k + 1, n):
            f = M[i][k] / M[k][k]
            if f:
                for j in range(k, n + 1):
                    M[i][j] -= f * M[k][j]
    x = [mpf(0)] * n
    for i in reversed(range(n)):
        x[i] = (M[i][n] - sum(M[i][j] * x[j] for j in range(i + 1, n))) / M[i][i]
    return x


def inv3(A):
    cols = [solve(A, [mpf(int(i == j)) for i in range(3)]) for j in range(3)]
    return [[cols[j][i] for j in range(3)] for i in range(3)]


# ---------------------------------------------------------------------------------------------------------------------------------------
# URDF text (kept as strings so every precision setting converts the decimals itself)
# ---------------------------------------------------------------------------------------------------------------------------------------
def _triple(el, attr, default="0 0 0"):
    s = default if el is None else el.get(attr, default)
    v = s.split()
    assert len(v) == 3, s
    return v


def read_urdf(text: str):
    """-> (links {name: None | (mass, xyz, rpy, (ixx, ixy, ixz, iyy, iyz, izz))}, joints [dict(name, type, parent, child, xyz, rpy, axis)])"""
    root = ET.fromstring(text)
    links = {}
    for ln in root.iter("link"):
        ine = ln.find("inertial")
        if ine is None:
            links[ln.get("name")] = None
            continue
        org = ine.find("origin")
        it = ine.find("inertia")
        links[ln.get("name")] = (ine.find("mass").get("value"), _triple(org, "xyz"), _triple(org, "rpy"),
                                 tuple(it.get(k) for k in ("ixx", "ixy", "ixz", "iyy", "iyz", "izz")))
    joints = []
    for jn in root.iter("joint"):
        org, ax = jn.find("origin"), jn.find("axis")
        joints.append(dict(name=jn.get("name"), type=jn.get("type"), parent=jn.find("parent").get("link"), child=jn.find("child").get("link"),
                           xyz=_triple(org, "xyz"), rpy=_triple(org, "rpy"), axis=_triple(ax, "xyz", "1 0 0")))
    return links, joints


def g1_joint_order(task_path=G1_WB_TASK):
    """MPC joint order: the joint annotations of task.info's initialState rows 6..6+nj (the reference lists them in its model order)"""
    rows = {}
    for line in Path(task_path).read_text().splitlines():
        m = re.match(r"\s*\((\d+),0\)\s+\S+\s*;\s*(\w+_joint)\b", line)
        if m:
            rows.setdefault(m.group(2), int(m.group(1)))
    names = sorted(rows, key=rows.get)
    task = parse_info(task_path)
    fixed = set(task["model_settings"]["fixedJointNames"].values())
    return [n for n in names if n not in fixed], fixed


# ---------------------------------------------------------------------------------------------------------------------------------------
# the robot
# ---------------------------------------------------------------------------------------------------------------------------------------
class Robot:
    """Floating-base tree of a URDF in mpmath.  `joint_names`: the generalised joint coordinates in order; every other revolute joint is
    locked at 0.  `frames`: {name: (link, offset xyz strings)} operational frames with identity rotation in the link frame.
    `extra`: [(parent link, mass, com xyz, inertia 3x3 about its com in the parent link's axes)] rigid payloads, each an extra fixed link."""

    def __init__(self, urdf_text, joint_names, frames=None, extra=(), dps=PRIMARY[0], step=PRIMARY[1]):
        self.dps, self.step_str = dps, step
        self.joint_names = list(joint_names)
        self.nj = len(self.joint_names)
        self.nv = 6 + self.nj
        self._links, self._joints = read_urdf(urdf_text)
        self._frames = dict(frames or {})
        self._extra = list(extra)
        child = {j["child"] for j in self._joints}
        roots = [l for l in self._links if l not in child]
        assert len(roots) == 1, roots
        self.root = roots[0]
        jid = {n: i for i, n in enumerate(self.joint_names)}
        for j in self._joints:
            assert j["type"] in ("revolute", "continuous", "fixed"), j
            assert j["type"] != "fixed" or j["name"] not in jid
        assert all(any(j["name"] == n for j in self._joints) for n in self.joint_names)
        self._jid = jid
        with mp.workdps(self.dps):
            self._setup()

    def _setup(self):
        self.h = mpf(self.step_str)
        self.g = mpf(GRAVITY)
        self.inertial = {}  # link -> (m, com in link frame, inertia about com in link axes)
        for name, v in self._links.items():
            if v is None:
                continue
            m, xyz, rpy, (ixx, ixy, ixz, iyy, iyz, izz) = v
            I = [[mpf(ixx), mpf(ixy), mpf(ixz)], [mpf(ixy), mpf(iyy), mpf(iyz)], [mpf(ixz), mpf(iyz), mpf(izz)]]
            Rin = rpy_matrix(*[mpf(s) for s in rpy])
            self.inertial[name] = [(mpf(m), [mpf(s) for s in xyz], _mm(Rin, _mm(I, _tr(Rin))))]
        for parent, m, c, I in self._extra:
            self.inertial.setdefault(parent, []).append((mpf(m), [mpf(s) for s in c], [[mpf(s) for s in row] for row in I]))
        self.children = {}
        for j in self._joints:
            ax = [mpf(s) for s in j["axis"]]
            n = mp.sqrt(_dot(ax, ax))
            self.children.setdefault(j["parent"], []).append(dict(j, R0=rpy_matrix(*[mpf(s) for s in j["rpy"]]), p0=[mpf(s) for s in j["xyz"]],
                                                                   a=_scale(1 / n, ax)))
        self.frames = {k: (l, [mpf(s) for s in off]) for k, (l, off) in self._frames.items()}
        self.total_mass = sum(m for lst in self.inertial.values() for m, _, _ in lst)

    def at(self, dps, step):
        """the same robot at another (digits, step) setting"""
        return Robot.__new__(Robot)._clone(self, dps, step)

    def _clone(self, other, dps, step):
        self.__dict__.update({k: other.__dict__[k] for k in ("joint_names", "nj", "nv", "_links", "_joints", "_frames", "_extra", "root", "_jid")})
        self.dps, self.step_str = dps, step
        with mp.workdps(dps):
            self._setup()
        return self

    # -- kinematics ------------------------------------------------------------------------------------------------------------------
    def kinematics(self, q):
        """{link: (R world, origin world, columns)}; a column is (k, kind, vec, point): kind 'T' = translation along vec, 'R' = rotation
        about the world axis vec through the world point"""
        p, (yaw, pitch, roll) = q[0:3], q[3:6]
        ex, ey, ez = [mpf(1), mpf(0), mpf(0)], [mpf(0), mpf(1), mpf(0)], [mpf(0), mpf(0), mpf(1)]
        Rz = rot_z(yaw)
        Rzy = _mm(Rz, rot_y(pitch))
        Rb = _mm(Rzy, rot_x(roll))
        cols = [(0, "T", ex, None), (1, "T", ey, None), (2, "T", ez, None),
                (3, "R", ez, p), (4, "R", _mv(Rz, ey), p), (5, "R", _mv(Rzy, ex), p)]
        out = {}
        stack = [(self.root, Rb, list(p), cols)]
        while stack:
            link, R, o, cl = stack.pop()
            out[link] = (R, o, cl)
            for j in self.children.get(link, []):
                oj = _add(o, _mv(R, j["p0"]))
                Rj = _mm(R, j["R0"])
                k = self._jid.get(j["name"])
                if k is None:
                    stack.append((j["child"], Rj, oj, cl))
                else:
                    aw = _mv(Rj, j["a"])
                    stack.append((j["child"], _mm(Rj, axis_angle(j["a"], q[6 + k])), oj, cl + [(6 + k, "R", aw, oj)]))
        return out

    @staticmethod
    def _col_lin(col, x):
        k, kind, v, pt = col
        return v if kind == "T" else _cross(v, _sub(x, pt))

    @staticmethod
    def _col_ang(col):
        return None if col[1] == "T" else col[2]

    def _bodies(self, kin):
        """(m, com world, inertia world about com, columns) of every mass in the tree"""
        for link, lst in self.inertial.items():
            R, o, cl = kin[link]
            for m, c, I in lst:
                yield m, _add(o, _mv(R, c)), _mm(R, _mm(I, _tr(R))), cl

    def point_velocity(self, cl, x, qd):
        v, w = [mpf(0)] * 3, [mpf(0)] * 3
        for col in cl:
            s = qd[col[0]]
            v = _add(v, _scale(s, self._col_lin(col, x)))
            if col[1] == "R":
                w = _add(w, _scale(s, col[2]))
        return v, w

    def point_jacobian(self, cl, x):
        """6 x nv LOCAL_WORLD_ALIGNED Jacobian (linear rows of the point x, angular rows) as a list of rows"""
        J = [[mpf(0)] * self.nv for _ in range(6)]
        for col in cl:
            lv = self._col_lin(col, x)
            for r in range(3):
                J[r][col[0]] = lv[r]
                if col[1] == "R":
                    J[3 + r][col[0]] = col[2][r]
        return J

    # -- energies and the mass matrix ------------------------------------------------------------------------------------------------
    def lagrangian(self, q, qd):
        kin = self.kinematics(q)
        T = V = mpf(0)
        for m, c, I, cl in self._bodies(kin):
            v, w = self.point_velocity(cl, c, qd)
            T += (m * _dot(v, v) + _dot(w, _mv(I, w))) / 2
            V += m * self.g * c[2]
        return T - V

    def momentum(self, q, qd):
        """generalised momentum dT/dqd = M(q) qd, summed link by link"""
        out = [mpf(0)] * self.nv
        for m, c, I, cl in self._bodies(self.kinematics(q)):
            v, w = self.point_velocity(cl, c, qd)
            Iw = _mv(I, w)
            for col in cl:
                out[col[0]] += m * _dot(self._col_lin(col, c), v) + (_dot(col[2], Iw) if col[1] == "R" else 0)
        return out

    def mass_matrix(self, q):
        M = [[mpf(0)] * self.nv for _ in range(self.nv)]
        for m, c, I, cl in self._bodies(self.kinematics(q)):
            lin = [self._col_lin(col, c) for col in cl]
            ang = [_mv(I, col[2]) if col[1] == "R" else None for col in cl]
            for a, ca in enumerate(cl):
                for b, cb in enumerate(cl[: a + 1]):
                    s = m * _dot(lin[a], lin[b])
                    if ang[b] is not None and ca[1] == "R":
                        s += _dot(ca[2], ang[b])
                    M[ca[0]][cb[0]] += s
                    if ca[0] != cb[0]:
                        M[cb[0]][ca[0]] += s
        return M

    def nle(self, q, qd):
        """Euler-Lagrange: nle = dM/dt qd - dL/dq  (L = T - V)"""
        h = self.h
        qp = [a + h * b for a, b in zip(q, qd)]
        qm = [a - h * b for a, b in zip(q, qd)]
        Mdqd = [(a - b) / (2 * h) for a, b in zip(self.momentum(qp, qd), self.momentum(qm, qd))]
        out = []
        for i in range(self.nv):
            qp, qm = list(q), list(q)
            qp[i] += h
            qm[i] -= h
            out.append(Mdqd[i] - (self.lagrangian(qp, qd) - self.lagrangian(qm, qd)) / (2 * h))
        return out

    # -- frames ----------------------------------------------------------------------------------------------------------------------
    def frame(self, kin, name):
        link, off = self.frames[name]
        R, o, cl = kin[link]
        return R, _add(o, _mv(R, off)), cl

    # -- centroidal ------------------------------------------------------------------------------------------------------------------
    def centroidal_map(self, q):
        """A_g (6 x nv): linear momentum and angular momentum about the centre of mass, world axes, per unit generalised velocity; com"""
        kin = self.kinematics(q)
        bodies = list(self._bodies(kin))
        G = _scale(1 / self.total_mass, [sum(m * c[r] for m, c, _, _ in bodies) for r in range(3)])
        A = [[mpf(0)] * self.nv for _ in range(6)]
        for m, c, I, cl in bodies:
            d = _sub(c, G)
            for col in cl:
                lv = _scale(m, self._col_lin(col, c))
                ang = _cross(d, lv)
                if col[1] == "R":
                    ang = _add(ang, _mv(I, col[2]))
                for r in range(3):
                    A[r][col[0]] += lv[r]
                    A[3 + r][col[0]] += ang[r]
        return A, G

    def composite_inertia(self, q):
        """rotational inertia of the whole robot about its centre of mass (world axes) and the centre of mass"""
        bodies = list(self._bodies(self.kinematics(q)))
        G = _scale(1 / self.total_mass, [sum(m * c[r] for m, c, _, _ in bodies) for r in range(3)])
        Ig = [[mpf(0)] * 3 for _ in range(3)]
        for m, c, I, _ in bodies:
            d = _sub(c, G)
            dd = _dot(d, d)
            for r in range(3):
                for s in range(3):
                    Ig[r][s] += I[r][s] + m * ((dd if r == s else 0) - d[r] * d[s])
        return Ig, G


def orientation_error_to_plane(R):
    """rotationMatrixDistanceToPlane(R, e_z): -vec of the quaternion turning R e_z onto e_z (RotationTransforms.h)"""
    a = [R[0][2], R[1][2], R[2][2]]
    c = _cross(a, [mpf(0), mpf(0), mpf(1)])
    w = 1 + a[2]
    n = mp.sqrt(_dot(c, c) + w * w)
    return [-c[0] / n, -c[1] / n, -c[2] / n]


# ---------------------------------------------------------------------------------------------------------------------------------------
# the G1 MPC quantities
# ---------------------------------------------------------------------------------------------------------------------------------------
class G1:
    """The whole-body and centroidal MPC quantities of the G1 (state / input layouts of WBAccelMpcRobotModel and CentroidalMpcRobotModel),
    from a Robot built on the URDF and task.info."""

    def __init__(self, robot: Robot, contact_frames=("foot_l_contact", "foot_r_contact")):
        self.r = robot
        self.contacts = list(contact_frames)
        self.nj, self.nv = robot.nj, robot.nv

    @classmethod
    def from_files(cls, urdf=G1_URDF, task=G1_WB_TASK, payloads=(), dps=PRIMARY[0], step=PRIMARY[1]):
        """payloads: [(body index of the MPC model: 0 = pelvis, i = child link of the i-th MPC joint, mass, com, inertia or None)]"""
        names, _ = g1_joint_order(task)
        t = parse_info(task)
        parents = [t["model_settings"]["contactParentJointNames"][k] for k in sorted(t["model_settings"]["contactParentJointNames"])]
        cnames = [t["model_settings"]["contactNames6DoF"][k] for k in sorted(t["model_settings"]["contactNames6DoF"])]
        ct = [t["contacts"]["contact_frame_translation"][a] for a in "xyz"]
        _, joints = read_urdf(Path(urdf).read_text())
        child_of = {j["name"]: j["child"] for j in joints}
        frames = {c: (child_of[p], ct) for c, p in zip(cnames, parents)}
        child = {j["child"] for j in joints}
        root = [j["parent"] for j in joints if j["parent"] not in child][0]
        extra = []
        for body, m, c, I in payloads:
            link = root if body == 0 else child_of[names[body - 1]]
            I = [[0] * 3] * 3 if I is None else I
            extra.append((link, repr(float(m)), [repr(float(v)) for v in c], [[repr(float(v)) for v in row] for row in I]))
        return cls(Robot(Path(urdf).read_text(), names, frames, extra, dps, step), cnames)

    def at(self, dps, step):
        return G1(self.r.at(dps, step), self.contacts)

    def _mp(self, v):
        return [a if isinstance(a, mpf) else mpf(float(a)) for a in v]

    def _contact_force(self, q, u):
        """J_l^T F_l + J_r^T F_r (LOCAL_WORLD_ALIGNED contact-frame Jacobians)"""
        kin = self.r.kinematics(q)
        tau = [mpf(0)] * self.nv
        for c, name in enumerate(self.contacts):
            _, p, cl = self.r.frame(kin, name)
            J = self.r.point_jacobian(cl, p)
            for r in range(6):
                f = u[6 * c + r]
                for k in range(self.nv):
                    tau[k] += J[r][k] * f
        return tau

    def dynamics(self, x, u):
        """everything of one whole-body (x, u): dict(M, nle, JtF, qddb, tau, xdot) as mpf; computeBaseAcceleration's block-diagonal inverse
        and computeJointTorques (DynamicsHelperFunctions.cpp:196-270)"""
        with mp.workdps(self.r.dps):
            x, u = self._mp(x), self._mp(u)
            nv, nj = self.nv, self.nj
            q, qd, qddj = x[:nv], x[nv:], u[12:]
            M, nle, JtF = self.r.mass_matrix(q), self.r.nle(q, qd), self._contact_force(q, u)
            mid = [-nle[i] - sum(M[i][6 + j] * qddj[j] for j in range(nj)) + JtF[i] for i in range(6)]
            qddb = solve([row[0:3] for row in M[0:3]], mid[0:3]) + solve([row[3:6] for row in M[3:6]], mid[3:6])
            qdd = qddb + qddj
            tau = [sum(M[6 + j][k] * qdd[k] for k in range(nv)) + nle[6 + j] - JtF[6 + j] for j in range(nj)]
            return dict(M=M, nle=nle, JtF=JtF, qddb=qddb, tau=tau, xdot=qd + qddb + qddj)

    def foot_state(self, x, qdd):
        """per contact: pos, R, oriErr, vlin, vang, alin (classical, d^2p/dt^2 along (qd, qdd)), aang"""
        with mp.workdps(self.r.dps):
            x, qdd = self._mp(x), self._mp(qdd)
            nv, h = self.nv, self.r.h
            q, qd = x[:nv], x[nv:]

            def state(s):
                qs = [a + s * b + s * s / 2 * c for a, b, c in zip(q, qd, qdd)]
                vs = [b + s * c for b, c in zip(qd, qdd)]
                kin = self.r.kinematics(qs)
                out = []
                for name in self.contacts:
                    R, p, cl = self.r.frame(kin, name)
                    v, w = self.r.point_velocity(cl, p, vs)
                    out.append((R, p, v, w))
                return out

            s0, sp, sm = state(mpf(0)), state(h), state(-h)
            feet = []
            for c in range(len(self.contacts)):
                R, p, v, w = s0[c]
                feet.append(dict(pos=p, R=R, oriErr=orientation_error_to_plane(R), vlin=v, vang=w,
                                 alin=[(a - b) / (2 * h) for a, b in zip(sp[c][2], sm[c][2])],
                                 aang=[(a - b) / (2 * h) for a, b in zip(sp[c][3], sm[c][3])]))
            return feet

    def rk4_defect(self, x, u, xnext, dt):
        """one RK4 step of the flow map minus the next node's state (the multiple-shooting dynamics defect b)"""
        with mp.workdps(self.r.dps):
            x, xn, dt = self._mp(x), self._mp(xnext), mpf(float(dt))
            f = lambda z: self.dynamics(z, u)["xdot"]
            k1 = f(x)
            k2 = f([a + dt / 2 * b for a, b in zip(x, k1)])
            k3 = f([a + dt / 2 * b for a, b in zip(x, k2)])
            k4 = f([a + dt * b for a, b in zip(x, k3)])
            return [a + dt / 6 * (b1 + 2 * b2 + 2 * b3 + b4) - c for a, b1, b2, b3, b4, c in zip(x, k1, k2, k3, k4, xn)]

    def eq_constraints(self, x, u, contact, swing, gains):
        """per foot, in the collection's order: ZeroWrenchConstraint (6) and SwingLegVerticalConstraintCppAd (1) of a swing foot
        (WBMpcPreComputation.cpp:92-103), ZeroAccelerationConstraintCppAd (6) of a stance foot.  gains: task.info foot_constraint block."""
        with mp.workdps(self.r.dps):
            G = {k: mpf(v) for k, v in gains.items()}
            xdot = self.dynamics(x, u)["xdot"]
            feet = self.foot_state(x, xdot[self.nv:])
            u = self._mp(u)
            Av = [G["linearVelocityErrorGain_xy"]] * 2 + [G["linearVelocityErrorGain_z"]] + [G["angularVelocityErrorGain"]] * 3
            Aa = [G["linearAccelerationErrorGain_xy"]] * 2 + [G["linearAccelerationErrorGain_z"]] + [G["angularAccelerationErrorGain"]] * 3
            out = []
            for c, f in enumerate(feet):
                if contact[c]:
                    out += [Av[k] * f["vlin"][k] + Aa[k] * f["alin"][k] + (G["positionErrorGain_z"] * f["pos"][2] if k == 2 else 0)
                            for k in range(3)]
                    out += [G["orientationErrorGain"] * f["oriErr"][k] + Av[3 + k] * f["vang"][k] + Aa[3 + k] * f["aang"][k] for k in range(3)]
                else:
                    z, vz, az = self._mp(swing[c])
                    out += u[6 * c:6 * c + 6]
                    out.append(G["positionErrorGain_z"] * (f["pos"][2] - z) + G["linearVelocityErrorGain_z"] * (f["vlin"][2] - vz)
                               + G["linearAccelerationErrorGain_z"] * (f["alin"][2] - az))
            return out

    def cen_rk4_defect(self, x, u, xnext, dt):
        """one RK4 step of the centroidal flow map minus the next node's state"""
        with mp.workdps(self.r.dps):
            x, xn, dt = self._mp(x), self._mp(xnext), mpf(float(dt))
            f = lambda z: self.cen_flow_map(z, u)
            k1 = f(x)
            k2 = f([a + dt / 2 * b for a, b in zip(x, k1)])
            k3 = f([a + dt / 2 * b for a, b in zip(x, k2)])
            k4 = f([a + dt * b for a, b in zip(x, k3)])
            return [a + dt / 6 * (b1 + 2 * b2 + 2 * b3 + b4) - c for a, b1, b2, b3, b4, c in zip(x, k1, k2, k3, k4, xn)]

    def cen_eq_constraints(self, x, u, contact, swing, gains):
        """the centroidal MPC's per-foot equality constraints, in the collection's order: ZeroWrenchConstraint (6) and NormalVelocityConstraint
        (1) of a swing foot, ZeroVelocityConstraintCppAd (6) of a stance foot (humanoid_centroidal_mpc/src/constraint/
        ZeroVelocityConstraintCppAd.cpp); the foot twist from the generalised velocity of the centroidal flow map"""
        with mp.workdps(self.r.dps):
            G = {k: mpf(v) for k, v in gains.items()}
            nv = self.nv
            v = self.cen_flow_map(x, u)[6:6 + nv]
            x, u = self._mp(x), self._mp(u)
            feet = self.foot_state(x[6:] + v, [mpf(0)] * nv)
            out = []
            for c, f in enumerate(feet):
                if contact[c]:
                    out += [f["vlin"][0], f["vlin"][1], f["vlin"][2] + G["positionErrorGain_z"] * f["pos"][2]]
                    out += [f["vang"][k] + G["orientationErrorGain"] * f["oriErr"][k] for k in range(3)]
                else:
                    z, vz, _ = self._mp(swing[c])
                    out += u[6 * c:6 * c + 6]
                    out.append(f["vlin"][2] - vz + G["positionErrorGain_z"] * (f["pos"][2] - z))
            return out

    def centroidal_map(self, q):
        with mp.workdps(self.r.dps):
            return self.r.centroidal_map(self._mp(q))

    def cen_flow_map(self, x, u):
        """PinocchioCentroidalDynamicsAD::getValueCppAd (full centroidal dynamics): x = (h/m 6, q nv), u = (F_l 6, F_r 6, qd_j nj)"""
        with mp.workdps(self.r.dps):
            x, u = self._mp(x), self._mp(u)
            nv, nj, m = self.nv, self.nj, self.r.total_mass
            q = x[6:]
            A, G = self.r.centroidal_map(q)
            kin = self.r.kinematics(q)
            lin, ang = [mpf(0), mpf(0), -self.r.g * m], [mpf(0)] * 3
            for c, name in enumerate(self.contacts):
                _, p, _ = self.r.frame(kin, name)
                F, T = u[6 * c:6 * c + 3], u[6 * c + 3:6 * c + 6]
                lin = _add(lin, F)
                ang = _add(ang, _add(_cross(_sub(p, G), F), T))
            mom = [m * x[r] - sum(A[r][6 + j] * u[12 + j] for j in range(nj)) for r in range(6)]
            # getPinocchioJointVelocity: the block inverse of [[m 1, A12], [0, A22]] (computeFloatingBaseCentroidalMomentumMatrixInverse)
            wb = solve([row[3:6] for row in A[3:6]], mom[3:6])
            vb = [(mom[r] - sum(A[r][3 + k] * wb[k] for k in range(3))) / A[0][0] for r in range(3)]
            return _scale(1 / m, lin) + _scale(1 / m, ang) + vb + wb + u[12:]


def to_float(v):
    if isinstance(v, dict):
        return {k: to_float(a) for k, a in v.items()}
    if isinstance(v, (list, tuple)):
        import numpy as np

        return np.array([to_float(a) for a in v], dtype=float)
    return float(v)
