"""Host-side loader: reference config files (URDF + task.info + reference.info + gait.info) -> flat model description.

The reference builds its rigid-body model and OCP constants inside C++ objects
(`createCustomPinocchioInterface`, humanoid_common_mpc/src/pinocchio_model/createPinocchioModel.cpp:144-182;
`ModelSettings`, src/common/ModelSettings.cpp:110-185; `HumanoidCostConstraintFactory`,
src/HumanoidCostConstraintFactory.cpp:77-245; `WBMpcInterface`, humanoid_wb_mpc/src/WBMpcInterface.cpp:69-199).
A GPU cannot consume those objects, so this loader re-derives the same constants from the same
files and emits one flat dictionary (see `build_wb_model`) that is (a) passed across the C ABI as
`b200sqp_model_desc` and (b) stored as JSON so the GPU box needs neither the reference nor a URDF parser.

Conventions reproduced from the reference / Pinocchio's URDF importer:
  * joints not in `mpcModelJointNames` are welded (FIXED) and the child link inertia is folded
    into the parent body (Pinocchio `appendBodyToJoint`), createPinocchioModel.cpp:156-164;
  * joint order is a depth-first walk with children sorted by joint name (urdfdom stores joints in a
    std::map), which yields the order listed in task.info `initialState` (task.info:119-186);
  * the floating base is `JointModelComposite(Translation, SphericalZYX)` (createPinocchioModel.cpp:60-67);
  * contact / collision frames are rigidly attached to the ankle-roll joint frame
    (createPinocchioModel.cpp:76-131).
"""
from __future__ import annotations

import copy
import json
import math
import re
import xml.etree.ElementTree as ET
from pathlib import Path

import numpy as np

# ----------------------------------------------------------------------------------------------
# boost::property_tree INFO subset parser (loadData::loadPtreeValue / loadEigenMatrix / loadStdVector,
# ocs2_core/include/ocs2_core/misc/LoadData.h)
# ----------------------------------------------------------------------------------------------


def _tokenize_info(text: str):
    toks = []
    for raw in text.splitlines():
        line = raw.split(";")[0]  # ';' starts a comment
        # '//' comments appear in the shipped task.info as well
        line = line.split("//")[0]
        for m in re.finditer(r'"[^"]*"|\{|\}|[^\s{}]+', line):
            toks.append(m.group(0))
        toks.append("\n")
    return toks


def parse_info(path: str | Path) -> dict:
    """Parse a boost INFO file into nested dicts (leaf values stay strings)."""
    toks = _tokenize_info(Path(path).read_text())
    pos = 0

    def parse_block():
        nonlocal pos
        node: dict = {}
        while pos < len(toks):
            t = toks[pos]
            if t == "\n":
                pos += 1
                continue
            if t == "}":
                pos += 1
                return node
            key = t.strip('"')
            pos += 1
            val = None
            # value on the same line?
            if pos < len(toks) and toks[pos] not in ("\n", "{", "}"):
                val = toks[pos].strip('"')
                pos += 1
                # swallow trailing tokens on the line (e.g. stray ';' less comments)
                while pos < len(toks) and toks[pos] not in ("\n", "{", "}"):
                    pos += 1
            # skip newlines before a possible '{'
            save = pos
            while pos < len(toks) and toks[pos] == "\n":
                pos += 1
            if pos < len(toks) and toks[pos] == "{":
                pos += 1
                child = parse_block()
                node[key] = child
            else:
                pos = save
                node[key] = val
        return node

    return parse_block()


def info_get(tree: dict, dotted: str, default=None):
    node = tree
    for k in dotted.split("."):
        if not isinstance(node, dict) or k not in node:
            if default is not None:
                return default
            raise KeyError(dotted)
        node = node[k]
    return node


def info_float(tree, dotted, default=None) -> float:
    v = info_get(tree, dotted, default)
    return float(str(v).rstrip(";"))


def info_matrix(tree: dict, name: str, rows: int, cols: int) -> np.ndarray:
    """loadData::loadEigenMatrix: entries '(i,j) v', optional 'scaling', missing entries = 0."""
    blk = tree[name]
    out = np.zeros((rows, cols))
    scaling = float(blk.get("scaling", 1.0))
    for k, v in blk.items():
        m = re.fullmatch(r"\((\d+),(\d+)\)", k)
        if m:
            out[int(m.group(1)), int(m.group(2))] = float(v)
    return out * scaling


def joint_torque_weights(task_path, nj: int = 23) -> np.ndarray | None:
    """joint_torque_weights of a task.info (WBMpcInterface::getJointTorqueCost: loadEigenMatrix into nj entries, MPC joint order; nj = the MPC
    model's joint count, model["nj"]), or None when the key is absent.  Reading the key does not switch the term on: in the reference the cost
    exists only where the interface adds it to the cost collection (B200SqpSolver.set_joint_torque_cost does that here)."""
    task = parse_info(task_path)
    if "joint_torque_weights" not in task:
        return None
    return info_matrix(task, "joint_torque_weights", nj, 1)[:, 0]


def info_list(tree: dict, dotted: str) -> list[str]:
    blk = info_get(tree, dotted)
    items = []
    for k, v in blk.items():
        m = re.fullmatch(r"\[(\d+)\]", k)
        if m:
            items.append((int(m.group(1)), v))
    return [v for _, v in sorted(items)]


# ----------------------------------------------------------------------------------------------
# URDF -> reduced kinematic tree
# ----------------------------------------------------------------------------------------------


def _rpy_to_R(rpy):
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = math.cos(r), math.sin(r), math.cos(p), math.sin(p), math.cos(y), math.sin(y)
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def _vec(s, n=3):
    v = [float(x) for x in s.split()]
    assert len(v) == n
    return np.array(v)


class _Inertia:
    """mass, com (in the frame it is expressed in), rotational inertia about the com (same axes)."""

    def __init__(self, m=0.0, c=None, I=None):
        self.m = m
        self.c = np.zeros(3) if c is None else np.array(c, float)
        self.I = np.zeros((3, 3)) if I is None else np.array(I, float)

    def transformed(self, R, p):
        """express in a parent frame: x_parent = R x + p"""
        return _Inertia(self.m, R @ self.c + p, R @ self.I @ R.T)

    def __add__(self, o):
        m = self.m + o.m
        if m == 0.0:
            return _Inertia()
        c = (self.m * self.c + o.m * o.c) / m

        def shift(I, mm, d):  # parallel axis: about point c from com at c+d
            return I + mm * (d @ d * np.eye(3) - np.outer(d, d))

        I = shift(self.I, self.m, self.c - c) + shift(o.I, o.m, o.c - c)
        return _Inertia(m, c, I)


def parse_urdf(urdf_path: str | Path):
    root = ET.parse(str(urdf_path)).getroot()
    links = {}
    for ln in root.findall("link"):
        ine = ln.find("inertial")
        if ine is None:
            links[ln.get("name")] = _Inertia()
            continue
        org = ine.find("origin")
        xyz = _vec(org.get("xyz", "0 0 0")) if org is not None else np.zeros(3)
        rpy = _vec(org.get("rpy", "0 0 0")) if org is not None else np.zeros(3)
        m = float(ine.find("mass").get("value"))
        it = ine.find("inertia")
        I = np.array(
            [
                [float(it.get("ixx")), float(it.get("ixy")), float(it.get("ixz"))],
                [float(it.get("ixy")), float(it.get("iyy")), float(it.get("iyz"))],
                [float(it.get("ixz")), float(it.get("iyz")), float(it.get("izz"))],
            ]
        )
        R = _rpy_to_R(rpy)
        links[ln.get("name")] = _Inertia(m, xyz, R @ I @ R.T)
    joints = {}
    for jn in root.findall("joint"):
        org = jn.find("origin")
        xyz = _vec(org.get("xyz", "0 0 0")) if org is not None else np.zeros(3)
        rpy = _vec(org.get("rpy", "0 0 0")) if org is not None else np.zeros(3)
        ax = jn.find("axis")
        lim = jn.find("limit")
        joints[jn.get("name")] = dict(
            type=jn.get("type"),
            parent=jn.find("parent").get("link"),
            child=jn.find("child").get("link"),
            R=_rpy_to_R(rpy),
            p=xyz,
            axis=_vec(ax.get("xyz")) if ax is not None else np.array([1.0, 0, 0]),
            lower=float(lim.get("lower")) if lim is not None and lim.get("lower") else -math.inf,
            upper=float(lim.get("upper")) if lim is not None and lim.get("upper") else math.inf,
        )
    return links, joints


def reduce_tree(links, joints, fixed_joint_names):
    """Weld fixed joints; return bodies in Pinocchio joint order.

    bodies[0] is the floating base body; bodies[i>0] belongs to the i-th MPC joint.
    """
    child_links = {j["child"] for j in joints.values()}
    roots = [l for l in links if l not in child_links]
    assert len(roots) == 1, roots
    root = roots[0]
    by_parent: dict[str, list[str]] = {}
    for name in sorted(joints):  # urdfdom keeps joints in a std::map -> alphabetical child order
        by_parent.setdefault(joints[name]["parent"], []).append(name)

    bodies = [dict(name="base", joint=None, parent=-1, R=np.eye(3), p=np.zeros(3), axis=None, inertia=_Inertia(), lower=0, upper=0)]
    link_body = {}  # link -> (body index, R, p of link frame in that body's joint frame)

    def visit(link, body_idx, R, p):
        link_body[link] = (body_idx, R, p)
        bodies[body_idx]["inertia"] = bodies[body_idx]["inertia"] + links[link].transformed(R, p)
        for jname in by_parent.get(link, []):
            j = joints[jname]
            Rj, pj = R @ j["R"], R @ j["p"] + p
            movable = j["type"] in ("revolute", "continuous") and jname not in fixed_joint_names
            if j["type"] in ("floating", "prismatic", "planar") and jname not in fixed_joint_names:
                raise ValueError(f"unsupported joint type {j['type']} for {jname}")
            if movable:
                bodies.append(
                    dict(name=j["child"], joint=jname, parent=body_idx, R=Rj, p=pj, axis=j["axis"] / np.linalg.norm(j["axis"]),
                         inertia=_Inertia(), lower=j["lower"], upper=j["upper"])
                )
                visit(j["child"], len(bodies) - 1, np.eye(3), np.zeros(3))
            else:
                visit(j["child"], body_idx, Rj, pj)

    visit(root, 0, np.eye(3), np.zeros(3))
    return bodies, link_body


# ----------------------------------------------------------------------------------------------
# Whole-body model description
# ----------------------------------------------------------------------------------------------

G1_REL = dict(
    urdf="robot_models/unitree_g1/g1_description/urdf/g1_29dof.urdf",
    task="robot_models/unitree_g1/g1_wb_mpc/config/mpc/task.info",
    reference="robot_models/unitree_g1/g1_wb_mpc/config/command/reference.info",
    gait="humanoid_nmpc/humanoid_common_mpc/config/command/gait.info",
    centroidal_task="robot_models/unitree_g1/g1_centroidal_mpc/config/mpc/task.info",
    centroidal_reference="robot_models/unitree_g1/g1_centroidal_mpc/config/command/reference.info",
)


def build_wb_model(urdf_path, task_path, reference_path=None, gait_path=None, kind="wb") -> dict:
    """Flat model description of the whole-body (kind="wb") or the centroidal (kind="centroidal") MPC. All matrices row-major nested lists.
    Both MPCs use the same reduced kinematic tree, contact frames and per-node reference data; they differ in the state/input layout
    (WBAccelMpcRobotModel.h:76-241 / CentroidalMpcRobotModel.h:52-160), the weights and the task-space terms."""
    task = parse_info(task_path)
    links, joints = parse_urdf(urdf_path)
    fixed = set(info_list(task, "model_settings.fixedJointNames"))
    bodies, link_body = reduce_tree(links, joints, fixed)
    nj = len(bodies) - 1
    joint_names = [b["joint"] for b in bodies[1:]]
    jidx = {n: i for i, n in enumerate(joint_names)}

    contact_names = info_list(task, "model_settings.contactNames6DoF")
    contact_parents = info_list(task, "model_settings.contactParentJointNames")
    ct = np.array([info_float(task, f"contacts.contact_frame_translation.{a}") for a in "xyz"])
    rect = {k: info_float(task, f"contacts.contact_rectangle.{k}") for k in ("x_max", "x_min", "y_max", "y_min")}

    # frames: (name, body index, translation in the body's joint frame); rotation is identity for all of them
    frames = []
    for cname, pj in zip(contact_names, contact_parents):
        b = jidx[pj] + 1
        frames.append((cname, b, ct))
        frames.append((cname + "_collision_p_1", b, ct + np.array([rect["x_max"] * 0.6, 0, 0])))
        frames.append((cname + "_collision_p_2", b, ct + np.array([rect["x_min"] * 0.6, 0, 0])))
    cc = "collision_constraint."
    for key in ("foot.leftAnkleFrame", "foot.rightAnkleFrame", "knee.leftKneeFrame", "knee.rightKneeFrame"):
        jn = info_get(task, cc + key)
        frames.append((jn, jidx[jn] + 1, np.zeros(3)))

    nx, nu = (2 * (6 + nj), 12 + nj) if kind == "wb" else (12 + nj, 12 + nj)
    Q = info_matrix(task, "Q", nx, nx)
    R = info_matrix(task, "R", nu, nu)
    Qf = info_matrix(task, "Q_final", nx, nx) * info_float(task, "terminalCostScaling")
    x_init = info_matrix(task, "initialState", nx, 1)[:, 0]

    fc = "model_settings.foot_constraint."
    w = "task_space_foot_cost_weights."
    # EndEffectorDynamicsWeights::getWeights (humanoid_wb_mpc/src/cost/EndEffectorDynamicsCostHelpers.cpp:97-110)
    # overwrites the velocity weights with the acceleration entries and leaves the acceleration weights at
    # their defaults 0.01 (EndEffectorDynamicsCostHelpers.h:45-50).  Reproduced on purpose.
    foot_w = np.concatenate(
        [
            [info_float(task, w + f"pos_{a}") for a in "xyz"],
            [info_float(task, w + f"orientation_{a}") for a in "xyz"],
            [info_float(task, w + f"lin_acceleration_{a}") for a in "xyz"],
            [info_float(task, w + f"ang_acceleration_{a}") for a in "xyz"],
            [0.01] * 3,
            [0.01] * 3,
        ]
    )
    if kind == "centroidal":
        # EndEffectorKinematicsWeights::toVector(): position, orientation, linear velocity, angular velocity (12 entries; the rest unused)
        foot_w = np.concatenate([_ee_kinematics_weights(task, w), np.zeros(6)])

    model = dict(
        name="g1_wb" if kind == "wb" else "g1_centroidal",
        kind=kind,
        nj=nj,
        nx=nx,
        nu=nu,
        gravity=9.81,
        joint_names=joint_names,
        parent=[b["parent"] for b in bodies],
        joint_R=[b["R"].tolist() for b in bodies],
        joint_p=[b["p"].tolist() for b in bodies],
        joint_axis=[[0, 0, 0]] + [b["axis"].tolist() for b in bodies[1:]],
        mass=[b["inertia"].m for b in bodies],
        com=[b["inertia"].c.tolist() for b in bodies],
        inertia=[b["inertia"].I.tolist() for b in bodies],
        q_lower=[b["lower"] for b in bodies[1:]],
        q_upper=[b["upper"] for b in bodies[1:]],
        frame_names=[f[0] for f in frames],
        frame_body=[f[1] for f in frames],
        frame_p=[np.asarray(f[2]).tolist() for f in frames],
        contact_frames=[0, 3],  # indices into frames of foot_l_contact / foot_r_contact
        contact_rect=[rect["x_min"], rect["x_max"], rect["y_min"], rect["y_max"]],
        Q_diag=np.diag(Q).tolist(),
        R_diag=np.diag(R).tolist(),
        Qf_diag=np.diag(Qf).tolist(),
        x_init=x_init.tolist(),
        foot_gains=dict(
            pos_z=info_float(task, fc + "positionErrorGain_z"),
            ori=info_float(task, fc + "orientationErrorGain"),
            linvel_z=info_float(task, fc + "linearVelocityErrorGain_z"),
            linvel_xy=info_float(task, fc + "linearVelocityErrorGain_xy"),
            angvel=info_float(task, fc + "angularVelocityErrorGain"),
            linacc_z=info_float(task, fc + "linearAccelerationErrorGain_z"),
            linacc_xy=info_float(task, fc + "linearAccelerationErrorGain_xy"),
            angacc=info_float(task, fc + "angularAccelerationErrorGain"),
        ),
        foot_cost_weights=foot_w.tolist(),
        friction=dict(
            mu_fric=info_float(task, "contacts.frictionForceConeSoftConstraint.frictionCoefficient"),
            mu=info_float(task, "contacts.frictionForceConeSoftConstraint.mu"),
            delta=info_float(task, "contacts.frictionForceConeSoftConstraint.delta"),
            regularization=25.0,  # FrictionForceConeConstraint.h:66-69 defaults
            hessian_shift=1e-6,
        ),
        moment_xy=dict(
            mu=info_float(task, "contacts.contactMomentXYSoftConstraint.mu"),
            delta=info_float(task, "contacts.contactMomentXYSoftConstraint.delta"),
        ),
        joint_limits=dict(mu=info_float(task, "jointLimits.mu"), delta=info_float(task, "jointLimits.delta")),
        collision=dict(
            mu=info_float(task, cc + "mu"),
            delta=info_float(task, cc + "delta"),
            r_foot=info_float(task, cc + "foot.footCollisionSphereRadius"),
            r_knee=info_float(task, cc + "knee.kneeCollisionSphereRadius"),
        ),
        arm_swing_joints=[
            jidx[info_get(task, "model_settings.armJointNames." + k)]
            for k in ("left_shoulder_y", "right_shoulder_y", "left_elbow_y", "right_elbow_y")
        ],
        swing=dict(
            liftOffVelocity=info_float(task, "swing_trajectory_config.liftOffVelocity"),
            touchDownVelocity=info_float(task, "swing_trajectory_config.touchDownVelocity"),
            swingHeight=info_float(task, "swing_trajectory_config.swingHeight"),
            touchDownHeightOffset=info_float(task, "swing_trajectory_config.touchDownHeightOffset"),
            swingTimeScale=info_float(task, "swing_trajectory_config.swingTimeScale"),
            ipfLiftOffVelocity=info_float(task, "swing_trajectory_config.impactProximityFactorLiftOffVelocity"),
            ipfTouchDownVelocity=info_float(task, "swing_trajectory_config.impactProximityFactorTouchDownVelocity"),
            ipfMidPointValue=info_float(task, "swing_trajectory_config.impactProximityFactorMidPointValue"),
        ),
        sqp=dict(
            dt=info_float(task, "multiple_shooting.dt"),
            sqpIteration=int(info_float(task, "multiple_shooting.sqpIteration")),
            deltaTol=info_float(task, "multiple_shooting.deltaTol"),
            g_max=info_float(task, "multiple_shooting.g_max"),
            g_min=info_float(task, "multiple_shooting.g_min"),
            timeHorizon=info_float(task, "mpc.timeHorizon"),
        ),
    )
    if kind == "centroidal":
        model["sqp"]["timeHorizon"] = info_float(task, "mpc.timeHorizon")
        model["centroidalModelType"] = int(info_float(task, "centroidalModelType"))
        # task_space_costs: one EndEffectorKinematicsQuadraticCost per listed link (CentroidalMpcInterface.cpp:331-362); G1 lists the torso lidar link
        costs = []
        for cname, blk in task["task_space_costs"].items():
            link = blk["link_name"]
            b, R, p = link_body[link]
            costs.append(dict(name=cname, link=link, body=b, R=np.asarray(R).tolist(), p=np.asarray(p).tolist(),
                              weights=_ee_kinematics_weights(task, f"task_space_costs.{cname}.weights.").tolist()))
        assert len(costs) == 1, "the device path carries exactly one task-space link cost (G1: torso)"
        model["task_space_cost"] = costs[0]
        model["icp_weight"] = info_float(task, "icp_cost_weights.icpErrorWeight")
        # ExternalTorqueQuadraticCostAD (HumanoidCostConstraintFactory.cpp:234-245)
        tq = []
        for side in ("left_leg_torque_cost", "right_leg_torque_cost"):
            names = info_list(task, side + ".activeJointNames")
            wts = info_matrix(task[side], "weights", len(names), 1)[:, 0]
            tq.append(dict(joints=[jidx[n] for n in names], weights=wts.tolist()))
        model["leg_torque_cost"] = tq
    if reference_path is not None:
        ref = parse_info(reference_path)
        model["reference"] = dict(
            defaultBaseHeight=info_float(ref, "defaultBaseHeight"),
            defaultJointState=info_matrix(ref, "defaultJointState", nj, 1)[:, 0].tolist(),
            targetDisplacementVelocity=info_float(ref, "targetDisplacementVelocity"),
            targetRotationVelocity=info_float(ref, "targetRotationVelocity"),
            maxDeltaPelvisHeight=info_float(ref, "maxDeltaPelvisHeight"),   # the dz clamp of pose commands (getDeltaBaseTarget)
            # ProceduralMpcMotionManager's command scales (ProceduralMpcMotionManager.cpp:54-57)
            maxDisplacementVelocityX=info_float(ref, "maxDisplacementVelocityX"),
            maxDisplacementVelocityY=info_float(ref, "maxDisplacementVelocityY"),
            maxRotationVelocity=info_float(ref, "maxRotationVelocity"),
        )
    if kind == "centroidal" and "reference" in model:
        model["srbd_nominal"] = srbd_nominal(model, model["reference"]["defaultJointState"])
    if gait_path is not None:
        g = parse_info(gait_path)
        gaits = {}
        for name in info_list(g, "list"):
            if name in g:
                gaits[name] = dict(
                    modeSequence=info_list(g, name + ".modeSequence"),
                    switchingTimes=[float(v) for v in info_list(g, name + ".switchingTimes")],
                )
        model["gaits"] = gaits
    return model


def srbd_nominal(model: dict, joint_angles) -> dict:
    """createCentroidalModelInfo for the SingleRigidBodyDynamics type (ocs2_centroidal_model/src/FactoryFunctions.cpp:113-121): pinocchio::ccrba at
    q = (0_6, nominalJointAngles) -> centroidal rotational inertia (about the centre of mass; world axes = base axes there) and base - com."""
    nb = model["nj"] + 1
    R, p = [np.eye(3)], [np.zeros(3)]
    for i in range(1, nb):
        pa = model["parent"][i]
        a = np.asarray(model["joint_axis"][i], float)
        th = joint_angles[i - 1]
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        Rq = np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * (K @ K)
        R.append(R[pa] @ np.asarray(model["joint_R"][i]) @ Rq)
        p.append(p[pa] + R[pa] @ np.asarray(model["joint_p"][i]))
    ms = np.asarray(model["mass"])
    c = np.array([p[i] + R[i] @ np.asarray(model["com"][i]) for i in range(nb)])
    G = (ms[:, None] * c).sum(0) / ms.sum()
    Ig = np.zeros((3, 3))
    for i in range(nb):
        d = c[i] - G
        Ig += R[i] @ np.asarray(model["inertia"][i]) @ R[i].T + ms[i] * (d @ d * np.eye(3) - np.outer(d, d))
    return dict(inertia=Ig.tolist(), com_to_base=(-G).tolist())


def with_robot_params(model: dict, params: dict) -> dict:
    """the model dictionary whose description carries the inertial parameters of a robot-parameter record (abi.RobotParams fields), bodies
    0..nj; on an SRBD centroidal model the record's nominal inertia and com offset too"""
    m = copy.deepcopy(model)
    nb = model["nj"] + 1
    m["mass"] = [float(v) for v in np.asarray(params["mass"])[:nb]]
    m["com"] = np.asarray(params["com"], float)[:nb].tolist()
    m["inertia"] = np.asarray(params["inertia"], float)[:nb].reshape(nb, 3, 3).tolist()
    if "srbd_nominal" in m and int(m.get("centroidalModelType", 0)) == 1:
        m["srbd_nominal"] = dict(inertia=np.asarray(params["inertia_nominal"], float).reshape(3, 3).tolist(),
                                 com_to_base=np.asarray(params["com_to_base_nominal"], float).tolist())
    return m


def add_payload(params: dict, body: int, mass: float, com, inertia=None, model: dict | None = None) -> dict:
    """A robot-parameter record (abi.RobotParams fields, e.g. B200SqpSolver.default_robot_params()) with a rigid payload fixed to `body`: mass
    [kg], com [m] in the body frame, inertia (3x3 about its own com, body axes; None: a point mass).  The payload and the body are combined
    into one body with the loader's composite-inertia arithmetic (the lumping of fixed links).  With `model` (the model dictionary of the
    handle) on an SRBD centroidal model, the nominal inertia and com offset are recomputed with srbd_nominal at the default joint angles.
    Returns a new record; `params` is not changed."""
    out = {k: np.array(v, dtype=np.float64, copy=True) for k, v in params.items() if k != "custom"}
    if not mass >= 0.0:
        raise ValueError(f"add_payload: mass must be >= 0, got {mass}")
    tot = _Inertia(float(out["mass"][body]), out["com"][body], out["inertia"][body].reshape(3, 3)) + _Inertia(float(mass), com, inertia)
    out["mass"][body] = tot.m
    out["com"][body] = tot.c
    out["inertia"][body] = tot.I.reshape(9)
    if model is not None and "srbd_nominal" in model and int(model.get("centroidalModelType", 0)) == 1:
        nom = srbd_nominal(with_robot_params(model, out), model["reference"]["defaultJointState"])
        out["inertia_nominal"] = np.asarray(nom["inertia"], float).reshape(9)
        out["com_to_base_nominal"] = np.asarray(nom["com_to_base"], float)
    return out


def _ee_kinematics_weights(task, prefix) -> np.ndarray:
    """EndEffectorKinematicsWeights::getWeights + toVector (humanoid_common_mpc/src/cost/EndEffectorKinematicCostHelpers.cpp)"""
    return np.array([info_float(task, prefix + f"{k}_{a}") for k in ("pos", "orientation", "lin_velocity", "ang_velocity") for a in "xyz"])


def build_g1_centroidal_from_reference(reference_root="/root/reference") -> dict:
    r = Path(reference_root)
    return build_wb_model(r / G1_REL["urdf"], r / G1_REL["centroidal_task"], r / G1_REL["centroidal_reference"], r / G1_REL["gait"],
                          kind="centroidal")


def centroidal_settings(task_path, nj: int) -> dict:
    """The centroidal MPC's weights and grid (robot_models/unitree_g1/g1_centroidal_mpc/config/mpc/task.info): state = (h/m 6, base pose 6,
    joints nj), input = (wrench_l 6, wrench_r 6, joint velocities nj).  Same kinematic tree and contact frames as the whole-body model."""
    task = parse_info(task_path)
    nx = nu = 12 + nj
    return dict(
        nx=nx, nu=nu,
        Q_diag=np.diag(info_matrix(task, "Q", nx, nx)).tolist(),
        R_diag=np.diag(info_matrix(task, "R", nu, nu)).tolist(),
        Qf_diag=(np.diag(info_matrix(task, "Q_final", nx, nx)) * info_float(task, "terminalCostScaling")).tolist(),
        x_init=info_matrix(task, "initialState", nx, 1)[:, 0].tolist(),
        dt=info_float(task, "multiple_shooting.dt"),
        timeHorizon=info_float(task, "mpc.timeHorizon"),
        centroidalModelType=int(info_float(task, "centroidalModelType")),
    )


def build_g1_wb_from_reference(reference_root="/root/reference") -> dict:
    r = Path(reference_root)
    m = build_wb_model(r / G1_REL["urdf"], r / G1_REL["task"], r / G1_REL["reference"], r / G1_REL["gait"])
    m["centroidal"] = centroidal_settings(r / G1_REL["centroidal_task"], m["nj"])
    return m


DATA_DIR = Path(__file__).resolve().parent / "data"


def load_packaged_model(name="g1_wb") -> dict:
    """Load the committed flat description (generated by tools/make_model_data.py)."""
    return json.loads((DATA_DIR / f"{name}_model.json").read_text())


if __name__ == "__main__":
    import sys

    m = build_g1_wb_from_reference(sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
    print(json.dumps({k: m[k] for k in ("nj", "nx", "nu", "joint_names", "parent")}, indent=1))
    print("total mass", sum(m["mass"]))


def write_flat(model: dict, path) -> None:
    """Flat text form of the model dictionary for the C++ host layer (host/model_file.hpp): one `key count values...` record per line,
    numbers with 17 significant digits (round-trip exact); gaits as `gait <name> <n> <modes...> <n+1 switching times>`."""
    import numpy as np

    def rec(key, vals):
        v = np.asarray(vals, dtype=float).reshape(-1)
        return f"{key} {len(v)} " + " ".join(repr(float(x)) for x in v)

    L = [f"name 1 {model['name']}"]
    for k in ("nj", "nx", "nu", "gravity"):
        L.append(rec(k, [model[k]]))
    cen = model.get("kind") == "centroidal"
    L.append(rec("kind", [1 if cen else 0]))
    frame_body, frame_p = list(model["frame_body"]), [list(p) for p in model["frame_p"]]
    if cen:  # the task-space link rides as the last frame of the table (b200sqp_cen_desc.torso_frame), as in abi.model_desc
        ts = model["task_space_cost"]
        L.append(rec("cen_torso_frame", [len(frame_body)]))
        frame_body.append(ts["body"])
        frame_p.append(ts["p"])
        L.append(rec("cen_torso_R", ts["R"]))
        L.append(rec("cen_torso_w", ts["weights"]))
        L.append(rec("cen_icp_weight", [model["icp_weight"]]))
        L.append(rec("cen_torque_joint", [j for side in model["leg_torque_cost"] for j in side["joints"]]))
        L.append(rec("cen_torque_w", [w for side in model["leg_torque_cost"] for w in side["weights"]]))
        L.append(rec("cen_model_type", [model.get("centroidalModelType", 0)]))
        L.append(rec("cen_inertia_nominal", model["srbd_nominal"]["inertia"]))
        L.append(rec("cen_com_to_base_nominal", model["srbd_nominal"]["com_to_base"]))
    L.append(rec("frame_body", frame_body))
    L.append(rec("frame_p", frame_p))
    for k in ("parent", "joint_R", "joint_p", "joint_axis", "mass", "com", "inertia", "q_lower", "q_upper", "contact_rect",
              "Q_diag", "R_diag", "Qf_diag", "x_init", "foot_cost_weights", "arm_swing_joints"):
        L.append(rec(k, model[k]))
    g = model["foot_gains"]
    L.append(rec("foot_gains", [g[k] for k in ("pos_z", "ori", "linvel_z", "linvel_xy", "angvel", "linacc_z", "linacc_xy", "angacc")]))
    f = model["friction"]
    L.append(rec("friction", [f[k] for k in ("mu_fric", "mu", "delta", "regularization", "hessian_shift")]))
    L.append(rec("moment_xy", [model["moment_xy"]["mu"], model["moment_xy"]["delta"]]))
    L.append(rec("joint_limits", [model["joint_limits"]["mu"], model["joint_limits"]["delta"]]))
    c = model["collision"]
    L.append(rec("collision", [c["mu"], c["delta"], c["r_foot"], c["r_knee"]]))
    sw = model["swing"]
    L.append(rec("swing", [sw[k] for k in ("liftOffVelocity", "touchDownVelocity", "swingHeight", "touchDownHeightOffset", "swingTimeScale",
                                           "ipfLiftOffVelocity", "ipfTouchDownVelocity", "ipfMidPointValue")]))
    sq = model["sqp"]
    L.append(rec("sqp", [sq[k] for k in ("dt", "sqpIteration", "deltaTol", "g_max", "g_min", "timeHorizon")]))
    r = model["reference"]
    L.append(rec("default_base_height", [r["defaultBaseHeight"]]))
    L.append(rec("default_joint_state", r["defaultJointState"]))
    L.append(rec("velocity_scales", [r[k] for k in ("maxDisplacementVelocityX", "maxDisplacementVelocityY", "maxRotationVelocity")]))
    L.append(rec("pose_command", [r[k] for k in ("targetDisplacementVelocity", "targetRotationVelocity", "maxDeltaPelvisHeight")]))
    for name, gt in model["gaits"].items():
        L.append(f"gait {name} {len(gt['modeSequence'])} " + " ".join(gt["modeSequence"]) + " " + " ".join(repr(float(t)) for t in gt["switchingTimes"]))
    from pathlib import Path

    Path(path).write_text("\n".join(L) + "\n")
