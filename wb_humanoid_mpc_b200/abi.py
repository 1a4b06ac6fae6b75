"""ctypes mirrors of the plain-data structs in include/b200sqp.h."""
from __future__ import annotations

import ctypes as C

import numpy as np

MAX_BODIES = 32
MAX_FRAMES = 16


class ModelDesc(C.Structure):
    _fields_ = [
        ("nj", C.c_int32),
        ("parent", C.c_int32 * MAX_BODIES),
        ("joint_R", (C.c_double * 9) * MAX_BODIES),
        ("joint_p", (C.c_double * 3) * MAX_BODIES),
        ("joint_axis", (C.c_double * 3) * MAX_BODIES),
        ("mass", C.c_double * MAX_BODIES),
        ("com", (C.c_double * 3) * MAX_BODIES),
        ("inertia", (C.c_double * 9) * MAX_BODIES),
        ("q_lower", C.c_double * MAX_BODIES),
        ("q_upper", C.c_double * MAX_BODIES),
        ("n_frames", C.c_int32),
        ("frame_body", C.c_int32 * MAX_FRAMES),
        ("frame_p", (C.c_double * 3) * MAX_FRAMES),
        ("gravity", C.c_double),
        ("contact_rect", C.c_double * 4),
        ("Q_diag", C.c_double * 64),
        ("R_diag", C.c_double * 48),
        ("Qf_diag", C.c_double * 64),
        ("foot_gain_pos_z", C.c_double),
        ("foot_gain_ori", C.c_double),
        ("foot_gain_linvel_z", C.c_double),
        ("foot_gain_linvel_xy", C.c_double),
        ("foot_gain_angvel", C.c_double),
        ("foot_gain_linacc_z", C.c_double),
        ("foot_gain_linacc_xy", C.c_double),
        ("foot_gain_angacc", C.c_double),
        ("foot_cost_w", C.c_double * 18),
        ("fric_coeff", C.c_double),
        ("fric_mu", C.c_double),
        ("fric_delta", C.c_double),
        ("fric_reg", C.c_double),
        ("fric_hess_shift", C.c_double),
        ("momxy_mu", C.c_double),
        ("momxy_delta", C.c_double),
        ("jlim_mu", C.c_double),
        ("jlim_delta", C.c_double),
        ("coll_mu", C.c_double),
        ("coll_delta", C.c_double),
        ("coll_r_foot", C.c_double),
        ("coll_r_knee", C.c_double),
        ("arm_swing_joint", C.c_int32 * 4),
    ]


class CenDesc(C.Structure):
    _fields_ = [
        ("torso_frame", C.c_int32),
        ("torso_R", C.c_double * 9),
        ("torso_w", C.c_double * 12),
        ("icp_weight", C.c_double),
        ("torque_joint", (C.c_int32 * 6) * 2),
        ("torque_w", (C.c_double * 6) * 2),
        ("model_type", C.c_int32),
        ("inertia_nominal", C.c_double * 9),
        ("com_to_base_nominal", C.c_double * 3),
    ]


class Settings(C.Structure):
    _fields_ = [
        ("sqp_iteration", C.c_int32),
        ("delta_tol", C.c_double),
        ("cost_tol", C.c_double),
        ("alpha_decay", C.c_double),
        ("alpha_min", C.c_double),
        ("gamma_c", C.c_double),
        ("g_max", C.c_double),
        ("g_min", C.c_double),
        ("armijo_factor", C.c_double),
        ("reg_prim", C.c_double),
        ("use_feedback_policy", C.c_int32),
        ("global_step", C.c_int32),
        ("create_value_function", C.c_int32),
    ]


class IterLog(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("base_merit", "base_cost", "base_dyn_sse", "base_eq_sse", "merit", "cost", "dyn_sse", "eq_sse",
                                          "step_size", "step_type", "dx_norm", "du_norm", "armijo", "convergence")] + [("pad", C.c_double * 2)]


class RolloutSettings(C.Structure):
    _fields_ = [
        ("abs_tol", C.c_double),
        ("rel_tol", C.c_double),
        ("time_step", C.c_double),
        ("max_steps_per_second", C.c_double),
    ]


def default_rollout_settings(**over) -> RolloutSettings:
    """rollout::Settings of the G1 whole-body task.info (ODE45, AbsTolODE 1e-5, RelTolODE 1e-3, timeStep 0.015, maxNumStepsPerSecond 10000),
    then keyword overrides."""
    s = RolloutSettings(abs_tol=1e-5, rel_tol=1e-3, time_step=0.015, max_steps_per_second=10000.0)
    for k, v in over.items():
        setattr(s, k, v)
    return s


def cen_default_rollout_settings(**over) -> RolloutSettings:
    """rollout::Settings of the G1 centroidal task.info (ODE45, AbsTolODE 5e-5, RelTolODE 5e-3, timeStep 0.015, maxNumStepsPerSecond 10000), the
    roll-out of the centroidal dummy simulation (b200sqp_cen_rollout_policy), then keyword overrides."""
    return default_rollout_settings(**{"abs_tol": 5e-5, "rel_tol": 5e-3, **over})


def default_settings(model: dict | None = None, **over) -> Settings:
    """sqp::Settings defaults (SqpSettings.h:42-86) overridden by the G1 task.info values, then by keyword arguments."""
    s = Settings(sqp_iteration=1, delta_tol=1e-4, cost_tol=1e-4, alpha_decay=0.5, alpha_min=1e-4, gamma_c=1e-6, g_max=1e-2, g_min=1e-6,
                 armijo_factor=1e-4, reg_prim=1e-12, use_feedback_policy=0, global_step=0, create_value_function=0)
    if model is not None:
        sq = model["sqp"]
        s.sqp_iteration, s.delta_tol, s.g_max, s.g_min = sq["sqpIteration"], sq["deltaTol"], sq["g_max"], sq["g_min"]
    for k, v in over.items():
        setattr(s, k, v)
    return s


def model_desc(model: dict) -> ModelDesc:
    """Flat model dictionary (model_loader.build_wb_model) -> b200sqp_model_desc."""
    d = ModelDesc()
    nj = model["nj"]
    nb = nj + 1
    assert nb <= MAX_BODIES and len(model["frame_body"]) <= MAX_FRAMES
    d.nj = nj
    for i in range(nb):
        d.parent[i] = model["parent"][i]
        R = np.asarray(model["joint_R"][i]).reshape(9)
        I = np.asarray(model["inertia"][i]).reshape(9)
        for k in range(9):
            d.joint_R[i][k] = R[k]
            d.inertia[i][k] = I[k]
        for k in range(3):
            d.joint_p[i][k] = model["joint_p"][i][k]
            d.joint_axis[i][k] = model["joint_axis"][i][k]
            d.com[i][k] = model["com"][i][k]
        d.mass[i] = model["mass"][i]
    for j in range(nj):
        d.q_lower[j] = model["q_lower"][j]
        d.q_upper[j] = model["q_upper"][j]
    d.n_frames = len(model["frame_body"])
    for f in range(d.n_frames):
        d.frame_body[f] = model["frame_body"][f]
        for k in range(3):
            d.frame_p[f][k] = model["frame_p"][f][k]
    if model.get("kind") == "centroidal":  # the task-space link rides as one more frame of the table
        ts = model["task_space_cost"]
        f = d.n_frames
        d.frame_body[f] = ts["body"]
        for k in range(3):
            d.frame_p[f][k] = ts["p"][k]
        d.n_frames = f + 1
    d.gravity = model["gravity"]
    for k in range(4):
        d.contact_rect[k] = model["contact_rect"][k]
    for i, v in enumerate(model["Q_diag"]):
        d.Q_diag[i] = v
    for i, v in enumerate(model["R_diag"]):
        d.R_diag[i] = v
    for i, v in enumerate(model["Qf_diag"]):
        d.Qf_diag[i] = v
    g = model["foot_gains"]
    d.foot_gain_pos_z, d.foot_gain_ori = g["pos_z"], g["ori"]
    d.foot_gain_linvel_z, d.foot_gain_linvel_xy, d.foot_gain_angvel = g["linvel_z"], g["linvel_xy"], g["angvel"]
    d.foot_gain_linacc_z, d.foot_gain_linacc_xy, d.foot_gain_angacc = g["linacc_z"], g["linacc_xy"], g["angacc"]
    for i, v in enumerate(model["foot_cost_weights"]):
        d.foot_cost_w[i] = v
    f = model["friction"]
    d.fric_coeff, d.fric_mu, d.fric_delta, d.fric_reg, d.fric_hess_shift = f["mu_fric"], f["mu"], f["delta"], f["regularization"], f["hessian_shift"]
    d.momxy_mu, d.momxy_delta = model["moment_xy"]["mu"], model["moment_xy"]["delta"]
    d.jlim_mu, d.jlim_delta = model["joint_limits"]["mu"], model["joint_limits"]["delta"]
    c = model["collision"]
    d.coll_mu, d.coll_delta, d.coll_r_foot, d.coll_r_knee = c["mu"], c["delta"], c["r_foot"], c["r_knee"]
    for i in range(4):
        d.arm_swing_joint[i] = model["arm_swing_joints"][i]
    return d


def cen_desc(model: dict) -> CenDesc:
    """Centroidal model dictionary (model_loader.build_g1_centroidal_from_reference) -> b200sqp_cen_desc."""
    assert model.get("kind") == "centroidal"
    c = CenDesc()
    ts = model["task_space_cost"]
    c.torso_frame = len(model["frame_body"])
    R = np.asarray(ts["R"]).reshape(9)
    for k in range(9):
        c.torso_R[k] = R[k]
    for k in range(12):
        c.torso_w[k] = ts["weights"][k]
    c.icp_weight = model["icp_weight"]
    for s in range(2):
        for k in range(6):
            c.torque_joint[s][k] = model["leg_torque_cost"][s]["joints"][k]
            c.torque_w[s][k] = model["leg_torque_cost"][s]["weights"][k]
    c.model_type = int(model.get("centroidalModelType", 0))
    I = np.asarray(model["srbd_nominal"]["inertia"]).reshape(9)
    for k in range(9):
        c.inertia_nominal[k] = I[k]
    for k in range(3):
        c.com_to_base_nominal[k] = model["srbd_nominal"]["com_to_base"][k]
    return c


MAX_GAITS = 16
MAX_GAIT_MODES = 8
MODE_NUMBER = {"FLY": 0, "RF": 1, "LF": 2, "STANCE": 3}


class BuilderDesc(C.Structure):
    _fields_ = [
        ("n_gaits", C.c_int32),
        ("gait_n_modes", C.c_int32 * MAX_GAITS),
        ("gait_modes", (C.c_int32 * MAX_GAIT_MODES) * MAX_GAITS),
        ("gait_switching_times", (C.c_double * (MAX_GAIT_MODES + 1)) * MAX_GAITS),
        ("swing", C.c_double * 8),
        ("default_joint_state", C.c_double * MAX_BODIES),
        ("total_mass", C.c_double),
        ("dt", C.c_double),
    ]


def builder_desc(model: dict) -> tuple[BuilderDesc, list[str]]:
    """b200sqp_builder_desc of the device-side instance builder + the gait names in table order (gait id = index).  The "stance" entry is the
    default schedule of GaitSchedule (STANCE phases of 0.5 s)."""
    d = BuilderDesc()
    names = list(model["gaits"].keys())
    assert len(names) <= MAX_GAITS
    d.n_gaits = len(names)
    for g, name in enumerate(names):
        gt = model["gaits"][name]
        modes = [m if isinstance(m, int) else MODE_NUMBER[m] for m in gt["modeSequence"]]
        assert 1 <= len(modes) <= MAX_GAIT_MODES
        times = [float(t) for t in gt["switchingTimes"]]
        if any(b <= a for a, b in zip(times, times[1:])):
            continue   # gait.info's "skip" template has a decreasing switching time (0.75 -> 0.08): left out of the device table (n_modes = 0)
        d.gait_n_modes[g] = len(modes)
        for i, m in enumerate(modes):
            d.gait_modes[g][i] = m
        for i, t in enumerate(gt["switchingTimes"]):
            d.gait_switching_times[g][i] = float(t)
    sw = model["swing"]
    for i, k in enumerate(["liftOffVelocity", "touchDownVelocity", "swingHeight", "touchDownHeightOffset", "swingTimeScale", "ipfLiftOffVelocity",
                           "ipfTouchDownVelocity", "ipfMidPointValue"]):
        d.swing[i] = float(sw[k])
    for j, q in enumerate(model["reference"]["defaultJointState"]):
        d.default_joint_state[j] = float(q)
    d.total_mass = float(sum(model["mass"]))
    d.dt = float(model["sqp"]["dt"])
    return d, names


MOTION_GAITS = ["stance", "slow_walk", "walk", "slower_trot", "slow_trot", "trot", "run"]   # the states of ProceduralMpcMotionManager


class MotionDesc(C.Structure):
    _fields_ = [
        ("gait", C.c_int32 * 7),
        ("max_velocity_x", C.c_double),
        ("max_velocity_y", C.c_double),
        ("max_rotation_velocity", C.c_double),
        ("filter_origin", C.c_double),
    ]


def motion_desc(model: dict, gait_names: list[str], filter_origin: float = 0.0) -> MotionDesc:
    """b200sqp_motion_desc: the builder gait ids of the manager's seven states (gait_names = builder_desc's table order) and the velocity
    scales of reference.info"""
    missing = [g for g in MOTION_GAITS if g not in gait_names]
    if missing:
        raise ValueError(f"the motion manager needs the gaits {missing} in gait.info (the builder's gait table has {gait_names})")
    d = MotionDesc()
    for s, g in enumerate(MOTION_GAITS):
        d.gait[s] = gait_names.index(g)
    r = model["reference"]
    d.max_velocity_x = float(r["maxDisplacementVelocityX"])
    d.max_velocity_y = float(r["maxDisplacementVelocityY"])
    d.max_rotation_velocity = float(r["maxRotationVelocity"])
    d.filter_origin = float(filter_origin)
    return d


class PoseDesc(C.Structure):
    _fields_ = [
        ("target_displacement_velocity", C.c_double),
        ("target_rotation_velocity", C.c_double),
        ("max_delta_pelvis_height", C.c_double),
        ("default_base_height", C.c_double),
    ]


def pose_desc(model: dict) -> PoseDesc:
    """b200sqp_pose_desc from model["reference"] (reference.info targetDisplacementVelocity, targetRotationVelocity, maxDeltaPelvisHeight,
    defaultBaseHeight)"""
    r = model["reference"]
    return PoseDesc(float(r["targetDisplacementVelocity"]), float(r["targetRotationVelocity"]), float(r["maxDeltaPelvisHeight"]),
                    float(r["defaultBaseHeight"]))


RESET_REASONS = ["none", "requested", "non_finite", "solve", "rollout", "height", "pitch", "roll"]   # b200sqp_download_episodes reason codes


class AutoResetDesc(C.Structure):
    _fields_ = [
        ("on_solve_failure", C.c_int32),
        ("on_rollout_failure", C.c_int32),
        ("max_height_deviation", C.c_double),
        ("max_pitch_deviation", C.c_double),
        ("max_roll_deviation", C.c_double),
    ]


class Gains(C.Structure):
    """b200sqp_gains: the per-instance cost weights and soft-constraint penalties of b200sqp_set_gains"""
    _fields_ = [
        ("Q_diag", C.c_double * 64),
        ("R_diag", C.c_double * 48),
        ("Qf_diag", C.c_double * 64),
        ("foot_cost_w", C.c_double * 18),
        ("torso_w", C.c_double * 12),
        ("jlim_mu", C.c_double), ("jlim_delta", C.c_double),
        ("coll_mu", C.c_double), ("coll_delta", C.c_double), ("coll_r_foot", C.c_double), ("coll_r_knee", C.c_double),
        ("fric_mu", C.c_double), ("fric_delta", C.c_double),
        ("momxy_mu", C.c_double), ("momxy_delta", C.c_double),
        ("final_cost_active", C.c_int32), ("foot_cost_active", C.c_int32), ("torso_cost_active", C.c_int32), ("joint_limits_active", C.c_int32),
        ("foot_collision_active", C.c_int32), ("friction_cone_active", C.c_int32), ("contact_moment_active", C.c_int32),
    ]


GAINS_DTYPE = np.dtype(Gains)          # the C layout as a numpy structured dtype (offsets and padding included)
GAINS_BYTES = C.sizeof(Gains)
GAIN_FIELDS = [f[0] for f in Gains._fields_]


def pack_gains(gains: dict, count: int | None = None) -> np.ndarray:
    """{field: array with a leading count axis} -> uint8 [count][GAINS_BYTES] in the b200sqp_gains layout (the rows of b200sqp_set_gains, or of
    b200sqp_set_gains_dev once copied to the device).  Every field is required; with `count` given, a single record's values are repeated."""
    missing = [k for k in GAIN_FIELDS if k not in gains]
    if missing:
        raise KeyError(f"pack_gains: missing fields {missing}")
    if count is None:
        count = int(np.shape(gains["final_cost_active"])[0]) if np.ndim(gains["final_cost_active"]) else 1
    rec = np.zeros(count, dtype=GAINS_DTYPE)
    for k in GAIN_FIELDS:
        rec[k] = gains[k]
    return rec.view(np.uint8).reshape(count, GAINS_BYTES)


def unpack_gains(rec: np.ndarray) -> dict:
    """uint8 [count][GAINS_BYTES] (or a GAINS_DTYPE array) -> {field: array with a leading count axis}"""
    rec = np.ascontiguousarray(rec)
    if rec.dtype != GAINS_DTYPE:
        rec = rec.reshape(-1, GAINS_BYTES).view(GAINS_DTYPE).reshape(-1)
    return {k: rec[k].copy() for k in GAIN_FIELDS}
