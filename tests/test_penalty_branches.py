"""The soft-constraint penalties of the LQ approximation where they act, without a GPU: foot collision and joint limits (piecewise-polynomial
barrier) in their polynomial pieces, the friction cone and the contact-moment rows (relaxed barrier) in their relaxed branch, and the exact
thresholds between branches.  The instances of the parity tests keep four of the six terms inactive or in their log branch, so this file
builds linearisation trajectories that reach every branch, asserts that they do (the counts of node x row per branch are printed), and pins:

- the two penalty functions of the device (through the CPU harness) and of the oracle (through its cost and quadratic cost) against a
  restatement in exact arithmetic (fractions for the polynomial pieces, mpmath or long double for the log);
- the oracle's cost gradient against central finite differences, and each term's Hessian against a NumPy Gauss-Newton assembly;
- the whole-body K1 node of the CPU harness (all three schedules) and the centroidal node against the oracle on every node of every recipe.

tests/test_gpu_penalty_branches.py runs the same recipes through the C ABI on the GPU."""
import copy
from collections import Counter
from fractions import Fraction

import numpy as np
import pytest

import emu_lib as emu
import oracle_lib as orc
from test_gpu_cen_ocp import make_instance as cen_make_instance
from test_gpu_wb import make_instances
from wb_humanoid_mpc_b200 import abi, model_loader

try:
    import mpmath
except ImportError:   # long double fallback for the log branch
    mpmath = None

# FootCollisionConstraint (humanoid_common_mpc/src/constraint/FootCollisionConstraint.cpp:112-137), by frame name; row 9 is the knee pair
COLLISION_PAIRS = [("foot_l_contact_collision_p_1", "foot_r_contact_collision_p_1"), ("foot_l_contact_collision_p_1", "foot_r_contact_collision_p_2"),
                   ("foot_l_contact_collision_p_2", "foot_r_contact_collision_p_1"), ("foot_l_contact_collision_p_2", "foot_r_contact_collision_p_2"),
                   ("foot_l_contact", "foot_r_contact_collision_p_1"), ("foot_l_contact", "foot_r_contact_collision_p_2"),
                   ("foot_r_contact", "foot_l_contact_collision_p_1"), ("foot_r_contact", "foot_l_contact_collision_p_2"),
                   ("foot_l_contact", "foot_r_contact"), ("left_knee_joint", "right_knee_joint"),
                   ("foot_l_contact", "right_ankle_roll_joint"), ("foot_l_contact_collision_p_1", "right_ankle_roll_joint"),
                   ("foot_l_contact_collision_p_2", "right_ankle_roll_joint"), ("foot_r_contact", "left_ankle_roll_joint"),
                   ("foot_r_contact_collision_p_1", "left_ankle_roll_joint"), ("foot_r_contact_collision_p_2", "left_ankle_roll_joint")]
KNEE_ROW = 9
WALK_CMD = [0.3, 0.0, 0.7925, 0.1]


# ---- exact restatement of the two penalties ---------------------------------------------------------------------------------------------------

def pwpoly_exact(mu, delta, h):
    """PieceWisePolynomialBarrierPenalty (ocs2_core/src/penalties/penalties/PieceWisePolynomialBarrierPenalty.cpp:37-75) in rationals"""
    mu, delta, h = Fraction(mu), Fraction(delta), Fraction(h)
    if h <= 0:
        return mu * (h * h / 2 - delta * h / 2 + delta * delta / 6), mu * (h - delta / 2), mu
    if h < delta:
        return (mu * (-h ** 3 / (6 * delta) + h * h / 2 - delta * h / 2 + delta * delta / 6), mu * (-h * h / (2 * delta) + h - delta / 2),
                mu * (1 - h / delta))
    return Fraction(0), Fraction(0), Fraction(0)


def _log(h):
    if mpmath is not None:
        with mpmath.workdps(40):
            return Fraction(str(mpmath.log(mpmath.mpf(float(h)))))
    return Fraction(float(np.log(np.longdouble(float(h)))))


def relaxed_exact(mu, delta, h):
    """RelaxedBarrierPenalty (ocs2_core/src/penalties/penalties/RelaxedBarrierPenalty.cpp:37-66): polynomial parts in rationals, the log
    at 40 digits (mpmath) or in long double"""
    mu, delta, h = Fraction(mu), Fraction(delta), Fraction(h)
    if h > delta:
        return -mu * _log(h), -mu / h, mu / (h * h)
    dh = (h - 2 * delta) / delta
    return mu * (-_log(delta) + dh * dh / 2 - Fraction(1, 2)), mu * (h - 2 * delta) / (delta * delta), mu / (delta * delta)


def assert_penalty_close(got, mu, delta, h, exact, what):
    """v, d1, d2 within about ten units in the last place of the exact value, or of the scale of the terms that cancel in it
    (mu (delta^2 + h^2 + |log|), mu (delta + |h| + 1 / delta), mu (1 + 1 / delta^2))"""
    v, d1, d2 = (float(e) for e in exact)
    scale_v = mu * (delta * delta + h * h + 1.0 + abs(float(np.log(max(abs(h), delta)))))
    scale_1 = mu * (delta + abs(h) + 1.0 / delta)
    scale_2 = mu * (1.0 + 1.0 / (delta * delta))
    for g, e, s, name in ((got[0], v, scale_v, "v"), (got[1], d1, scale_1, "d1"), (got[2], d2, scale_2, "d2")):
        assert abs(g - e) <= 2e-15 * (abs(e) + s), (what, name, h, g, e)


def threshold_points(delta):
    """both sides of every threshold of either penalty, and exactly on it"""
    up, dn = lambda v: float(np.nextafter(v, np.inf)), lambda v: float(np.nextafter(v, -np.inf))
    return [-2 * delta, -delta, dn(0.0), 0.0, up(0.0), 0.25 * delta, 0.5 * delta, dn(delta), delta, up(delta), 1.5 * delta, 2 * delta, 10 * delta]


# ---- branch bookkeeping ------------------------------------------------------------------------------------------------------------------------

def pw_branch(h, delta):
    return "h<=0" if h <= 0 else ("0<h<delta" if h < delta else "off")


def relaxed_branch(h, delta):
    return "relaxed" if h <= delta else "log"


def is_cen(model):
    return model.get("kind") == "centroidal"


class Geometry:
    """the penalty constraint values h of a node, from oracle quantities: frame positions and foot rotations of WbOracle.foot_state (the
    centroidal state maps onto the whole-body state of the same robot: base pose, joint positions), joint limits and the wrenches of u"""

    def __init__(self, model):
        self.model = model
        self.cen = is_cen(model)
        self.wb = orc.WbOracle(model_loader.load_packaged_model())
        names = self.wb.model["frame_names"]
        self.pairs = [(names.index(a), names.index(b)) for a, b in COLLISION_PAIRS]
        self.qlo, self.qhi = np.array(model["q_lower"]), np.array(model["q_upper"])
        c, f, mxy = model["collision"], model["friction"], model["moment_xy"]
        self.r2 = np.array([2 * (c["r_knee"] if r == KNEE_ROW else c["r_foot"]) for r in range(16)])
        self.rect = model["contact_rect"] if "contact_rect" in model else self.wb.model["contact_rect"]
        self.mu_c, self.reg = f["mu_fric"], f["regularization"]
        self.jl_delta, self.coll_delta, self.fric_delta, self.mom_delta = model["joint_limits"]["delta"], c["delta"], f["delta"], mxy["delta"]

    def q(self, x):
        return x[12:35] if self.cen else x[6:29]

    def wb_state(self, x, u):
        if not self.cen:
            return x, u
        xw = np.zeros(58)
        xw[0:6], xw[6:29] = x[6:12], x[12:35]
        uw = np.zeros(35)
        uw[:12] = u[:12]
        return xw, uw

    def feet(self, x, u):
        xw, uw = self.wb_state(x, u)
        return self.wb.foot_state(xw, uw)

    def joint_limits(self, x):
        """46 values: upper (q_hi - q) then lower (q - q_lo), in the arithmetic of both codes"""
        q = self.q(x)
        return np.concatenate([self.qhi - q, q - self.qlo])

    def collision(self, x, u):
        _, fp = self.feet(x, u)
        return np.array([np.sqrt(np.dot(fp[a] - fp[b], fp[a] - fp[b])) for a, b in self.pairs]) - self.r2

    def friction(self, u, c):
        F = u[6 * c:6 * c + 3]
        return self.mu_c * F[2] - np.sqrt(F[0] * F[0] + F[1] * F[1] + self.reg)

    def moment(self, x, u, c):
        feet, _ = self.feet(x, u)
        R = feet[c]["R"]
        lf, lm = R.T @ u[6 * c:6 * c + 3], R.T @ u[6 * c + 3:6 * c + 6]
        r = self.rect
        return np.array([lm[0] - r[2] * lf[2], -lm[0] + r[3] * lf[2], -lm[1] - r[0] * lf[2], lm[1] + r[1] * lf[2]])

    def moments_for(self, x, u, c, row, target):
        """the world moment of foot c that puts contact-moment row `row` at h = target (the other component of the local moment zero)"""
        feet, _ = self.feet(x, u)
        R = feet[c]["R"]
        lfz = (R.T @ u[6 * c:6 * c + 3])[2]
        r = self.rect
        lm = np.zeros(3)
        if row == 0:
            lm[0] = target + r[2] * lfz
        elif row == 1:
            lm[0] = r[3] * lfz - target
        elif row == 2:
            lm[1] = -r[0] * lfz - target
        else:
            lm[1] = target - r[1] * lfz
        return R @ lm

    def node_values(self, inst, k):
        """{term: array of h} of the stage cost of node k, only the rows its contact mode evaluates"""
        x, u = inst["x_init"][k], inst["u_init"][k]
        cf = inst["contact_flags"][k]
        out = dict(joint_limits=self.joint_limits(x))
        if not (cf[0] and cf[1]):
            out["collision"] = self.collision(x, u)
        out["friction"] = np.array([self.friction(u, c) for c in range(2) if cf[c]])
        out["moment"] = np.concatenate([self.moment(x, u, c) for c in range(2) if cf[c]] or [np.zeros(0)])
        return out

    def counts(self, inst, deltas=None):
        """Counter {(term, branch): node x row} over the intermediate nodes; 'edge' entries count values exactly on a threshold"""
        d = dict(joint_limits=self.jl_delta, collision=self.coll_delta, friction=self.fric_delta, moment=self.mom_delta)
        d.update(deltas or {})
        cnt = Counter()
        for k in stage_nodes(inst):
            for term, h in self.node_values(inst, k).items():
                for r, v in enumerate(h):
                    if term in ("joint_limits", "collision"):
                        cnt[(term, pw_branch(v, d[term]))] += 1
                        if v == 0.0:
                            cnt[(term, "edge h=0")] += 1
                        if v == d[term]:
                            cnt[(term, "edge h=delta")] += 1
                        if term == "collision" and r == KNEE_ROW and v < d[term]:
                            cnt[("collision", "knee row active")] += 1
                    else:
                        cnt[(term, relaxed_branch(v, d[term]))] += 1
                        if v == d[term]:
                            cnt[(term, "edge h=delta")] += 1
            if "collision" in self.node_values(inst, k):
                h = self.collision(inst["x_init"][k], inst["u_init"][k])
                act = h < d["collision"]
                if act[KNEE_ROW] and act.sum() == 1:
                    cnt[("collision", "knee row alone")] += 1
                if not inst["contact_flags"][k].any() and act.any():
                    cnt[("collision", "flight node active")] += 1
        return cnt


def stage_nodes(inst):
    """nodes with a stage cost: intermediate nodes that are not event (jump) nodes"""
    n = len(inst["t_nodes"])
    return [k for k in range(n - 1) if inst["node_event"][k] == 0]


def format_counts(name, cnt):
    return f"{name}: " + ", ".join(f"{t}/{b} {v}" for (t, b), v in sorted(cnt.items()))


# ---- recipes -----------------------------------------------------------------------------------------------------------------------------------

class Layout:
    """state indices of a family: joint positions, base orientation (yaw, pitch, roll)"""

    def __init__(self, model):
        self.cen = is_cen(model)
        self.q0 = 12 if self.cen else 6
        self.ori = 9 if self.cen else 3


def base_instance(model, gait="walk", horizon=0.8, seed=2):
    if is_cen(model):
        return cen_make_instance(model, np.random.default_rng(seed), gait, horizon, WALK_CMD)
    return make_instances(model, np.random.default_rng(seed), [(gait, horizon, WALK_CMD)])[0]


def _copy(inst):
    """a copy whose linearisation trajectory the recipes overwrite.  Inputs are only written on nodes with a stage cost: an event (jump)
    node has no input in the reference (Initialization.cpp: "no input at event node"), the builder leaves it zero, and the oracle and the
    device treat a nonzero one differently (the oracle clears it, the device keeps it), which no caller can produce."""
    out = dict(inst)
    out["x_init"], out["u_init"] = inst["x_init"].copy(), inst["u_init"].copy()
    return out


def cross_legs(model, inst, lo, hi):
    """hip rolls inward, ramped from lo to hi rad over the nodes: the feet (and ankles) cross into each other's collision spheres"""
    L = Layout(model)
    n = len(inst["t_nodes"])
    for k, roll in enumerate(np.linspace(lo, hi, n)):
        inst["x_init"][k, L.q0 + 1] = -roll
        inst["x_init"][k, L.q0 + 7] = roll
    return inst


def knees_together(model, inst):
    """hips rotated outward, flexed and rolled inward: the knees meet while the feet stay apart (the knee row alone)"""
    L = Layout(model)
    n = len(inst["t_nodes"])
    for k, roll in enumerate(np.linspace(0.2, 0.32, n)):
        x = inst["x_init"][k]
        x[L.q0 + 0] = x[L.q0 + 6] = -0.6
        x[L.q0 + 3] = x[L.q0 + 9] = 1.2
        x[L.q0 + 2], x[L.q0 + 8] = -0.3, 0.3
        x[L.q0 + 1], x[L.q0 + 7] = -roll, roll
    return inst


# (joint, bound): leg, waist and arm joints pushed onto a limit; the distance to the bound is ramped from past it to beyond delta
LIMIT_JOINTS = [(3, "lo"), (4, "hi"), (11, "hi"), (13, "lo"), (14, "hi"), (16, "hi"), (18, "lo"), (20, "hi"), (21, "lo")]


def joints_at_limits(model, inst):
    L = Layout(model)
    qlo, qhi = np.array(model["q_lower"]), np.array(model["q_upper"])
    n = len(inst["t_nodes"])
    for k, off in enumerate(np.linspace(-0.04, 0.13, n)):
        for i, (j, side) in enumerate(LIMIT_JOINTS):
            o = off if i % 2 == 0 else 0.09 - off   # half of the joints ramp the other way: every node has both pieces
            inst["x_init"][k, L.q0 + j] = qhi[j] - o if side == "hi" else qlo[j] + o
    return inst


def exact_thresholds(model, inst):
    """joints exactly at q_hi - delta, q_hi, q_lo + delta, q_lo (h computed as both codes compute it: only joints whose limit is small
    enough for q_hi - q or q - q_lo to round to delta can sit exactly on it), and a friction cone at h = delta"""
    L = Layout(model)
    qlo, qhi = np.array(model["q_lower"]), np.array(model["q_upper"])
    delta = model["joint_limits"]["delta"]

    def solve(f, target, x, increasing):   # a float x with f(x) == target exactly, searched ulp by ulp around x
        for _ in range(64):
            v = f(x)
            if v == target:
                return x
            x = float(np.nextafter(x, np.inf if (v < target) == increasing else -np.inf))
        raise AssertionError("no exact threshold found")

    n = len(inst["t_nodes"])
    for k in range(n):
        x = inst["x_init"][k]
        x[L.q0 + 5] = solve(lambda v: qhi[5] - v, delta, qhi[5] - delta, False)    # left ankle roll: upper h = delta
        x[L.q0 + 11] = solve(lambda v: v - qlo[11], delta, qlo[11] + delta, True)   # right ankle roll: lower h = delta
        x[L.q0 + 4] = qhi[4]                                                        # left ankle pitch: upper h = 0
        x[L.q0 + 10] = qlo[10]                                                      # right ankle pitch: lower h = 0
    f = model["friction"]
    fz = (f["delta"] + np.sqrt(f["regularization"])) / f["mu_fric"]
    for k in stage_nodes(inst):
        if inst["contact_flags"][k][0]:
            u = inst["u_init"][k]
            u[0:3] = [0.0, 0.0, fz]
    return inst


def unload_feet(model, geo, inst, fz_lo=2.0, fz_hi=45.0):
    """left foot unloaded, fz ramped from fz_lo to fz_hi over the nodes, with tangential forces (the regularised norm and the off-diagonal
    second derivatives of the cone matter); the right foot carries the rest, with the opposite tangential force"""
    n = len(inst["t_nodes"])
    mg = sum(model["mass"]) * 9.81
    for k, fz in enumerate(np.linspace(fz_lo, fz_hi, n - 1)):
        if inst["node_event"][k] == 1:
            continue
        cf, u = inst["contact_flags"][k], inst["u_init"][k]
        if cf[0]:
            u[0:3] = [3.0, -2.0, fz]
            if cf[1]:
                u[6:9] = [-3.0, 2.0, mg - fz]
        elif cf[1]:
            u[6:9] = [-1.5, 4.0, 0.5 * fz]
    return inst


def edge_moments(model, geo, inst, lo=-0.02, hi=0.05):
    """the local moment of each stance foot places one contact-moment row at h in [lo, hi], a different row at each node"""
    n = len(inst["t_nodes"])
    for k, target in enumerate(np.linspace(lo, hi, n - 1)):
        if inst["node_event"][k] == 1:
            continue
        cf, x, u = inst["contact_flags"][k], inst["x_init"][k], inst["u_init"][k]
        for c in range(2):
            if cf[c]:
                M = geo.moments_for(x, u, c, (k + 2 * c) % 4, target)
                u[6 * c + 3:6 * c + 6] = M
    return inst


def rotate_base(model, inst, pitch, roll):
    """large base orientation on the linearisation trajectory: yaw ramped across +-pi, pitch and roll of about 0.6 rad"""
    L = Layout(model)
    n = len(inst["t_nodes"])
    inst["x_init"][:, L.ori] = np.linspace(np.pi - 0.35, np.pi + 0.35, n)
    inst["x_init"][:, L.ori + 1] = pitch
    inst["x_init"][:, L.ori + 2] = roll
    return inst


# every recipe: (name, builder(model, geo) -> instance, {(term, branch): minimum node x row count})
def recipes(model):
    cen = is_cen(model)
    horizon = 0.5 if cen else 0.8
    walk = lambda: _copy(base_instance(model, "walk", horizon))
    out = [
        ("collision_crossed", lambda g: cross_legs(model, walk(), 0.12, 0.26),
         {("collision", "h<=0"): 8, ("collision", "0<h<delta"): 8}),
        ("collision_knee", lambda g: knees_together(model, walk()),
         {("collision", "knee row alone"): 3}),
        ("joint_limits", lambda g: joints_at_limits(model, walk()),
         {("joint_limits", "h<=0"): 8, ("joint_limits", "0<h<delta"): 8}),
        ("friction_relaxed", lambda g: unload_feet(model, g, walk()),
         {("friction", "relaxed"): 6, ("friction", "log"): 6}),
        ("moment_relaxed", lambda g: edge_moments(model, g, walk()),
         {("moment", "relaxed"): 8}),
        ("rotated_contact", lambda g: edge_moments(model, g, unload_feet(model, g, rotate_base(model, walk(), 0.6, -0.6))),
         {("friction", "relaxed"): 4, ("moment", "relaxed"): 6}),
        ("rotated_collision", lambda g: cross_legs(model, rotate_base(model, walk(), -0.6, 0.6), 0.12, 0.26),
         {("collision", "h<=0"): 8, ("collision", "0<h<delta"): 8}),
        ("exact_thresholds", lambda g: exact_thresholds(model, walk()),
         {("joint_limits", "edge h=delta"): 8, ("joint_limits", "edge h=0"): 8, ("friction", "edge h=delta"): 4}),
    ]
    return out


def flight_recipe(model):
    """a run gait with the legs crossed: flight nodes evaluate all 16 collision rows"""
    return ("collision_flight", lambda g: cross_legs(model, _copy(base_instance(model, "run", 0.8, seed=13)), 0.12, 0.26),
            {("collision", "flight node active"): 2, ("collision", "h<=0"): 8})


def build_recipes(model, geo, with_flight=True):
    """[(name, instance, counts)], every recipe asserted to reach the branches it is for"""
    out = []
    for name, make, need in recipes(model) + ([flight_recipe(model)] if with_flight else []):
        inst = make(geo)
        cnt = geo.counts(inst)
        print(format_counts(name, cnt))
        for key, m in need.items():
            assert cnt[key] >= m, (name, key, cnt[key], m, format_counts(name, cnt))
        out.append((name, inst, cnt))
    return out


# ---- fixtures -----------------------------------------------------------------------------------------------------------------------------------

FAMILIES = ["g1_wb", "g1_centroidal"]


@pytest.fixture(scope="module", params=FAMILIES)
def model(request):
    return model_loader.load_packaged_model(request.param) if request.param != "g1_wb" else model_loader.load_packaged_model()


@pytest.fixture(scope="module")
def geo(model):
    return Geometry(model)


@pytest.fixture(scope="module")
def built(model, geo):
    return build_recipes(model, geo)


def new_oracle(model):
    return orc.CenOracle(model) if is_cen(model) else orc.WbOracle(model)


def node_oracle(model, inst, k, arm=None):
    """an oracle whose node 0 is node k of the instance (arm phase overridable)"""
    o = new_oracle(model)
    sl = slice(k, k + 1)
    o.set_nodes(inst["contact_flags"][sl], inst["swing_ref"][sl], inst["impact_factor"][sl],
                inst["arm_phase"][sl] if arm is None else np.array([arm]), inst["x_ref"][sl])
    return o


def without(model, term):
    """the model with one penalty term switched off (mu = 0)"""
    m = copy.deepcopy(model)
    m[{"joint_limits": "joint_limits", "collision": "collision", "friction": "friction", "moment": "moment_xy"}[term]]["mu"] = 0.0
    return m


def term_params(model, term):
    d = model[{"joint_limits": "joint_limits", "collision": "collision", "friction": "friction", "moment": "moment_xy"}[term]]
    return d["mu"], d["delta"]


def penalty_sum(model, term, h):
    mu, delta = term_params(model, term)
    f = pwpoly_exact if term in ("joint_limits", "collision") else relaxed_exact
    return float(sum((f(mu, delta, v)[0] for v in h), Fraction(0)))


# ---- 1. the penalty functions --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["pwpoly", "relaxed"])
@pytest.mark.parametrize("mu,delta", [(1500.0, 0.04), (1200.0, 0.1), (0.2, 5.0), (0.6, 0.03), (30000.0, 0.05)])
def test_device_penalty_functions_on_both_sides_of_every_threshold(kind, mu, delta):
    exact = pwpoly_exact if kind == "pwpoly" else relaxed_exact
    for h in threshold_points(delta):
        if kind == "relaxed" and h <= 0 and abs(h) < 1e-300:
            continue
        assert_penalty_close(emu.penalty(kind, mu, delta, h), mu, delta, h, exact(mu, delta, h), (kind, mu, delta))


def test_oracle_joint_limit_penalty_on_both_sides_of_every_threshold():
    """the oracle's piecewise-polynomial barrier through its cost: one knee joint at upper-limit distance h, all other joints far from their
    limits; the cost, gradient and Hessian entry of the knee differ from the model without the term by (v, -d1, d2) at h"""
    model = model_loader.load_packaged_model()
    mu, delta = term_params(model, "joint_limits")
    off = without(model, "joint_limits")
    qhi = model["q_upper"][3]
    u = np.zeros(35)
    for target in threshold_points(delta):
        x = np.array(model["x_init"], float)
        x[6 + 3] = qhi - target
        h = qhi - x[6 + 3]
        a, b = node_oracle(model, _single(model), 0), node_oracle(off, _single(model), 0)
        qa, qb = a.cost_quad(0, x, u), b.cost_quad(0, x, u)
        v, d1, d2 = pwpoly_exact(mu, delta, h)
        scale = max(1.0, abs(qa["f"]))
        assert abs((qa["f"] - qb["f"]) - float(v)) <= 1e-12 * scale + 4e-16 * mu * delta * delta, (h, qa["f"] - qb["f"], float(v))
        assert abs((a.cost(0, x, u) - b.cost(0, x, u)) - float(v)) <= 1e-12 * scale + 4e-16 * mu * delta * delta
        assert abs((qa["q"][9] - qb["q"][9]) - float(-d1)) <= 1e-12 * max(1.0, abs(qa["q"][9])) + 4e-16 * mu, (h, qa["q"][9] - qb["q"][9], -float(d1))
        dQ = qa["Q"] - qb["Q"]
        assert abs(dQ[9, 9] - float(d2)) <= 1e-12 * max(1.0, abs(qa["Q"][9, 9])), (h, dQ[9, 9], float(d2))
        dQ[9, 9] = 0.0
        assert not dQ.any()


def test_oracle_friction_penalty_on_both_sides_of_every_threshold():
    """the oracle's relaxed barrier through the friction cone of a stance foot without tangential force: h = mu_c fz - sqrt(reg); the cost,
    the fz gradient and the fz Hessian entry differ from the model without the term by v, mu_c d1 and mu_c^2 d2 - shift (d1 of both feet)"""
    model = model_loader.load_packaged_model()
    f = model["friction"]
    mu, delta, mu_c, reg, shift = f["mu"], f["delta"], f["mu_fric"], f["regularization"], f["hessian_shift"]
    off = without(model, "friction")
    inst = _single(model)
    x = np.array(model["x_init"], float)
    for target in threshold_points(delta):
        u = np.zeros(35)
        u[2] = (target + np.sqrt(reg)) / mu_c
        u[8] = 200.0
        h = mu_c * u[2] - np.sqrt(u[0] * u[0] + u[1] * u[1] + reg)
        hr = mu_c * u[8] - np.sqrt(reg)
        a, b = node_oracle(model, inst, 0), node_oracle(off, inst, 0)
        qa, qb = a.cost_quad(0, x, u), b.cost_quad(0, x, u)
        v, d1, d2 = relaxed_exact(mu, delta, h)
        vr, d1r, _ = relaxed_exact(mu, delta, hr)
        scale = max(1.0, abs(qa["f"]))
        assert abs((qa["f"] - qb["f"]) - float(v + vr)) <= 1e-12 * scale, (h, qa["f"] - qb["f"], float(v + vr))
        assert abs((qa["r"][2] - qb["r"][2]) - float(mu_c * d1)) <= 1e-12 * max(1.0, abs(qa["r"][2])), (h,)
        want = float(Fraction(mu_c) ** 2 * d2 - Fraction(shift) * (d1 + d1r))
        assert abs((qa["R"][2, 2] - qb["R"][2, 2]) - want) <= 1e-12 * max(1.0, abs(qa["R"][2, 2])), (h, qa["R"][2, 2] - qb["R"][2, 2], want)


def _single(model):
    """a one-node double-stance instance at the model's initial state (for the single-node oracle queries)"""
    xr = np.array(model["x_init"], float)[None]
    return dict(contact_flags=np.array([[1, 1]], dtype=np.uint8), swing_ref=np.zeros((1, 2, 3)), impact_factor=np.ones((1, 2)),
                arm_phase=np.zeros(1), x_ref=xr)


# ---- 2. the recipes reach their branches, and h is what the oracle penalises -------------------------------------------------------------------

def test_recipes_reach_their_branches_and_h_matches_the_oracle_cost(model, geo, built):
    """Each recipe reaches the branches it is built for (asserted in build_recipes), and the h computed here from oracle quantities is the h
    the oracle penalises: for every term, the cost of the model minus the cost of the model without that term equals the exact penalty sum."""
    total = Counter()
    for name, inst, cnt in built:
        total.update(cnt)
        for k in stage_nodes(inst)[::3]:
            x, u = inst["x_init"][k], inst["u_init"][k]
            vals = geo.node_values(inst, k)
            base = node_oracle(model, inst, k).cost(0, x, u)
            for term, h in vals.items():
                d = base - node_oracle(without(model, term), inst, k).cost(0, x, u)
                want = penalty_sum(model, term, h)
                assert abs(d - want) <= 1e-10 * max(1.0, abs(base)), (name, k, term, d, want)
    print(format_counts("all recipes", total))
    for term, branches in (("collision", ("h<=0", "0<h<delta", "off", "knee row alone", "flight node active")),
                           ("joint_limits", ("h<=0", "0<h<delta", "off", "edge h=0", "edge h=delta")),
                           ("friction", ("relaxed", "log", "edge h=delta")), ("moment", ("relaxed", "log"))):
        for b in branches:
            assert total[(term, b)] > 0, (term, b)


# ---- 3. the oracle's gradient and the Hessian of each term --------------------------------------------------------------------------------------

def _nz(model):
    return model["nx"], model["nu"]


def _fd(f, z, eps=1e-6):
    f0 = np.atleast_1d(f(z))
    J = np.zeros((len(f0), len(z)))
    for i in range(len(z)):
        zp, zm = z.copy(), z.copy()
        zp[i] += eps
        zm[i] -= eps
        J[:, i] = (np.atleast_1d(f(zp)) - np.atleast_1d(f(zm))) / (2 * eps)
    return J


def test_oracle_gradient_matches_finite_differences(model, built):
    """test_oracle_wb.py::test_cost_gradient_vs_finite_differences at the recipes' nodes, without the push into the log branch (arm phase 0:
    the quadratic cost treats its yaw-dependent arm-swing reference as constant)"""
    nx, nu = _nz(model)
    for name, inst, _ in built:
        for k in stage_nodes(inst)[1::7]:
            o = node_oracle(model, inst, k, arm=0.0)
            x, u = inst["x_init"][k], inst["u_init"][k]
            q = o.cost_quad(0, x, u)
            g = _fd(lambda z: o.cost(0, z[:nx], z[nx:]), np.concatenate([x, u]))[0]
            scale = max(1.0, np.max(np.abs(g)))
            assert np.max(np.abs(q["q"] - g[:nx])) < 1e-5 * scale, (name, k, np.max(np.abs(q["q"] - g[:nx])) / scale)
            assert np.max(np.abs(q["r"] - g[nx:])) < 1e-5 * scale, (name, k, np.max(np.abs(q["r"] - g[nx:])) / scale)


def _hess(q):
    return np.block([[q["Q"], q["S"].T], [q["S"], q["R"]]])


def expected_term(model, geo, term, x, u, cf):
    """NumPy Gauss-Newton assembly of one term (the reference's SoftConstraintPenalty on a first-order constraint): gradient sum d1 J and
    Hessian sum d2 J'J, J by central differences of h; the friction cone is the quadratic-order constraint d2 dh dh' + d1 ddh (+ the Hessian
    shift -fricShift (d1_0 + d1_1) on the whole diagonal); joint limits are diagonal"""
    nx, nu = _nz(model)
    nz = nx + nu
    mu, delta = term_params(model, term)
    z0 = np.concatenate([x, u])
    g, H = np.zeros(nz), np.zeros((nz, nz))
    if term in ("collision", "moment"):
        if term == "collision":
            fn = lambda z: geo.collision(z[:nx], z[nx:])
        else:
            fn = lambda z: np.concatenate([geo.moment(z[:nx], z[nx:], c) for c in range(2) if cf[c]])
        h = fn(z0)
        J = _fd(fn, z0)
        pen = pwpoly_exact if term == "collision" else relaxed_exact
        for r in range(len(h)):
            _, d1, d2 = (float(v) for v in pen(mu, delta, h[r]))
            g += d1 * J[r]
            H += d2 * np.outer(J[r], J[r])
    elif term == "friction":
        f = model["friction"]
        for c in range(2):
            if not cf[c]:
                continue
            F = u[6 * c:6 * c + 3]
            Ft2 = F[0] ** 2 + F[1] ** 2 + f["regularization"]
            Ft = np.sqrt(Ft2)
            _, d1, d2 = (float(v) for v in relaxed_exact(mu, delta, f["mu_fric"] * F[2] - Ft))
            dh = np.array([-F[0] / Ft, -F[1] / Ft, f["mu_fric"]])
            ddh = np.zeros((3, 3))
            ddh[:2, :2] = np.array([[-(F[1] ** 2 + f["regularization"]), F[0] * F[1]], [F[0] * F[1], -(F[0] ** 2 + f["regularization"])]]) / (Ft * Ft2)
            i = nx + 6 * c
            g[i:i + 3] += d1 * dh
            H[i:i + 3, i:i + 3] += d2 * np.outer(dh, dh) + d1 * ddh
            H[np.diag_indices(nz)] += -f["hessian_shift"] * d1
    else:
        q0 = 12 if geo.cen else 6
        h = geo.joint_limits(x)
        nj = len(h) // 2
        for j in range(nj):
            _, d1u, d2u = (float(v) for v in pwpoly_exact(mu, delta, h[j]))
            _, d1l, d2l = (float(v) for v in pwpoly_exact(mu, delta, h[nj + j]))
            g[q0 + j] += d1l - d1u
            H[q0 + j, q0 + j] += d2u + d2l
    return g, H


def test_each_term_hessian_is_the_gauss_newton_assembly(model, geo, built):
    """cost_quad(model) - cost_quad(model with the term's mu = 0) against expected_term at nodes of every recipe; FD Jacobians: 1e-6 of the
    term's largest entry"""
    nx, nu = _nz(model)
    for name, inst, _ in built:
        for k in stage_nodes(inst)[2::6]:
            x, u, cf = inst["x_init"][k], inst["u_init"][k], inst["contact_flags"][k]
            qa = node_oracle(model, inst, k).cost_quad(0, x, u)
            for term, h in geo.node_values(inst, k).items():
                if not len(h):
                    continue
                qb = node_oracle(without(model, term), inst, k).cost_quad(0, x, u)
                g = np.concatenate([qa["q"] - qb["q"], qa["r"] - qb["r"]])
                H = _hess(qa) - _hess(qb)
                ge, He = expected_term(model, geo, term, x, u, cf)
                sg, sh = max(1e-9, np.max(np.abs(ge))), max(1e-9, np.max(np.abs(He)))
                tol = 1e-6 if term in ("collision", "moment") else 1e-10
                assert np.max(np.abs(g - ge)) <= tol * sg + 1e-9 * max(1.0, np.max(np.abs(qa["q"]))), (name, k, term, "gradient")
                assert np.max(np.abs(H - He)) <= tol * sh + 1e-12 * np.max(np.abs(_hess(qa))), (name, k, term, "Hessian", np.max(np.abs(H - He)), sh)


# ---- 4. the CPU harness against the oracle on every node of every recipe -------------------------------------------------------------------------

KEYS = ["A", "B", "b", "Q", "S", "R", "q", "r", "C", "D", "e"]


def rel(a, b):
    return np.max(np.abs(a - b)) / max(1e-12, np.max(np.abs(b))) if b.size else 0.0


def interval_duration(inst, k):
    """getIntervalDuration (ocs2_sqp TimeDiscretization.cpp): a post-event node starts and a pre-event node ends numeric_traits::weakEpsilon
    inside the interval"""
    t, ev = inst["t_nodes"], inst["node_event"]
    return (t[k + 1] - (1e-9 if ev[k + 1] == 1 else 0.0)) - (t[k] + (1e-9 if ev[k] == 2 else 0.0))


def oracle_raw(model, inst):
    o = new_oracle(model)
    o.set_nodes(inst["contact_flags"], inst["swing_ref"], inst["impact_factor"], inst["arm_phase"], inst["x_ref"])
    st = abi.default_settings(model, sqp_iteration=1)
    o.sqp(inst["t_nodes"], inst["node_event"], inst["x0"], inst["x_init"], inst["u_init"], st, keep_raw=True)
    return o.last_raw_blocks(len(inst["t_nodes"])), o


def test_harness_lq_node_matches_oracle_on_every_recipe(model, built):
    """whole-body: emu.lq_node in the one-pass schedule and in both CUDA K1b schedules (mode 1, 2); centroidal: emu.cen_node.  Raw blocks
    1e-10 relative (the whole-body tolerance of tests/test_emu_k1.py; test_emu_cen.py allows 1e-9, which these nodes do not need)."""
    worst = Counter()
    for name, inst, _ in built:
        raw, o = oracle_raw(model, inst)
        for k in stage_nodes(inst):
            args = (inst["x_init"][k], inst["u_init"][k], inst["x_init"][k + 1], inst["x_ref"][k], interval_duration(inst, k), inst["contact_flags"][k],
                    inst["swing_ref"][k], inst["impact_factor"][k], inst["arm_phase"][k])
            outs = [emu.cen_node(o.desc, o.cdesc, *args)] if is_cen(model) else [emu.lq_node(o.desc, *args, mode=m) for m in (0, 1, 2)]
            for mode, e in enumerate(outs):
                assert e["raw"]["nc"] == raw[k]["nc"], (name, k)
                for key in KEYS:
                    d = rel(e["raw"][key], raw[k][key])
                    worst[key] = max(worst[key], d)
                    assert d < 1e-10, (name, k, mode, key, d)
                assert abs(e["raw"]["c"] - raw[k]["c"]) < 1e-10 * max(1.0, abs(raw[k]["c"])), (name, k, mode)
    print("largest relative differences, harness against oracle: " + ", ".join(f"{k} {v:.1e}" for k, v in worst.items()))
