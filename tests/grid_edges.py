"""Inputs that put gait events on the edges of timeDiscretizationWithEvents (references.time_discretization_with_events, bldGridInstance in
wb_humanoid_mpc_b200/csrc/wb_builder.cuh), shared by tests/test_emu_grid_edges.py (CPU harness) and tests/test_gpu_grid_edges.py (C ABI).

The grid accumulates t0 + dt + dt + ... until the next event, takes the event instead of any node at or past it, restarts the accumulation
from the event, replaces the last node when the new one lies within dtMin = 1e-5 of it, and ends at tf.  A recipe is (family, gait, gait_start,
t0): the gait's template tiled from gait_start (an event at exactly gait_start, the next ones accumulated from it) on the horizon of the family.
The search places one event on a chosen branch, to the last bit where the branch is an exact float comparison, and `trace` replays the grid
loop to record which branches the recipe reaches; every recipe asserts that its own branch is among them."""
from __future__ import annotations

import bisect
import copy
from collections import Counter

import numpy as np

from wb_humanoid_mpc_b200 import model_loader, references

DT_MIN = 10.0 * references.LIMIT_EPS
WEAK_EPS = references.WEAK_EPS
EV_NONE, EV_PRE, EV_POST = references.EV_NONE, references.EV_PRE, references.EV_POST
# (packaged model name, dt, horizon) of the two OCP families
FAMILIES = {"wb": (None, 0.035, 1.1), "cen": ("g1_centroidal", 0.02, 1.2)}
# the 14 templates of gait.info the device table holds ("skip" is refused: its switching times decrease)
DEVICE_GAITS = ("stance", "left_leg", "right_leg", "trot", "fast_trot", "slow_trot", "slower_trot", "walk", "fast_walk", "slow_walk", "very_slow_walk",
                "run", "fast_run", "jump")
# gait.info has no phase shorter than 0.1 s, so no two of its events are one grid step apart; this run-like template (appended to the gait table
# of the model, which the builder ABI accepts) has flight phases of 0.6 dt
SHORT_FLIGHT = "short_flight_run"
BRANCHES = ("event_on_node", "event_ulp_before_node", "event_ulp_after_node", "gap_dtmin_minus_ulp", "gap_dtmin", "gap_dtmin_plus_ulp",
            "short_stage_before_event", "short_stage_after_event", "event_at_t0", "event_at_tf", "event_near_tf", "events_within_dt",
            "restart_from_event")
# ulp-exact branches: the recipes that hit the grid loop's float comparisons on the nose
T0 = 0.0125   # the initial time of every recipe: one cycle of an 80 Hz MPC after t = 0
EXACT = {"event_on_node", "event_ulp_before_node", "event_ulp_after_node", "gap_dtmin_minus_ulp", "gap_dtmin", "gap_dtmin_plus_ulp", "event_at_t0",
         "event_at_tf"}


def load_model(family):
    """the packaged model of the family with the short-flight template appended to its gait table"""
    name, dt, _ = FAMILIES[family]
    m = model_loader.load_packaged_model() if name is None else model_loader.load_packaged_model(name)
    m = copy.deepcopy(m)
    assert m["sqp"]["dt"] == dt
    f = 0.6 * dt
    m["gaits"][SHORT_FLIGHT] = dict(modeSequence=["LF", "FLY", "RF", "FLY"], switchingTimes=[0.0, 0.3, 0.3 + f, 0.6 + f, 0.6 + 2 * f])
    return m


def events(model, gait, gait_start, t0, horizon):
    """the event times build_instance discretises: the gait tiled from gait_start, then getModeSchedule(t0 - T, tf + T)"""
    tf = t0 + horizon
    gs = references.GaitSchedule()
    if gait != "stance":
        g = model["gaits"][gait]
        gs.insert_template([references.MODE_NAMES[m] for m in g["modeSequence"]], g["switchingTimes"], gait_start, tf + horizon)
    return gs.get_mode_schedule(t0 - horizon, tf + horizon).event_times


def trace(t0, tf, dt, ev):
    """the loop of time_discretization_with_events, replayed -> (times, event kinds, Counter of branches hit).  Only events inside [t0, tf]
    count; the grid itself must equal the restatement's (checked by the caller)."""
    hits = Counter()
    up, down = lambda v: np.nextafter(v, np.inf), lambda v: np.nextafter(v, -np.inf)
    idx = bisect.bisect_left(ev, t0)
    if idx < len(ev) and ev[idx] == t0:
        hits["event_at_t0"] += 1
    inside = [e for e in ev if t0 <= e <= tf]
    hits["events_within_dt"] += sum(b - a <= dt for a, b in zip(inside, inside[1:]))
    td = [[t0, EV_NONE]]
    nxt = t0
    while td[-1][0] < tf:
        cand = nxt + dt
        if idx < len(ev) and ev[idx] <= tf:
            e = ev[idx]
            hits["event_on_node"] += e == cand
            hits["event_ulp_before_node"] += e == down(cand)
            hits["event_ulp_after_node"] += e == up(cand)
        nxt, kind = cand, EV_NONE
        if idx < len(ev) and nxt >= ev[idx]:
            nxt, kind = ev[idx], EV_PRE
            idx += 1
            thr = td[-1][0] + DT_MIN
            hits["gap_dtmin_minus_ulp"] += nxt == down(thr)
            hits["gap_dtmin"] += nxt == thr
            hits["gap_dtmin_plus_ulp"] += nxt == up(thr)
            hits["event_at_tf"] += nxt == tf
            hits["event_near_tf"] += tf - DT_MIN < nxt < tf
            hits["restart_from_event"] += nxt < tf
        if nxt >= tf:
            nxt, kind = tf, EV_NONE
        if nxt > td[-1][0] + DT_MIN:
            td.append([nxt, kind])
        else:
            td[-1] = [nxt, kind]
    if td[0][1] == EV_PRE:
        td[0][1] = EV_POST
    t, e = [], []
    for ti, ei in td:
        t.append(ti)
        e.append(ei)
        if ei == EV_PRE:
            t.append(ti)
            e.append(EV_POST)
    for k in range(len(t) - 1):
        if 0.0 < t[k + 1] - t[k] < 2.0 * DT_MIN:
            hits["short_stage_before_event"] += e[k + 1] == EV_PRE
            hits["short_stage_after_event"] += e[k] == EV_POST
    return np.array(t), np.array(e, np.uint8), +hits


def grid_nodes(t0, dt, k):
    """the k-th accumulated node t0 + dt + ... + dt of a grid that meets no event before it"""
    c = t0
    for _ in range(k):
        c = c + dt
    return c


def solve_ulps(f, x, target, span=512):
    """an input within span ulps of x with f(input) == target, or None (the roundings of an accumulated sum can step over the target)"""
    lo = hi = x
    if f(x) == target:
        return x
    for _ in range(span):
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        for v in (lo, hi):
            if f(v) == target:
                return v
    return None


def tiled_event(model, gait, gait_start, j):
    """the j-th event of the gait tiled from gait_start, accumulated as GaitSchedule's tiling does"""
    t = model["gaits"][gait]["switchingTimes"]
    m = len(t) - 1
    e = gait_start
    for i in range(j):
        e = e + (t[i % m + 1] - t[i % m])
    return e


def _before(model, gait, target, j0=1):
    """the first event index j >= j0 whose gait start, for event j at target, obeys the builder's bound gait_start <= 0.5"""
    j = j0
    while target - (tiled_event(model, gait, 0.0, j)) > 0.5:
        j += 1
    return j


def recipe(family, model, gait, branch, k=6):
    """-> dict(family, gait, branch, gait_start, t0, horizon) that reaches `branch`.  Every recipe of a family has the same t0 (T0), so that
    all of them go into one fleet build; k: the accumulated node the event is placed against (or, against tf, the event index)."""
    _, dt, H = FAMILIES[family]
    t0 = T0
    tf = t0 + H
    c = grid_nodes(t0, dt, k)
    if branch == "event_on_node":
        gs = c
    elif branch == "event_ulp_before_node":
        gs = np.nextafter(c, -np.inf)
    elif branch == "event_ulp_after_node":
        gs = np.nextafter(c, np.inf)
    elif branch in ("gap_dtmin_minus_ulp", "gap_dtmin", "gap_dtmin_plus_ulp"):
        thr = c + DT_MIN
        gs = {"gap_dtmin_minus_ulp": np.nextafter(thr, -np.inf), "gap_dtmin": thr, "gap_dtmin_plus_ulp": np.nextafter(thr, np.inf)}[branch]
    elif branch == "short_stage_before_event":
        gs = c + 1.1 * DT_MIN
    elif branch in ("events_within_dt", "restart_from_event"):
        gs = c + 0.37 * dt
    elif branch == "event_at_t0":
        gs = t0
    else:   # against tf: event j of the tiled gait placed by moving gait_start
        target = {"event_at_tf": tf, "event_near_tf": tf - 0.5 * DT_MIN, "short_stage_after_event": tf - 1.1 * DT_MIN}[branch]
        j = _before(model, gait, target, k)
        gs = None
        while gs is None:   # exactly on tf: the first event index at which some gait start lands there
            g0 = target - tiled_event(model, gait, 0.0, j)
            gs = solve_ulps(lambda g: tiled_event(model, gait, g, j), g0, target) if branch == "event_at_tf" else g0
            j += 1
    return dict(family=family, gait=gait, branch=branch, gait_start=float(gs), t0=float(t0), horizon=H)


# (branch, gait, k) of the recipes of each family: every branch on a multi-phase gait, the ulp-exact ones on two
PLAN = {
    "wb": [("event_on_node", "walk", 6), ("event_on_node", "run", 9), ("event_ulp_before_node", "walk", 7), ("event_ulp_before_node", "fast_run", 11),
           ("event_ulp_after_node", "run", 5), ("event_ulp_after_node", "fast_walk", 8), ("gap_dtmin_minus_ulp", "walk", 9),
           ("gap_dtmin", "trot", 4), ("gap_dtmin_plus_ulp", "run", 12), ("short_stage_before_event", "walk", 10),
           ("short_stage_before_event", "right_leg", 3), ("short_stage_after_event", "run", 2), ("event_at_t0", "walk", 1),
           ("event_at_tf", "run", 3), ("event_at_tf", "slow_trot", 5), ("event_near_tf", "fast_walk", 4), ("events_within_dt", SHORT_FLIGHT, 3)],
    "cen": [("event_on_node", "walk", 10), ("event_on_node", "run", 17), ("event_ulp_before_node", "run", 12), ("event_ulp_before_node", "fast_trot", 19),
            ("event_ulp_after_node", "walk", 15), ("event_ulp_after_node", "very_slow_walk", 8), ("gap_dtmin_minus_ulp", "run", 14),
            ("gap_dtmin", "walk", 21), ("gap_dtmin_plus_ulp", "slow_walk", 7), ("short_stage_before_event", "run", 11),
            ("short_stage_before_event", "right_leg", 6), ("short_stage_after_event", "walk", 2), ("event_at_t0", "run", 1),
            ("event_at_tf", "walk", 3), ("event_at_tf", "fast_run", 6), ("event_near_tf", "trot", 4), ("events_within_dt", SHORT_FLIGHT, 9)],
}


def name(r):
    return f"{r['family']}-{r['branch']}-{r['gait']}"


def recipes(family, model):
    """the recipes of PLAN, each checked to reach its branch and to give the restatement's grid -> [(recipe, hits)]"""
    out = []
    _, dt, _ = FAMILIES[family]
    for branch, gait, k in PLAN[family]:
        r = recipe(family, model, gait, branch, k)
        assert r["gait_start"] <= 0.5, (name(r), r["gait_start"])   # the builder ABI's bound (the default schedule's first event)
        tf = r["t0"] + r["horizon"]
        ev = events(model, gait, r["gait_start"], r["t0"], r["horizon"])
        t, e, hits = trace(r["t0"], tf, dt, ev)
        rt, re_ = references.time_discretization_with_events(r["t0"], tf, dt, ev)
        assert np.array_equal(t, rt) and np.array_equal(e, re_), name(r)
        assert hits[branch] > 0, (name(r), dict(hits))
        out.append((r, hits))
    return out


def branch_counts(built):
    total = Counter()
    for _, hits in built:
        total.update(hits)
    return total


def format_counts(family, total):
    return f"{family}: " + ", ".join(f"{b} {total[b]}" for b in BRANCHES)


def build_host(model, r, x0, cmd=None, previous=None, t0=None):
    """references.build_instance of a recipe (t0: a warm build's later initial time)"""
    return references.build_instance(model, x0, t0=r["t0"] if t0 is None else t0, horizon=r["horizon"], gait=r["gait"], gait_start=r["gait_start"],
                                     cmd=cmd, previous=previous)


def x0_of(model, rng):
    """a measured state near the model's initial state (zero momentum on the centroidal family)"""
    x0 = np.array(model["x_init"], float)
    if model.get("kind") == "centroidal":
        x0[6:8] += rng.uniform(-0.02, 0.02, 2)
        x0[9:12] += rng.uniform(-0.05, 0.05, 3)
        x0[12:] += rng.uniform(-0.1, 0.1, model["nj"])
    else:
        x0[2] = model["reference"]["defaultBaseHeight"]
        x0[0:2] += rng.uniform(-0.02, 0.02, 2)
        x0[3:6] += rng.uniform(-0.05, 0.05, 3)
        x0[6:29] += rng.uniform(-0.1, 0.1, 23)
        x0[29:] += rng.uniform(-0.2, 0.2, 29)
    return x0


def sub_dt_stages(inst):
    """stage indices k whose interval [t_k, t_k+1] is shorter than dtMin * 2 (and not the zero-length event stage)"""
    t = inst["t_nodes"]
    return [k for k in range(len(t) - 1) if 0.0 < t[k + 1] - t[k] < 2.0 * DT_MIN]


def projected_qp(model, inst, raw, P_N, p_N, reg):
    """the QP of one SQP iteration from its raw stage blocks (oracle or device layout, unpacked), each stage's constraints eliminated with the
    oracle's LU projection (du = Pu du~ + Px dx + u0) -> (riccati_ref arguments, [(Pu, Px, u0)] per stage).  Event (PreEvent) stages have no
    input.  P_N, p_N: the terminal cost-to-go of the value function (P_N = Q_N + reg I)."""
    import oracle_lib as orc

    N, nx, nu = len(inst["t_nodes"]) - 1, model["nx"], model["nu"]
    A, Bm, b = np.zeros((N, nx, nx)), np.zeros((N, nx, nu)), np.zeros((N, nx))
    Q, S, R = np.zeros((N + 1, nx, nx)), np.zeros((N, nu, nx)), np.zeros((N, nu, nu))
    q, r, n_in, proj = np.zeros((N + 1, nx)), np.zeros((N, nu)), np.zeros(N, np.int32), []
    for k in range(N):
        g = raw[k]
        if inst["node_event"][k] == EV_PRE:
            A[k], b[k], Q[k], q[k] = g["A"], g["b"], g["Q"], g["q"]
            proj.append(None)
            continue
        Pu, Px, u0, _ = orc.lu_projection(g["C"], g["D"], g["e"]) if g["nc"] else (np.eye(nu), np.zeros((nu, nx)), np.zeros(nu), 0)
        pr = orc.change_of_input_variables(g["A"], g["B"], g["b"], g["Q"], g["S"], g["R"], g["q"], g["r"], g["c"], Pu, Px, u0)
        m = Pu.shape[1]
        A[k], b[k], Q[k], q[k] = pr["A"], pr["b"], pr["Q"], pr["q"]
        Bm[k][:, :m], S[k][:m], R[k][:m, :m], r[k][:m] = pr["B"], pr["S"], pr["R"], pr["r"]
        n_in[k] = m
        proj.append((Pu, Px, u0))
    Q[N], q[N] = P_N - reg * np.eye(nx), p_N
    return (A, Bm, b, Q, S, R, q, r), n_in, proj


def to_input_space(sol, n_in, proj, nu):
    """a Riccati solution in the eliminated inputs -> (dx, du, K) in the model's inputs (K [N, nu, nx]; zero on event stages)"""
    dx = np.asarray(sol["dx"], dtype=np.longdouble)
    N, nx = len(proj), dx.shape[1]
    du, K = np.zeros((N, nu), dtype=np.longdouble), np.zeros((N, nu, nx), dtype=np.longdouble)
    for k, p in enumerate(proj):
        if p is None:
            continue
        Pu, Px, u0 = (np.asarray(a, dtype=np.longdouble) for a in p)
        m = n_in[k]
        du[k] = Pu @ np.asarray(sol["du"][k][:m], dtype=np.longdouble) + Px @ dx[k] + u0
        K[k] = Pu @ np.asarray(sol["K"][k][:m], dtype=np.longdouble) + Px
    return dx, du, K


def rel_ld(a, b):
    """max |a - b| / max(1, max |b|), in np.longdouble"""
    a, b = np.asarray(a, dtype=np.longdouble), np.asarray(b, dtype=np.longdouble)
    return float(np.max(np.abs(a - b)) / max(np.longdouble(1), np.max(np.abs(b))))
